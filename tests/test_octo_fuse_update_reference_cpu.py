"""Pins tests/octo_fuse_update_reference.py (the numpy statement of tslam_octo_fuse_update) on hand-worked cases, and
against octo_logodds_reference.fuse and the CPU oracle's orc_octo_fuse."""
import numpy as np
import pytest

import octo_logodds_reference as lr
import octo_fuse_update_reference as ofr

I3 = np.eye(3)


def test_half_ties_round_away_from_zero_and_negative_cells():
    # vs = 0.5 is exact: (i vs + 0.25) / vs = i + 0.5 exactly
    idx = np.array([[0, 0, 0], [-1, -1, -1], [2, -3, 1]])
    c = ofr.place(idx, I3, [0.25, -0.25, 0.25], 0.5)
    assert c.tolist() == [[1, -1, 1], [-1, -2, -1], [3, -4, 2]]


def test_cells_outside_the_volume_are_dropped():
    rows = {0: (np.array([[1, 0, 0], [0, 0, 0], [-2, 0, 0]]), np.array([5, 6, 7], np.uint32), None)}
    idx, cnt, _ = ofr.fuse(rows, {0: (I3, [0.5, 0.0, 0.0])}, 0.5, 4, 4, thres=3)  # i in [-2, 2); +1 cell
    assert idx.tolist() == [[-1, 0, 0], [1, 0, 0]] and cnt.tolist() == [7, 6]


def test_hit_threshold_and_sums():
    rows = {0: (np.array([[0, 0, 0], [1, 1, 1]]), np.array([3, 4], np.uint32), None),
            1: (np.array([[0, 0, 0], [1, 1, 1]]), np.array([9, 5], np.uint32), None)}
    poses = {0: (I3, [0, 0, 0]), 1: (I3, [0, 0, 0])}
    idx, cnt, _ = ofr.fuse(rows, poses, 0.1, 16, 16, thres=3)
    assert idx.tolist() == [[0, 0, 0], [1, 1, 1]] and cnt.tolist() == [9, 9]   # c = 3 is not > 3
    idx, cnt, _ = ofr.fuse(rows, poses, 0.1, 16, 16, thres=3, include={0})
    assert idx.tolist() == [[1, 1, 1]] and cnt.tolist() == [4]


def test_hit_sums_wrap_mod_2_32():
    rows = {0: (np.array([[0, 0, 0]]), np.array([0xFFFFFFF0], np.uint32), None),
            1: (np.array([[0, 0, 0]]), np.array([0x20], np.uint32), None)}
    poses = {0: (I3, [0, 0, 0]), 1: (I3, [0, 0, 0])}
    _, cnt, _ = ofr.fuse(rows, poses, 0.1, 16, 16, thres=3)
    assert cnt.tolist() == [0x10]


def test_logodds_sum_clamped_once_and_brought_back_by_a_removal():
    rows = {s: (np.array([[2, 2, 2]]), np.array([L], np.int32), None) for s, L in enumerate([3000, 3000, -2000])}
    poses = {s: (I3, [0, 0, 0]) for s in range(3)}
    kw = dict(model="logodds", l_min=-2048, l_max=3595)
    assert ofr.fuse(rows, poses, 0.1, 16, 16, **kw)[1].tolist() == [3595]           # 4000 -> l_max
    assert ofr.fuse(rows, poses, 0.1, 16, 16, include={0, 2}, **kw)[1].tolist() == [1000]
    assert ofr.fuse(rows, poses, 0.1, 16, 16, include={0, 1}, **kw)[1].tolist() == [3595]
    assert ofr.fuse(rows, poses, 0.1, 16, 16, include={2}, **kw)[1].tolist() == [-2000]
    # the sum word and its readout
    co = ofr.sum_word(3, 4000)
    assert ofr.readout(co, -2048, 3595) == (3595 << 1) | 1
    assert ofr.readout(co - ofr.sum_word(1, 3000), -2048, 3595) == (1000 << 1) | 1
    assert ofr.readout(ofr.sum_word(1, -5000), -2048, 3595) == ((-2048 << 1) | 1) & 0xFFFFFFFF
    assert ofr.readout(ofr.sum_word(0, 0), -2048, 3595) == 0


def test_colour_max_and_its_recompute_after_a_removal():
    w1, w2 = (5 << 24) | 0x102030, (9 << 24) | 0x0A0B0C
    rows = {0: (np.array([[0, 0, 0]]), np.array([7], np.uint32), np.array([w1], np.uint64)),
            1: (np.array([[0, 0, 0]]), np.array([7], np.uint32), np.array([w2], np.uint64)),
            2: (np.array([[0, 0, 0]]), np.array([2], np.uint32), np.array([(12 << 24) | 1], np.uint64))}  # below the threshold
    poses = {s: (I3, [0, 0, 0]) for s in range(3)}
    assert ofr.fuse(rows, poses, 0.1, 16, 16, thres=3)[2].tolist() == [w2]
    assert ofr.fuse(rows, poses, 0.1, 16, 16, thres=3, include={0, 2})[2].tolist() == [w1]


def test_agrees_with_the_logodds_reference_fusion():
    rng = np.random.default_rng(3)
    vs = 0.1
    src = lr.LogoddsMap(64, 64, vs)
    poses = {}
    for s in range(3):
        for f in range(2):
            xyz = rng.uniform(-2.0, 2.0, (300, 3)).astype(np.float32)
            src.integrate_points(xyz, I3, rng.uniform(-0.2, 0.2, 3), submap=s)
        a = rng.uniform(-0.5, 0.5)
        R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
        poses[s] = (R, rng.uniform(-0.5, 0.5, 3))
    dst = lr.LogoddsMap(64, 64, vs)
    lr.fuse(dst, src, poses)
    gi, gL = dst.gather(0)
    rows = {s: src.gather(s) + (None,) for s in range(3)}
    idx, L, _ = ofr.fuse(rows, poses, vs, 64, 64, model="logodds", l_min=src.p["l_min"], l_max=src.p["l_max"])
    idx, L = ofr.sorted_rows(idx, L)
    gi, gL = ofr.sorted_rows(gi, gL)
    assert np.array_equal(idx, gi) and np.array_equal(L, gL)


def test_agrees_with_the_oracle_fusion():
    oracle = pytest.importorskip("oracle.oracle")
    rng = np.random.default_rng(5)
    src = oracle.OracleOctomap(map_scale=(6.4, 6.4), voxel_scale=0.1, min_occupy_thres=1)
    dst = oracle.OracleOctomap(map_scale=(6.4, 6.4), voxel_scale=0.1, min_occupy_thres=1)
    poses = {}
    for s in range(3):
        for f in range(3):
            xyz = rng.uniform(-1.0, 1.0, (400, 3)).astype(np.float32)
            xyz[:200] = np.round(xyz[:200] * 4) / 4  # repeated points: counts above the threshold
            src.integrate_points(I3, np.zeros(3), xyz, submap=s)
        a = rng.uniform(-0.7, 0.7)
        R = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
        poses[s] = (R, rng.uniform(-0.4, 0.4, 3))
        dst.set_submap_pose(s, *poses[s])
    dst.fuse_from(src)
    oi, oc = dst.gather(0)
    rows = {s: src.gather(s) + (None,) for s in range(3)}
    idx, cnt, _ = ofr.fuse(rows, poses, 0.1, src.N, src.Nz, thres=1)
    assert idx.shape[0] > 100
    a = ofr.sorted_rows(idx, cnt)
    b = ofr.sorted_rows(oi, oc)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
