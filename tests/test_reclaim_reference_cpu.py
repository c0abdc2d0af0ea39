"""The numpy statement of tslam_tsdf_reclaim (tests/reclaim_reference.py) on hand-worked cases: the sphere test at and
just past contact, negative block coordinates, submaps 0 and 1023, masks, everything and nothing dropped, and every
kept block above n_keep."""
import numpy as np

import reclaim_reference as rr

VS = 0.05


def test_block_touching_the_sphere_is_kept_and_one_just_outside_is_dropped():
    # block bx = 1 spans voxel positions 16 * 0.05 .. 31 * 0.05 (f32 products, widened); centre on the x axis below it
    lo = float(np.float32(16) * np.float32(VS))
    keys = np.array([[0, 1, 0, 0]], np.int64)
    c = np.array([lo - 0.5, 0.0, 0.0])
    r_touch = lo - c[0]                                   # exact in f64: the distance to the block's nearest voxel
    assert rr.outside(keys, c, r_touch, VS).tolist() == [False]
    assert rr.outside(keys, c, np.nextafter(r_touch, 0.0), VS).tolist() == [True]
    # inside the span on y and z: only the x gap counts; the block's y, z span [0, 15 vs] contains 0
    assert rr.axis_d2(0.0, 0, VS) == 0.0 and rr.axis_d2(0.75, 0, VS) == 0.0
    assert rr.axis_d2(float(np.float32(15) * np.float32(VS)) + 0.25, 0, VS) == 0.25 * 0.25


def test_negative_block_coordinates():
    # block -1 spans voxels -16 .. -1: positions -0.8 .. -0.05 (f32); the centre at the origin is 0.05 away
    keys = np.array([[3, -1, 0, 0], [3, -2, 0, 0], [3, 0, -1, -1]], np.int64)
    hi = float(np.float32(-1) * np.float32(VS))
    d_m1 = 0.0 - hi
    r = d_m1
    out = rr.outside(keys, [0.0, 0.0, 0.0], r, VS)
    # block -2 ends at voxel -17: position -0.85 > r away; (0, -1, -1) is sqrt(2) * 0.05 away
    assert out.tolist() == [False, True, True]
    assert rr.outside(keys[2:], [0.0, 0.0, 0.0], np.sqrt(2.0 * d_m1 * d_m1), VS).tolist() == [False]


def test_submaps_0_and_1023_and_masks():
    keys = np.array([[0, 0, 0, 0], [1023, 0, 0, 0], [5, 0, 0, 0], [1023, 2, 0, 0]], np.int64)
    empty = np.array([True, True, False, True])
    keep, order, st = rr.reclaim(keys, empty, rr.EMPTY)
    assert keep.tolist() == [False, False, True, False]
    assert order.tolist() == [2] and st.tolist() == [4, 4, 3, 0, 1, 1]
    mask = np.zeros(1024, bool)
    mask[1023] = True
    keep, order, st = rr.reclaim(keys, empty, rr.EMPTY, mask=mask)
    assert keep.tolist() == [True, False, True, False]
    # n_keep 2: hole 1, mover 2
    assert order.tolist() == [0, 2] and st.tolist() == [4, 2, 2, 0, 1, 2]
    keep, order, st = rr.reclaim(keys, empty, rr.ALL, mask=mask)
    assert keep.tolist() == [True, False, True, False] and st[3] == 0
    mask0 = np.zeros(1024, bool)
    mask0[0] = True
    keep, order, st = rr.reclaim(keys, empty, rr.ALL, mask=mask0)
    assert keep.tolist() == [False, True, True, True]
    assert order.tolist() == [3, 1, 2] and st.tolist() == [4, 1, 1, 0, 1, 3]


def test_everything_and_nothing_dropped():
    keys = np.array([[0, i, -i, 2 * i] for i in range(6)], np.int64)
    empty = np.array([False, True, False, True, False, False])
    keep, order, st = rr.reclaim(keys, empty, rr.ALL)
    assert not keep.any() and order.tolist() == [] and st.tolist() == [6, 6, 6, 4, 0, 0]
    keep, order, st = rr.reclaim(keys, np.zeros(6, bool), rr.EMPTY)
    assert keep.all() and order.tolist() == list(range(6)) and st.tolist() == [6, 6, 0, 0, 0, 6]
    keep, order, st = rr.reclaim(keys, empty, rr.OUTSIDE, center=[0.0, 0.0, 0.0], radius=1e9)
    assert keep.all() and st[2] == 0


def test_all_kept_blocks_above_n_keep():
    # the first three slots dropped, the last three kept: every kept block moves, in ascending order
    keys = np.array([[1, i, 0, 0] for i in range(6)], np.int64)
    empty = np.array([True, True, True, False, False, False])
    keep, order, st = rr.reclaim(keys, empty, rr.EMPTY)
    n_keep, pairs, _ = rr.compact(keep)
    assert n_keep == 3 and pairs.tolist() == [[0, 3], [1, 4], [2, 5]]
    assert order.tolist() == [3, 4, 5] and st.tolist() == [6, 6, 3, 0, 3, 3]


def test_mixed_rules_and_interleaved_holes():
    rng = np.random.default_rng(7)
    n = 200
    keys = np.stack([rng.integers(0, 4, n), rng.integers(-20, 20, n), rng.integers(-20, 20, n), rng.integers(-3, 3, n)], 1)
    empty = rng.random(n) < 0.3
    mask = np.array([True, True, False, True])
    keep, order, st = rr.reclaim(keys, empty, rr.EMPTY | rr.OUTSIDE, mask=mask, center=[0.1, -0.2, 0.0], radius=0.6)
    cand = mask[keys[:, 0]]
    far = rr.outside(keys, [0.1, -0.2, 0.0], 0.6, VS)
    assert np.array_equal(keep, ~(cand & (empty | far)))
    # the new order holds every kept slot once, the unmoved ones in place
    n_keep = int(keep.sum())
    assert sorted(order.tolist()) == np.flatnonzero(keep).tolist()
    stay = np.flatnonzero(keep[:n_keep])
    assert np.array_equal(order[stay], stay)
    assert st[4] == int((~keep[:n_keep]).sum()) == int(keep[n_keep:].sum())
