"""The ESDF query reference (tests/esdf_query_reference.py) pinned on its own, before any GPU run is held to it:
linear fields are reproduced, the gradient is the derivative of the interpolated distance, each validity rule holds
by itself, and on an oracle-built map the distance is positive in free space."""
import numpy as np
import pytest

import esdf_query_reference as eqr

F = np.float32
VS = 0.05


def grid_rows(lo, hi, fn):
    r = [np.arange(a, b) for a, b in zip(lo, hi)]
    I, J, K = np.meshgrid(*r, indexing="ij")
    idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
    return idx, fn(idx)


def linear_state(a, b, lo=(-20, -20, -12), hi=(20, 20, 12), N=64, Nz=32):
    a32 = np.asarray(a, F)
    idx, e = grid_rows(lo, hi, lambda idx: ((idx.astype(F) * F(VS)) @ a32 + F(b)).astype(F))
    return eqr.EsdfState(idx, np.ones(len(e), F), e, N, Nz, VS), idx, e


def points_in(lo, hi, n, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(np.asarray(lo) * VS, (np.asarray(hi) - 1) * VS, size=(n, 3)).astype(F)


def test_linear_field_is_reproduced_with_its_gradient():
    a, b = [0.3, -0.7, 0.5], 1.25
    st, _, _ = linear_state(a, b)
    p = points_in((-20, -20, -12), (20, 20, 12), 20000, 1)
    d, g, v = eqr.query(st, p)
    assert v.all()
    exact = p.astype(np.float64) @ np.asarray(a, np.float64) + b
    assert np.abs(d - exact).max() <= 2e-6 * (1 + np.abs(exact).max())
    assert np.abs(g - np.asarray(a, F)).max() <= 1e-4
    # exact voxel centres (f = 0): the stored value itself
    c = (np.array([[3, -4, 2], [-20, -20, -12], [18, 18, 10]], F) * F(VS)).astype(F)
    dc, _, vc = eqr.query(st, c)
    ref_c = (np.array([[3, -4, 2], [-20, -20, -12], [18, 18, 10]], F) * F(VS)) @ np.asarray(a, F) + F(b)
    assert vc.all() and np.abs(dc - ref_c).max() <= 1e-6


def test_gradient_matches_central_differences():
    rng = np.random.default_rng(2)
    idx, e = grid_rows((-10, -10, -10), (10, 10, 10), lambda idx: rng.random(len(idx)).astype(F))
    st = eqr.EsdfState(idx, np.ones(len(e), F), e, 64, 64, VS)
    # points whose fractional parts keep +-h inside the same cell
    i0 = rng.integers(-10, 9, size=(5000, 3))
    f = rng.uniform(0.1, 0.9, size=(5000, 3))
    p = ((i0 + f) * VS).astype(F)
    d, g, v = eqr.query(st, p)
    assert v.all()
    h = 1e-3
    for ax in range(3):
        dp = p.astype(np.float64).copy(); dp[:, ax] += h
        dm = p.astype(np.float64).copy(); dm[:, ax] -= h
        fd = (eqr.query(st, dp.astype(F))[0].astype(np.float64) - eqr.query(st, dm.astype(F))[0]) / (2 * h)
        assert np.abs(fd - g[:, ax]).max() <= 2e-3 * (1 + np.abs(g[:, ax]).max()), ax
    assert np.abs(g).max() > 5  # a field that actually varies


def test_each_validity_rule_alone():
    a, b = [0.3, -0.7, 0.5], 1.25
    st, idx, e = linear_state(a, b)
    base = np.array([[2.5, 3.5, 1.5]], F) * F(VS)        # cube (2..3, 3..4, 1..2), all known
    assert eqr.query(st, base)[2].all()
    # one unknown corner
    drop = np.all(idx == [3, 4, 2], axis=1)
    st1 = eqr.EsdfState(idx[~drop], np.ones(int((~drop).sum()), F), e[~drop], 64, 32, VS)
    d, g, v = eqr.query(st1, np.concatenate([base, np.array([[0.5, 0.5, 0.5]], F) * F(VS)]))
    assert not v[0] and v[1] and np.isnan(d[0]) and np.isnan(g[0]).all()
    # an INERT corner (observed, NaN TSDF)
    t = np.ones(len(e), F)
    t[np.nonzero(np.all(idx == [2, 3, 1], axis=1))[0]] = np.nan
    st2 = eqr.EsdfState(idx, t, e, 64, 32, VS)
    assert not eqr.query(st2, base)[2][0]
    # out of the volume: N = 64 -> indices [-32, 32); z: Nz = 32 -> [-16, 16).  A full grid of the volume:
    full, fe = grid_rows((-32, -32, -16), (32, 32, 16), lambda idx: np.zeros(len(idx), F))
    st3 = eqr.EsdfState(full, np.ones(len(fe), F), fe, 64, 32, VS)
    u = np.array([[30.999, 0, 0], [31.0, 0, 0], [-32.0, 0, 0], [-32.001, 0, 0], [0, 0, 14.9], [0, 0, 15.0],
                  [0, 0, -16.0], [0, 0, -16.01]], F)
    assert eqr.query(st3, u * F(VS))[2].tolist() == [True, False, True, False, True, False, True, False]
    # non-finite and huge coordinates
    bad = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1e30, 0, 0], [0, -1e30, 0]], F)
    d, g, v = eqr.query(st3, bad)
    assert not v.any() and np.isnan(d).all() and np.isnan(g).all()


def test_negative_coordinates_floor_not_trunc():
    a, b = [0.3, -0.7, 0.5], 1.25
    st, idx, e = linear_state(a, b)
    p = np.array([[-0.3, -0.6, -0.2]], F) * F(VS)         # floor -> cube (-1..0)^3; trunc would give (0..1)^3
    d, g, v = eqr.query(st, p)
    assert v[0] and abs(float(d[0]) - float(p[0].astype(np.float64) @ np.asarray(a) + b)) <= 1e-6
    drop = np.all(idx == [-1, -1, -1], axis=1)            # only the floor cube contains (-1, -1, -1)
    st1 = eqr.EsdfState(idx[~drop], np.ones(int((~drop).sum()), F), e[~drop], 64, 32, VS)
    assert not eqr.query(st1, p)[2][0]


def test_slice_selection_literal_index():
    idx, e = grid_rows((-4, -4, -16), (4, 4, 16), lambda idx: idx[:, 2].astype(F))
    st = eqr.EsdfState(idx, np.ones(len(e), F), e, 64, 32, VS)
    for z, k in ((0.0, 0), (0.1, 2), (-0.3, -6), (0.74, 15)):
        xyz, val = eqr.slice_rows(st, z)
        assert xyz.shape[0] == 64 and np.all(val == k), (z, k, np.unique(val))
        assert np.all(xyz[:, 2] == F(k) * F(VS))


def test_oracle_room_free_space_distance_is_positive(oracle_lib):
    from oracle.oracle import OracleTSDF
    from taichislam_b200 import synthetic as syn
    o = OracleTSDF(map_scale=[12.8, 12.8], K=syn.K_DEPTH, is_global_map=True, max_ray_length=4.0)
    o.integrate_depth(np.eye(3), np.zeros(3), syn.scene_room())
    o.esdf_update()
    gi, gt, _, _ = o.gather()
    ei, ee = o.esdf_gather()
    from util import as_dict_rows
    gi, gt = as_dict_rows(gi, gt)
    ei, ee = as_dict_rows(ei, ee)
    assert np.array_equal(gi, ei)
    st = eqr.EsdfState(gi, gt, ee, o.N, o.Nz, VS)
    tst = eqr.EsdfState(gi, gt, gt, o.N, o.Nz, VS)             # the same corners carrying their TSDF
    rng = np.random.default_rng(4)
    p = rng.uniform([-3, -2, -0.5], [3, 2, 5.5], size=(200000, 3)).astype(F)
    d, g, v = eqr.query(st, p)
    assert 0.05 < v.mean() < 0.95
    # free space: all eight corners on the positive side.  The interpolated TSDF is then > 0 only where they all are;
    # test the corners directly
    u = p / F(VS)
    i0 = np.floor(u).astype(np.int64)
    pos = np.ones(len(p), bool)
    for c in range(8):
        t, k = tst.corner(i0[:, 0] + (c >> 2), i0[:, 1] + ((c >> 1) & 1), i0[:, 2] + (c & 1))
        pos &= k & (t > 0)
    free = v & pos
    assert free.sum() > 10000
    assert np.all(d[free] > 0)
