"""Exploration tours on the GPU: every restart's tour, cost pair, passes and converged flag, the best restart and info2
bit for bit equal to the numpy statement of the contract (tour_reference.py), on matrices built here from fixed seeds;
refusals; and Octomap.exploration_tour on a log-odds map."""
import math

import numpy as np
import pytest

import tour_reference as tr
from taichislam_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

F32 = np.float32
VS = 0.05


def euclid(rng, n, asym=1.3, sym=False, inf_frac=0.0, zero_frac=0.0, unreachable=0):
    """random points in a 10 m cube, distances times noise in [1, asym); sym takes the smaller of each pair"""
    xy = rng.uniform(0, 10, (n, 3))
    C = np.linalg.norm(xy[:, None] - xy[None], axis=2) * rng.uniform(1.0, asym, (n, n))
    if sym:
        C = np.minimum(C, C.T)
    C[rng.random((n, n)) < inf_frac] = np.inf
    C[rng.random((n, n)) < zero_frac] = 0.0
    if unreachable:
        C[0, rng.choice(np.arange(1, n), unreachable, replace=False)] = np.inf
    np.fill_diagonal(C, 0)
    return C.astype(F32)


def gpu(C, **kw):
    from taichislam_b200.tour import solve_open_tour
    return solve_open_tour(C, **kw)


def check(C, restarts, seed=0, max_passes=None):
    g = gpu(C, restarts=restarts, seed=seed, max_passes=max_passes)
    w = tr.solve(C, restarts=restarts, seed=seed, max_passes=max_passes)
    assert [g["m"], g["unit_exp"]] == w["info2"].tolist()
    bad = np.nonzero((g["tours"] != w["tours"]).any(1))[0]
    assert bad.size == 0, f"restarts {bad[:8]} differ, first gpu {g['tours'][bad[0]][:12]} ref {w['tours'][bad[0]][:12]}"
    assert np.array_equal(g["cost2"], w["cost2"])
    assert np.array_equal(g["passes"], w["passes"]) and np.array_equal(g["converged"], w["converged"].astype(bool))
    assert g["best"] == w["best"]
    b, m = w["best"], g["m"]
    assert np.array_equal(g["order"], w["tours"][b, 1:m + 1]) and g["inf_legs"] == w["cost2"][b, 0]
    assert g["cost"] == math.ldexp(float(w["cost2"][b, 1]), g["unit_exp"])
    assert sorted(g["order"].tolist() + g["unreachable"].tolist()) == list(range(1, C.shape[0]))
    return g


def test_small_m():
    rng = np.random.default_rng(1)
    check(np.zeros((1, 1), F32), 4)                                   # m = 0, n = 1
    C = euclid(rng, 6)
    C[0, 1:] = np.inf
    g = check(C, 3)                                                   # m = 0: every goal unreachable
    assert g["order"].size == 0 and g["cost"] == 0.0 and g["unreachable"].tolist() == [1, 2, 3, 4, 5]
    check(euclid(rng, 2), 3)                                          # m = 1
    for n in (3, 4, 8):                                               # m = 2, 3, 7
        for kw in (dict(), dict(sym=True), dict(zero_frac=0.1), dict(inf_frac=0.2)):
            check(euclid(rng, n, **kw), 16, seed=n)


@pytest.mark.parametrize("kind", ["asym", "sym", "zeros", "inf", "unreachable", "truncated"])
def test_m31_and_m100(kind):
    rng = np.random.default_rng(len(kind))
    kw = dict(asym=dict(), sym=dict(sym=True), zeros=dict(zero_frac=0.05), inf=dict(inf_frac=0.1),
              unreachable=dict(unreachable=5), truncated=dict())[kind]
    mp = 3 if kind == "truncated" else None
    g = check(euclid(rng, 32, **kw), 24, seed=7, max_passes=mp)
    if kind == "truncated":
        assert not g["converged"][1:].any() and (g["passes"][1:] == 3).all()
    if kind == "unreachable":
        assert g["m"] == 26
    check(euclid(rng, 105, **kw), 6, seed=9, max_passes=mp)


@pytest.mark.parametrize("n", [230, 240, 256])
def test_shared_and_l2_staging(n):
    """C staged in shared memory at n = 230 (4n^2 = 207 KB), read through L2 at 240 and 256 (m = 255)"""
    rng = np.random.default_rng(n)
    check(euclid(rng, n, unreachable=(n == 240) * 3), 3, seed=n)


def test_m1023_few_restarts():
    rng = np.random.default_rng(3)
    g = check(euclid(rng, 1024), 2, seed=1, max_passes=10)
    assert g["m"] == 1023 and (g["passes"] == 10).all() and not g["converged"].any()


def test_torch_and_numpy_inputs_and_wide_range():
    import torch
    rng = np.random.default_rng(5)
    C = euclid(rng, 40)
    C[1:, 1:] *= np.ldexp(1.0, rng.integers(0, 22, (39, 39))).astype(F32)   # a 2^22 value range
    a = check(C, 8, seed=2)
    b = gpu(torch.from_numpy(C).cuda(), restarts=8, seed=2)
    for k in ("tours", "cost2", "passes", "converged"):
        assert np.array_equal(a[k], b[k]), k
    assert a["best"] == b["best"] and a["cost"] == b["cost"]
    # the largest and smallest seeds wrap as uint64
    check(C, 5, seed=(1 << 64) - 1)


def test_refusals():
    from taichislam_b200 import _capi as capi

    def refused(C, **kw):
        with pytest.raises(capi.TslamError) as e:
            gpu(C, **kw)
        assert e.value.code == capi.E_INVALID

    rng = np.random.default_rng(2)
    ok = euclid(rng, 6)
    for bad in (np.nan, -1.0, -np.inf, 1e-40):
        C = ok.copy()
        C[2, 3] = bad
        refused(C)
    C = ok.copy()
    C[1, 1], C[2, 2] = np.nan, -1.0                                   # the diagonal is ignored
    check(C, 2)
    C = np.ones((4, 4), F32)
    C[1, 2] = 2.0 ** 28                                               # range 28 accepted, 29 refused
    check(C, 2)
    C[1, 2] = 2.0 ** 29
    refused(C)
    refused(np.zeros((1025, 1025), F32))
    for R in (0, 4097):
        refused(ok, restarts=R)
    refused(ok, max_passes=-1)
    check(ok, 4096, max_passes=0)
    # a refusal writes nothing the next call could see
    check(ok, 3)


def octomap(scene):
    from taichislam_b200.mapping.taichi_octomap import Octomap
    o = Octomap(map_scale=[12.8, 12.8], voxel_scale=VS, occupancy_model="logodds", max_ray_length=3.0, max_disp_particles=1024)
    o.set_dep_camera_intrinsic(syn.K_DEPTH)
    o.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    d = syn.scene_room() if scene == "room" else syn.scene_plane(3.0)
    o.recast_depth_to_map(np.eye(3), np.zeros(3), d, None)
    o.recast_depth_to_map(np.eye(3), np.array([0.1, 0.0, 0.0]), d, None)
    return o


@pytest.mark.parametrize("scene", ["S1", "room"])
def test_octomap_exploration_tour(scene):
    import torch
    o = octomap(scene)
    idx, L = o._h.gather(0)
    free = idx[L <= o.l_occ]
    rng = np.random.default_rng(4)
    goals = free[rng.choice(len(free), 24, replace=False)].astype(F32) * F32(VS)
    goals = np.concatenate([goals, np.array([[6.0, 6.0, 6.0]], F32)])   # in unknown space
    start = np.zeros(3, F32)
    res = o.exploration_tour(start, goals, seed=3)
    pts = np.concatenate([start[None], goals]).astype(F32)
    M = o.travel_cost_multi(pts)                                      # the fields the tour left readable
    reach = np.nonzero(np.isfinite(M[0, 1:]))[0]
    assert len(goals) - 1 in res["unreachable"].tolist() and len(reach) >= 12
    assert sorted(res["order"].tolist()) == reach.tolist()
    assert sorted(res["order"].tolist() + res["unreachable"].tolist()) == list(range(len(goals)))
    tour = np.concatenate([[0], res["order"] + 1])
    legs = M[tour[:-1], tour[1:]]
    assert np.array_equal(res["leg_costs"].view(np.int32), legs.view(np.int32))
    assert res["inf_legs"] == int(np.isinf(legs).sum())
    assert res["cost"] == math.fsum(float(x) for x in legs[np.isfinite(legs)])
    # the same tour as the solver on the matrix itself
    w = tr.solve(M, restarts=64, seed=3)
    assert np.array_equal(res["order"] + 1, w["tours"][w["best"], 1:w["info2"][0] + 1])
    assert res["converged"] == bool(w["converged"][w["best"]])
    first = o.travel_path_multi(0, goals[res["order"][0]])
    assert first is not None and np.array_equal(res["path"], first)
    # torch inputs
    r2 = o.exploration_tour(torch.from_numpy(start).cuda(), torch.from_numpy(goals).cuda(), seed=3)
    assert np.array_equal(r2["order"], res["order"]) and r2["cost"] == res["cost"]


def test_octomap_exploration_tour_occ_start_clearance_and_refusals():
    from taichislam_b200.mapping.taichi_octomap import Octomap
    o = octomap("room")
    idx, L = o._h.gather(0)
    free = idx[L <= o.l_occ]
    rng = np.random.default_rng(6)
    goals = free[rng.choice(len(free), 10, replace=False)].astype(F32) * F32(VS)
    occ = idx[L > o.l_occ][0].astype(F32) * F32(VS)
    r = o.exploration_tour(occ, goals)
    assert r["order"].size == 0 and r["unreachable"].tolist() == list(range(10)) and r["path"] is None
    assert r["cost"] == 0.0 and r["inf_legs"] == 0
    assert getattr(o, "esdf_max_dist", None) is None
    r = o.exploration_tour(np.zeros(3, F32), goals, clearance=0.1)   # runs esdf_update(max_ray_length) first
    assert o.esdf_max_dist == 3.0
    pts = np.concatenate([np.zeros((1, 3), F32), goals])
    st = o.travel_update_multi(pts, clearance=0.1)
    M = o.travel_cost_multi(pts)
    assert sorted(r["order"].tolist()) == np.nonzero(np.isfinite(M[0, 1:]))[0].tolist()
    assert r["cost"] == math.fsum(float(x) for x in r["leg_costs"][np.isfinite(r["leg_costs"])]) and st["start_ok"][0]
    with pytest.raises(ValueError):
        o.exploration_tour(np.zeros(3), np.zeros((1024, 3), F32))
    hits = Octomap(map_scale=[3.2, 3.2], voxel_scale=VS, max_disp_particles=16)
    with pytest.raises(ValueError):
        hits.exploration_tour(np.zeros(3), np.zeros((2, 3), F32))
