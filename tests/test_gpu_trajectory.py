"""Trajectory optimisation against the ESDF on the GPU (tslam_esdf_trajectory / tslam_octo_esdf_trajectory) held to the
numpy reference (trajectory_reference.py) bit for bit, with the library's own esdf_query as the reference's field."""
import numpy as np
import pytest

import trajectory_reference as tref
from taichislam_b200 import synthetic as syn
from taichislam_b200.trajectory import control_points
from test_gpu_octo_travel import VS, handle as octo_handle, two_rooms, refused

pytestmark = pytest.mark.gpu

F32 = np.float32


def field_of(query):
    def f(x):
        d, g, v = query(np.ascontiguousarray(x, F32))
        return np.asarray(d, F32), np.asarray(g, F32), np.asarray(v, bool)
    return f


def assert_same(got, ref):
    assert got["ctrl"].tobytes() == ref["ctrl"].tobytes()
    c = np.array([got["J_s"], got["J_c"], got["J_f"], got["J_u"], got["J_in"], got["min_dist"]])
    assert c.tobytes() == ref["cost"].tobytes(), (c, ref["cost"])
    i = ref["info"]
    at = got["min_at"] if got["min_at"] is not None else (-1, -1)
    assert [got["iterations"], got["evaluations"], got["status"], got["invalid"], got["close"], at[0], at[1]] == list(i), (got, i)


def doorway():
    h = octo_handle(128, 128, min_ray_length=0.0)
    two_rooms(h)
    h.esdf_update(0, 1.0)
    h.travel_update(0, np.zeros(3, F32), 0.0, None)
    targets = np.array([[1.25, 0.5, 0.5], [1.25, 0.0, 0.0], [1.5, 0.25, -0.25], [1.4, -0.3, 0.2]], F32)
    cells, ln = h.travel_path(targets)
    assert ln[0] > 1                                        # the known path of test_two_rooms_doorway
    paths = [cells[t, :ln[t]].astype(np.float64) * VS for t in range(len(targets)) if ln[t] > 1]
    assert len(paths) >= 2
    return h, [control_points(p, 2 * VS) for p in paths]


def test_doorway_bit_exact_and_behaviour():
    """Bit-exact against the reference on the doorway paths.  The two-rooms world is built from sparse point rays, so
    unknown cells lie next to the travel path and some samples of the raw path are invalid: the solve must not add
    invalid samples, must lower J, and must keep the six end control points."""
    h, qs = doorway()
    kw = dict(max_iters=100, samples=4, check_samples=16)
    got = h.esdf_trajectory(qs, 0.1, **kw)
    raw = h.esdf_trajectory(qs, 0.1, max_iters=0, samples=4, check_samples=16)
    fld = field_of(h.esdf_query)
    for g, q in zip(got, qs):
        assert_same(g, tref.solve(q, fld, VS, clearance=0.1, **kw))
    for g, r, q in zip(got, raw, qs):
        print("doorway:", {k: v for k, v in g.items() if k != "ctrl"})
        assert g["J_u"] <= r["J_u"] and g["invalid"] <= r["invalid"]
        J = ((g["J_s"] + 100.0 * g["J_c"]) + g["J_f"]) + 1000.0 * g["J_u"]
        assert J <= g["J_in"]
        assert g["ctrl"][:3].tobytes() == q[:3].tobytes() and g["ctrl"][-3:].tobytes() == q[-3:].tobytes()


def test_check_mode_matches_esdf_query_and_batches():
    h, qs = doorway()
    got = h.esdf_trajectory(qs, 0.1, max_iters=0, check_samples=8)
    for g, q in zip(got, qs):
        assert g["ctrl"].tobytes() == q.tobytes() and g["iterations"] == 0
        x = tref.positions(q, tref.basis(8)).astype(F32)[tref.sample_mask(len(q) - 3, 8)]
        d, _, v = h.esdf_query(x)
        assert g["invalid"] == int((~v).sum()) and g["close"] == int((v & (d.astype(np.float64) < 0.1)).sum())
        assert g["min_dist"] == (float(d[v].min()) if v.any() else np.inf)
    # T = 1, 7 and 64 give the single calls' bits, and a repeat gives the same
    rng = np.random.default_rng(3)
    many = [qs[i % len(qs)] + np.concatenate([np.zeros((3, 3)), rng.normal(0, 0.02, (len(qs[i % len(qs)]) - 6, 3)), np.zeros((3, 3))])
            for i in range(64)]
    kw = dict(max_iters=30)
    single = [h.esdf_trajectory([q], 0.1, **kw)[0] for q in many[:7]]
    for T in (1, 7, 64):
        for rep in range(2):
            out = h.esdf_trajectory(many[:T], 0.1, **kw)
            for a, b in zip(out[:7], single):
                assert a["ctrl"].tobytes() == b["ctrl"].tobytes() and a["J_in"] == b["J_in"] and a["J_s"] == b["J_s"]
                assert (a["iterations"], a["evaluations"], a["status"]) == (b["iterations"], b["evaluations"], b["status"])


def test_no_side_effects_and_readability():
    h, qs = doorway()
    before = (h.esdf_gather(0), h.travel_gather(0) if hasattr(h, "travel_gather") else None, h.gather(0))
    n0 = h.launch_count() if hasattr(h, "launch_count") else None
    h.esdf_trajectory(qs, 0.1, max_iters=20)
    n1 = h.launch_count() if n0 is not None else None
    after = (h.esdf_gather(0), h.travel_gather(0) if hasattr(h, "travel_gather") else None, h.gather(0))
    for a, b in zip(before, after):                        # rows in a canonical order (gathers append in any order)
        if a is not None:
            oa, ob = np.lexsort(np.asarray(a[0]).T[::-1]), np.lexsort(np.asarray(b[0]).T[::-1])
            for x, y in zip(a, b):
                assert np.asarray(x)[oa].tobytes() == np.asarray(y)[ob].tobytes()
    if n0 is not None:
        assert n1 == n0 + 1
    refused(h.esdf_trajectory, qs, 0.1, submap=1)          # the last update was for submap 0
    refused(h.esdf_trajectory, qs, 1.5)                    # clearance above max_dist
    h.reset()
    refused(h.esdf_trajectory, qs, 0.1)                    # reset: no readable field


def room_tsdf():
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True, max_ray_length=4.0)
    g.integrate_depth(syn.scene_room(), np.eye(3)[None], np.zeros((1, 3)))
    g.esdf_update()
    return g


def test_tsdf_room_bit_exact_and_refusals():
    g = room_tsdf()
    rng = np.random.default_rng(7)
    qs = []
    for t in range(6):
        a, b = rng.uniform(-0.8, 0.8, 3), rng.uniform(-0.8, 0.8, 3)
        a[2], b[2] = rng.uniform(1.0, 2.5, 2)
        qs.append(control_points(np.stack([a, b]), 2 * VS))
    kw = dict(max_iters=60, samples=3, check_samples=10, memory=5)
    got = g.trajectory(qs, 0.15, **kw)
    fld = field_of(g.esdf_query)
    for r, q in zip(got, qs):
        assert_same(r, tref.solve(q, fld, VS, clearance=0.15, **kw))
    refused(g.trajectory, qs, 5.0)                         # clearance above max_ray_length
    refused(g.trajectory, qs, 0.1, submap=1)
    g.reset()
    refused(g.trajectory, qs, 0.1)


def test_sphere_scatter_field_bit_exact():
    """The analytic sphere TSDF loaded with scatter, and trajectories grazing it."""
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    m = DenseTSDF(map_scale=[6.4, 6.4], voxel_scale=VS, is_global_map=True, max_ray_length=1.0)
    r = np.arange(-24, 24)
    I, J, K = np.meshgrid(r, r, r, indexing="ij")
    idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
    p = idx.astype(np.float64) * VS
    t = (np.sqrt((p * p).sum(1)) - 0.5).astype(F32)
    m.load_numpy(0, idx, t, np.ones_like(t), np.zeros(len(t), np.int8), np.array([]))
    qs = [control_points(np.array([[-1.0, y, 0.0], [1.0, y, 0.05]]), 0.1) for y in (0.3, 0.55, -0.62)]
    out = m.optimize_trajectories(qs, clearance=0.2, ctrl=True, max_iters=80)
    fld = field_of(lambda x: m.esdf_query(x, update=False))
    for r_, q in zip(out, qs):
        assert_same(r_, tref.solve(q, fld, VS, clearance=0.2, max_iters=80))
    assert out[0]["J_c"] < tref.evaluate(qs[0], fld, dict(tref.DEFAULTS, clearance=0.2), tref.basis(4))[1][1]


def test_octomap_class_flow():
    from taichislam_b200.mapping.taichi_octomap import Octomap
    m = Octomap(map_scale=[6.4, 6.4], voxel_scale=VS, occupancy_model="logodds", max_ray_length=5.0, K=2)
    two_rooms(m._h)
    m.esdf_update(1.0)
    m.travel_update(np.zeros(3), 0.0)
    cells, ln = m._h.travel_path(np.array([[1.25, 0.5, 0.5]], F32))
    path = cells[0, :ln[0]].astype(np.float64) * VS
    out = m.optimize_trajectories([path], clearance=0.1, max_iters=50)
    assert len(out) == 1 and out[0]["ctrl"].shape[1] == 3 and out[0]["status"] in (0, 1, 2)
    with pytest.raises(ValueError):
        Octomap(map_scale=[6.4, 6.4], voxel_scale=VS, K=2).optimize_trajectories([path], clearance=0.1)
