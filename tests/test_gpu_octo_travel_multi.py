"""Many-source travel costs of the log-odds Octomap on the GPU: every row bit for bit (int32 views) equal to the
single-source field from the same start (travel_update + travel_query), some rows also against the numpy reference
(octo_travel_reference.py); the cost matrix; paths cell for cell against travel_path; staleness, state and refusals."""
import ctypes as C
import math

import numpy as np
import pytest

import octo_logodds_reference as ref
import octo_travel_reference as tr
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu

VS = 0.05
LO = ref.params()
F32 = np.float32
D = 1.0


def handle(N=256, Nz=256, **kw):
    from taichislam_b200.octo_handle import OctoHandle
    kw.setdefault("Kcam", syn.K_DEPTH)
    kw.setdefault("max_ray_length", 5.0)
    return OctoHandle(N, Nz, K=2, voxel_scale=VS, logodds=LO, **kw)


def refused(fn, *a, **kw):
    from taichislam_b200 import _capi as capi
    with pytest.raises(capi.TslamError) as e:
        fn(*a, **kw)
    assert e.value.code == capi.E_INVALID


def reference(h, start, clearance=0.0, max_cost=None, submap=0):
    idx, L = h.gather(submap)
    esdf = h.esdf_gather(submap) if clearance > 0 else None
    return tr.Field(idx, L, LO["l_occ"], VS, np.asarray(start, F32), clearance, max_cost, esdf)


def free_cells(h, submap=0):
    idx, L = h.gather(submap)
    return idx[L <= LO["l_occ"]]


def single_rows(h, starts, pts, clearance=0.0, max_cost=None, submap=0):
    """(rows f32[S,n], stats) of one travel_update + travel_query per start"""
    rows, stats = [], []
    for p in starts:
        stats.append(h.travel_update(submap, p, clearance, max_cost))
        rows.append(h.travel_query(pts, submap))
    return np.stack(rows), stats


def check_multi(h, starts, pts, clearance=0.0, max_cost=None, submap=0):
    """travel_multi_update + travel_multi_query against the single-source path, row by row -> (multi stats, rows)"""
    st = h.travel_multi_update(submap, starts, clearance, max_cost)
    M = h.travel_multi_query(pts, submap)
    want, ss = single_rows(h, starts, pts, clearance, max_cost, submap)
    assert M.shape == (len(starts), pts.shape[0])
    for s in range(len(starts)):
        bad = np.nonzero(M[s].view(np.int32) != want[s].view(np.int32))[0]
        assert bad.size == 0, f"row {s}: {bad.size} costs differ, first gpu {M[s, bad[:4]]} single {want[s, bad[:4]]}"
        assert st["reachable"][s] == ss[s]["reachable"] and st["start_ok"][s] == ss[s]["start_ok"], (s, st, ss[s])
        assert st["traversable"] == ss[s]["traversable"]
    assert st["sweeps"] >= 1
    return st, M


def scene_starts(h, Ts, rng, clearance_d=None):
    """the sensor cell, 26 random FREE cells, a duplicate, and one each of UNKNOWN, OCC, outside the volume and a FREE
    cell less than 0.2 m from an obstacle (when the ESDF is given)"""
    free = free_cells(h)
    idx, L = h.gather(0)
    st = [np.asarray(Ts, F32)] + [free[q].astype(F32) * F32(VS) for q in rng.choice(len(free), 26, replace=False)]
    st.append(st[3].copy())
    known = {tuple(x) for x in idx.tolist()}
    u = next(c for c in (np.array([x, 0, 0]) for x in range(120, -128, -1)) if tuple(c) not in known)
    st += [u.astype(F32) * F32(VS), idx[L > LO["l_occ"]][0].astype(F32) * F32(VS), np.array([100.0, 0.0, 0.0], F32)]
    if clearance_d is not None:
        e_i, e_E = clearance_d
        st.append(e_i[(e_E > 0) & (e_E < 0.1)][0].astype(F32) * F32(VS))
    return np.stack(st).astype(F32)


def query_points(h, rng):
    idx, _ = h.gather(0)
    j = idx[rng.integers(len(idx), size=4096)].astype(F32) * F32(VS) + rng.uniform(-0.45, 0.45, (4096, 3)).astype(F32) * F32(VS)
    bad = np.zeros((8, 3), F32)
    bad[:4, 0] = np.nan
    bad[4:, 1] = np.inf
    return np.concatenate([idx.astype(F32) * F32(VS), j, bad]).astype(F32)


SCENES = {"S1": lambda: syn.scene_plane(3.0), "S2": lambda: syn.scene_sphere(4.0), "S4": lambda: syn.scene_noise(4),
          "room": lambda: syn.scene_room()}


@pytest.mark.parametrize("scene", list(SCENES))
def test_rows_equal_single_source_fields(scene):
    h = handle()
    d = SCENES[scene]()
    Rs, Ts = syn.stream_poses(2, start=40)
    for q in range(2):
        h.integrate_depth(d, Rs[q], Ts[q])
    h.esdf_update(0, D)
    rng = np.random.default_rng(len(scene))
    starts = scene_starts(h, Ts[1], rng, h.esdf_gather(0))
    assert 30 <= len(starts) <= 40
    pts = query_points(h, rng)
    st0, M0 = check_multi(h, starts, pts)
    st2, M2 = check_multi(h, starts, pts, clearance=0.2)
    ok0, ok2 = st0["start_ok"], st2["start_ok"]
    assert ok0[:-4].all() and not ok0[-4:-1].any() and ok0[-1] and not ok2[-1] and st0["reachable"][0] > 1000
    assert np.array_equal(M0[3].view(np.int32), M0[27].view(np.int32))      # the duplicate start
    assert st2["traversable"] < st0["traversable"]
    # three rows against the numpy reference
    for s, cl, M in ((0, 0.0, M0), (5, 0.0, M0), (9, 0.2, M2)):
        f = reference(h, starts[s], cl)
        assert np.array_equal(M[s].view(np.int32), f.query(pts, h.N, h.Nz).view(np.int32)), (s, cl)
        assert (st0 if cl == 0 else st2)["reachable"][s] == f.reachable()[0].shape[0]


def test_one_start_and_1024_starts():
    h = handle(128, 128)
    d = syn.scene_room()
    h.integrate_depth(d, np.eye(3), np.zeros(3))
    h.integrate_depth(d, rot_xyz(0.0, 0.5, 0.1), np.array([0.1, 0.0, 0.05]))
    rng = np.random.default_rng(4)
    free = free_cells(h)
    pts = query_points(h, rng)[-6000:]
    check_multi(h, np.zeros((1, 3), F32), pts)
    starts = free[rng.integers(len(free), size=1024)].astype(F32) * F32(VS)
    st, M = check_multi(h, starts, pts)
    assert st["start_ok"].all() and M.shape == (1024, pts.shape[0])
    for S in (0, 1025):
        refused(h.travel_multi_update, 0, np.zeros((S, 3), F32))
    # the refused calls left the last fields readable
    assert np.array_equal(h.travel_multi_query(pts).view(np.int32), M.view(np.int32))


def two_rooms(h):
    """test_gpu_octo_travel.two_rooms: room A around the origin, room B behind a wall at x = 1 m (cells i = 20, |j|, |k|
    <= 20), joined by a 5 x 5 cell doorway at |j|, |k| <= 2"""
    g = np.arange(-20, 21)
    J, K = np.meshgrid(g, g, indexing="ij")
    J, K = J.ravel(), K.ravel()
    door_m = (np.abs(J) <= 2) & (np.abs(K) <= 2)
    wall = np.stack([np.full(J.size, 20), J, K], 1)[~door_m].astype(F32) * F32(VS)
    back = np.stack([np.full(J.size, 40), J, K], 1).astype(F32) * F32(VS)
    through = back[(np.abs(J) <= 4) & (np.abs(K) <= 4)]
    h.integrate_points(np.concatenate([wall, through]).astype(F32), np.eye(3), np.zeros(3))
    TB = np.array([1.5, 0.0, 0.0])
    h.integrate_points((np.concatenate([wall, back]) - TB.astype(F32)).astype(F32), np.eye(3), TB)


def close_door(h):
    g = np.arange(-2, 3)
    J, K = np.meshgrid(g, g, indexing="ij")
    dcell = np.stack([np.full(J.size, 20), J.ravel(), K.ravel()], 1).astype(F32) * F32(VS)
    for _ in range(4):
        h.integrate_points(dcell, np.eye(3), np.zeros(3))


def matrix_bound(M):
    """|M - M.T| allowed where both are finite: twice the f32 rounding bound of test_octo_travel_multi_reference_cpu"""
    hi = np.maximum(M, M.T).astype(np.float64) * (1 + 2.0 ** -18)
    return 2 * hi * (hi / VS + 4) * 2.0 ** -22


def chamfer(a, b):
    s = np.sort(np.abs(np.asarray(a) - np.asarray(b)))[::-1]
    return s[2] * math.sqrt(3) * VS + (s[1] - s[2]) * math.sqrt(2) * VS + (s[0] - s[1]) * VS


def test_cost_matrix_two_rooms_and_closed_door():
    h = handle(128, 128, min_ray_length=0.0)
    two_rooms(h)
    A = [(0, 0, 0), (5, 3, -2), (10, -6, 4), (15, 9, -12)]     # cell centres on A's rays to the wall
    B = [(25, 10, 10), (35, -5, 5), (35, 5, -5)]                 # ... and on B's rays from (30, 0, 0)
    cells = np.array(A + B)
    starts = cells.astype(F32) * F32(VS)
    st = h.travel_multi_update(0, starts)
    assert st["start_ok"].all()
    M = h.travel_multi_query(starts)
    check_multi(h, starts, starts)
    fin = np.isfinite(M)
    assert fin.all() and (np.diag(M) == 0).all()
    assert np.array_equal(fin, fin.T) and (np.abs(M - M.T)[fin] <= matrix_bound(M)[fin]).all()
    # cross-room costs are at least the chamfer distance through the doorway, and exceed the plain chamfer distance
    # wherever no chamfer-shortest path fits through the doorway
    door = [(20, j, k) for j in range(-2, 3) for k in range(-2, 3)]
    blocked = 0
    for a in range(len(A)):
        for b in range(len(A), len(cells)):
            via = min(chamfer(cells[a], d) + chamfer(d, cells[b]) for d in door)
            assert min(M[a, b], M[b, a]) >= via - via * (via / VS + 4) * 2.0 ** -22
            if via > chamfer(cells[a], cells[b]) + 1e-6:
                blocked += 1
                assert M[a, b] > chamfer(cells[a], cells[b]) and M[b, a] > chamfer(cells[a], cells[b])
    assert blocked >= 6
    close_door(h)
    st2 = h.travel_multi_update(0, starts)
    M2 = h.travel_multi_query(starts)
    same = np.zeros(M2.shape, bool)
    same[:len(A), :len(A)] = same[len(A):, len(A):] = True
    assert np.isfinite(M2[same]).all() and np.isinf(M2[~same]).all() and (np.diag(M2) == 0).all()
    assert (st2["reachable"] < st["reachable"]).all()


def seam_map(h):
    """test_gpu_octo_travel.test_block_seams_and_a_start_on_a_block_corner: a shell of OCC points on the seams i & 7 == 7"""
    rng = np.random.default_rng(3)
    T = np.array([-0.05, -0.05, -0.05])
    for q in range(3):
        d = rng.normal(size=(400, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        pts = (d * rng.uniform(0.4, 1.4, (400, 1))).astype(F32)
        h.integrate_points(pts, np.eye(3), T)
    g = np.argwhere(np.ones((4, 4, 4), bool)) * 8 - 9
    g = g[~(g == -1).all(1)]
    h.integrate_points((g.astype(F32) * F32(VS) - T.astype(F32)).astype(F32), np.eye(3), T)
    return T.astype(F32)


def test_paths_match_single_source_paths():
    from taichislam_b200 import _capi as capi
    h = handle(64, 64, min_ray_length=0.0)
    T = seam_map(h)
    rng = np.random.default_rng(8)
    f = reference(h, T)
    ri, _ = f.reachable()
    seam = ri[((ri & 7) == 7).any(1) | ((ri & 7) == 0).any(1)]
    starts = np.concatenate([T[None], seam[rng.choice(len(seam), 7, replace=False)].astype(F32) * F32(VS)]).astype(F32)
    st = h.travel_multi_update(0, starts)
    assert st["start_ok"].all()
    src = rng.integers(len(starts), size=256).astype(np.int32)
    tg = seam[rng.integers(len(seam), size=256)].astype(F32) * F32(VS)
    cells, ln = h.travel_multi_path(src, tg)
    short, sl = h.travel_multi_path(src, tg, max_len=6)
    assert np.array_equal(sl, ln) and (ln > 6).any() and (ln > 0).mean() > 0.9
    crossings = 0
    for s in range(len(starts)):
        q = np.nonzero(src == s)[0]
        h.travel_update(0, starts[s])
        c1, l1 = h.travel_path(tg[q])
        assert np.array_equal(l1, ln[q]), s
        for a, b in enumerate(q):
            assert np.array_equal(cells[b, :ln[b]], c1[a, :l1[a]]), (s, b)
            assert np.array_equal(short[b, :min(6, ln[b])], c1[a, :min(6, l1[a])])
            crossings += int((np.diff(cells[b, :ln[b]] >> 3, axis=0) != 0).any(1).sum())
    assert crossings > 100
    # the reference agrees on the paths of the first start
    for b in np.nonzero(src == 0)[0][:16]:
        assert np.array_equal(cells[b, :ln[b]], f.path(tg[b]))
    # torch in -> torch out
    import torch
    tc, tl = h.travel_multi_path(torch.from_numpy(src).cuda(), torch.from_numpy(tg).cuda())
    assert isinstance(tl, torch.Tensor) and np.array_equal(tl.cpu().numpy(), ln)
    # a source outside [0, S): len 0, and the next sync reports it
    _, good = h.travel_multi_path(np.array([0, 2], np.int32), tg[[0, 3]])
    _, lb = h.travel_multi_path(np.array([0, len(starts), -1, 2], np.int32), tg[:4])
    assert lb[1] == 0 and lb[2] == 0 and lb[0] == good[0] > 0 and lb[3] == good[1] > 0
    with pytest.raises(capi.TslamError) as e:
        h.sync()
    assert e.value.code == capi.E_INVALID
    h.sync()                                                     # reported once


def test_staleness_submaps_reset_fusion_and_recycled_slots():
    h = handle(128, 128, max_submaps=2)
    d = syn.scene_room()
    h.integrate_depth(d, np.eye(3), np.zeros(3))
    rng = np.random.default_rng(5)
    free = free_cells(h)
    starts = np.concatenate([np.zeros((1, 3), F32), free[rng.choice(len(free), 7, replace=False)].astype(F32) * F32(VS)])
    idx, _ = h.gather(0)
    pts = query_points(h, rng)
    st, M = check_multi(h, starts, pts)
    src = rng.integers(8, size=64).astype(np.int32)
    tg = free[rng.choice(len(free), 64, replace=False)].astype(F32) * F32(VS)
    cells, ln = h.travel_multi_path(src, tg)
    # more integration changes nothing the readers return; blocks allocated since read +inf
    before = {tuple(x) for x in (idx >> 3).tolist()}
    h.integrate_depth(d, rot_xyz(0.0, 2.5, 0.0), np.array([0.0, 0.2, 0.0]))
    assert np.array_equal(h.travel_multi_query(pts).view(np.int32), M.view(np.int32))
    c2, l2 = h.travel_multi_path(src, tg)
    assert np.array_equal(l2, ln) and all(np.array_equal(c2[q, :ln[q]], cells[q, :ln[q]]) for q in range(64))
    i2, _ = h.gather(0)
    new = np.array([x for x in i2.tolist() if tuple(np.array(x) >> 3) not in before])
    assert len(new) > 0
    assert np.isinf(h.travel_multi_query(new[:4096].astype(F32) * F32(VS))).all()
    # two submaps
    h.integrate_depth(syn.scene_sphere(3.0), np.eye(3), np.zeros(3), submap=1)
    p1 = (free_cells(h, 1)[:64].astype(F32) * F32(VS)).astype(F32)
    check_multi(h, np.concatenate([np.zeros((1, 3), F32), p1[:5]]), p1, submap=1)
    refused(h.travel_multi_query, pts, 0)
    refused(h.travel_multi_path, src, tg, 0)
    check_multi(h, starts, pts)
    # reset: readers refuse until the next update; recycled pool slots leak nothing
    h.reset()
    refused(h.travel_multi_query, pts, 0)
    refused(h.travel_multi_path, src, tg, 0)
    h.integrate_points(np.array([[1.0, 0.2, 0.3], [0.1, 1.2, 0.0]], F32), np.eye(3), np.zeros(3))
    st, M = check_multi(h, starts[:3], pts)
    assert st["start_ok"][0] and 0 < st["reachable"][0] < 200
    h.integrate_depth(d, rot_xyz(0.0, 0.2, 0.0), np.zeros(3))
    check_multi(h, starts, query_points(h, rng))
    # fusion
    src_map = handle(128, 128)
    src_map.integrate_depth(d, np.eye(3), np.zeros(3))
    h.set_submap_pose(0, np.eye(3), np.zeros(3))
    h.fuse_from(src_map)
    refused(h.travel_multi_query, pts, 0)
    refused(h.travel_multi_path, src, tg, 0)
    check_multi(h, starts, query_points(h, rng))


def test_independent_of_the_single_source_field_and_no_side_effects():
    a, b = handle(128, 128), handle(128, 128)
    d = syn.scene_room()
    for h in (a, b):
        h.integrate_depth(d, np.eye(3), np.zeros(3))
        h.esdf_update(0, D)
        h.frontier_update(0)
    rng = np.random.default_rng(6)
    free = free_cells(a)
    starts = free[rng.choice(len(free), 12, replace=False)].astype(F32) * F32(VS)
    pts = query_points(a, rng)
    src = rng.integers(12, size=32).astype(np.int32)
    tg = free[rng.choice(len(free), 32, replace=False)].astype(F32) * F32(VS)
    # a single-source update between a multi update and its readers changes no multi answer ...
    a.travel_multi_update(0, starts, clearance=0.1)
    M = a.travel_multi_query(pts)
    cells, ln = a.travel_multi_path(src, tg)
    a.travel_update(0, np.zeros(3), clearance=0.0)
    g = a.travel_query(pts)
    gi = as_dict_rows(*a.travel_gather(0))
    assert np.array_equal(a.travel_multi_query(pts).view(np.int32), M.view(np.int32))
    c2, l2 = a.travel_multi_path(src, tg)
    assert np.array_equal(l2, ln) and all(np.array_equal(c2[q, :ln[q]], cells[q, :ln[q]]) for q in range(32))
    # ... and the reverse
    a.travel_multi_update(0, starts[:3])
    assert np.array_equal(a.travel_query(pts).view(np.int32), g.view(np.int32))
    g2 = as_dict_rows(*a.travel_gather(0))
    assert np.array_equal(g2[0], gi[0]) and np.array_equal(g2[1].view(np.int32), gi[1].view(np.int32))
    # against a twin map that never ran them: stats, gathers, and the next incremental ESDF and frontier updates
    for h in (a, b):
        h.integrate_depth(d, rot_xyz(0.0, 0.4, 0.6), np.array([0.2, -0.1, 0.0]))
    assert a.stats() == b.stats()
    ai, aL = as_dict_rows(*a.gather(0))
    bi, bL = as_dict_rows(*b.gather(0))
    assert np.array_equal(ai, bi) and np.array_equal(aL, bL)
    assert a.esdf_update(0, D) == b.esdf_update(0, D)
    ae, be = as_dict_rows(*a.esdf_gather(0)), as_dict_rows(*b.esdf_gather(0))
    assert np.array_equal(ae[0], be[0]) and np.array_equal(ae[1].view(np.int32), be[1].view(np.int32))
    sa, sb = a.frontier_update(0), b.frontier_update(0)
    assert sa == sb and not sa["full"]
    af, bf = as_dict_rows(*a.frontier_gather(0)), as_dict_rows(*b.frontier_gather(0))
    assert np.array_equal(af[0], bf[0]) and np.array_equal(af[1], bf[1])


def test_refusals():
    import torch
    from taichislam_b200 import _capi as capi
    from taichislam_b200.octo_handle import OctoHandle
    L = capi.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    x = torch.zeros((4, 3), dtype=torch.float32, device=dev)
    fo = torch.zeros((64, 4), dtype=torch.float32, device=dev)
    si = torch.zeros(4, dtype=torch.int32, device=dev)
    ci = torch.zeros((4, 8, 3), dtype=torch.int32, device=dev)
    li = torch.zeros(4, dtype=torch.int32, device=dev)
    X, FO, SI, CI, LI = (capi.tptr(t) for t in (x, fo, si, ci, li))
    two = np.zeros((2, 3), F32)

    def upd(h, starts=two, n=None, cl=0.0, mc=1.0, sub=0):
        p = capi.np_ptr(np.ascontiguousarray(starts, F32)) if starts is not None else None
        return L.tslam_octo_travel_multi_update(h.h, sub, len(starts) if n is None else n, p, cl, mc, None, None, None, None)

    def qry(h, sub=0, n=4, xyz=X, out=FO):
        return L.tslam_octo_travel_multi_query(h.h, sub, n, xyz, out, None)

    def pth(h, sub=0, n=4, source=SI, xyz=X, max_len=8, cells=CI, ln=LI):
        return L.tslam_octo_travel_multi_path(h.h, sub, n, source, xyz, max_len, cells, ln, None)

    hits = OctoHandle(64, 64, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH)
    assert upd(hits) == capi.E_INVALID and qry(hits) == capi.E_INVALID and pth(hits) == capi.E_INVALID
    h = handle(64, 64, max_submaps=2)
    h.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    assert qry(h) == capi.E_INVALID and pth(h) == capi.E_INVALID        # before any update
    h.travel_update(0, np.zeros(3))
    assert qry(h) == capi.E_INVALID and pth(h) == capi.E_INVALID        # a single-source update is not a multi update
    assert upd(h, starts=None, n=2) == capi.E_INVALID
    big = np.zeros((1025, 3), F32)
    for n in (0, -1, 1025):
        assert upd(h, starts=big, n=n) == capi.E_INVALID, n
    for s in ((np.nan, 0, 0), (0, np.inf, 0), (0, 0, -np.inf)):
        assert upd(h, starts=np.array([[0, 0, 0], s], F32)) == capi.E_INVALID, s
    limit = h.travel_limit()
    for cl, mc in ((-0.1, 1.0), (np.nan, 1.0), (np.inf, 1.0), (0.0, 0.0), (0.0, -1.0), (0.0, np.nan), (0.0, np.inf),
                   (0.0, float(np.nextafter(F32(limit), F32(np.inf))))):
        assert upd(h, cl=cl, mc=mc) == capi.E_INVALID, (cl, mc)
    assert upd(h, mc=limit) == capi.TSLAM_OK and upd(h, starts=big, n=1024) == capi.TSLAM_OK
    assert upd(h, cl=0.1) == capi.E_INVALID                     # clearance without an ESDF
    h.esdf_update(0, 0.5)
    assert upd(h, cl=0.5) == capi.TSLAM_OK and upd(h, cl=float(np.nextafter(F32(0.5), F32(1)))) == capi.E_INVALID
    assert upd(h, cl=0.1, sub=1) == capi.E_INVALID              # the ESDF is of submap 0
    assert upd(h, sub=2) == capi.E_INVALID and upd(h, sub=-1) == capi.E_INVALID
    assert upd(h) == capi.TSLAM_OK
    for sub in (1, 2, -1):
        assert qry(h, sub) == capi.E_INVALID and pth(h, sub) == capi.E_INVALID
    assert qry(h, n=-1) == capi.E_INVALID and qry(h, xyz=None) == capi.E_INVALID and qry(h, out=None) == capi.E_INVALID
    assert pth(h, n=-1) == capi.E_INVALID and pth(h, xyz=None) == capi.E_INVALID and pth(h, source=None) == capi.E_INVALID
    assert pth(h, cells=None) == capi.E_INVALID and pth(h, ln=None) == capi.E_INVALID
    assert pth(h, max_len=0) == capi.E_INVALID and pth(h, max_len=-3) == capi.E_INVALID
    assert qry(h, n=0, xyz=None, out=None) == capi.TSLAM_OK and pth(h, n=0, source=None, xyz=None, cells=None, ln=None) == capi.TSLAM_OK
    assert qry(h) == capi.TSLAM_OK and pth(h) == capi.TSLAM_OK
    h.sync()


def test_octomap_class_flow():
    import torch
    from taichislam_b200.mapping.taichi_octomap import Octomap
    o = Octomap(map_scale=[12.8, 12.8], voxel_scale=VS, occupancy_model="logodds", max_ray_length=3.0, max_disp_particles=1024)
    o.set_dep_camera_intrinsic(syn.K_DEPTH)
    o.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    d = syn.scene_room()
    o.recast_depth_to_map(np.eye(3), np.zeros(3), d, None)
    o.recast_depth_to_map(rot_xyz(0.0, 0.0, 0.4), np.array([0.1, 0.0, 0.0]), d, None)
    rng = np.random.default_rng(2)
    free = free_cells(o._h)
    starts = np.concatenate([np.zeros((1, 3), F32), free[rng.choice(len(free), 5, replace=False)].astype(F32) * F32(VS)])
    st = o.travel_update_multi(starts, clearance=0.1)           # runs esdf_update(max_ray_length) first
    assert st["start_ok"][0] and o.esdf_max_dist == 3.0
    M = o.travel_cost_multi(starts)
    assert isinstance(M, np.ndarray) and M.shape == (6, 6)
    ok = st["start_ok"]
    assert (np.diag(M)[ok] == 0).all() and np.isinf(np.diag(M)[~ok]).all()
    f = reference(o._h, starts[0], 0.1)
    pts = f.reachable()[0][rng.choice(f.reachable()[0].shape[0], 100, replace=False)].astype(F32) * F32(VS)
    c = o.travel_cost_multi(pts)
    assert np.array_equal(c[0].view(np.int32), f.query(pts, o.N, o.Nz).view(np.int32))
    ct = o.travel_cost_multi(torch.from_numpy(pts).cuda())
    assert isinstance(ct, torch.Tensor) and ct.is_cuda and np.array_equal(ct.cpu().numpy(), c)
    far = pts[np.argmax(c[0])]
    path = o.travel_path_multi(0, far, max_len=4)                # retried with the reported length
    want = f.path(far)[::-1]
    assert path.shape == (want.shape[0], 3) and want.shape[0] > 4
    assert np.array_equal(path, want.astype(np.float64) * float(F32(VS)))
    assert o.travel_path_multi(0, np.array([6.0, 6.0, 6.0])) is None
    for s in (-1, 6):
        with pytest.raises(ValueError):
            o.travel_path_multi(s, far)
    with pytest.raises(ValueError):
        o.travel_update_multi(starts, clearance=3.5)
    hits = Octomap(map_scale=[3.2, 3.2], voxel_scale=VS, max_disp_particles=16)
    for call in (lambda: hits.travel_update_multi(np.zeros((2, 3))), lambda: hits.travel_cost_multi(np.zeros((1, 3))),
                 lambda: hits.travel_path_multi(0, np.zeros(3))):
        with pytest.raises(ValueError):
            call()
