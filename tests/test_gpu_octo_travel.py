"""Travel-cost field of the log-odds Octomap on the GPU against the numpy reference (octo_travel_reference.py): the
reachable cells and their costs bit for bit as int32 views, queries, and paths cell for cell."""
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


def reference(h, start, clearance=0.0, max_cost=None, submap=0, esdf=None):
    idx, L = h.gather(submap)
    if clearance > 0 and esdf is None:
        esdf = h.esdf_gather(submap)
    return tr.Field(idx, L, LO["l_occ"], VS, np.asarray(start, F32), clearance, max_cost, esdf)


def check_field(h, start, clearance=0.0, max_cost=None, submap=0, esdf=None):
    """travel_update, then the gathered field against the reference; -> (stats, reference field)"""
    st = h.travel_update(submap, start, clearance, max_cost)
    f = reference(h, start, clearance, max_cost, submap, esdf)
    gi, gG = as_dict_rows(*h.travel_gather(submap))
    ri, rG = as_dict_rows(*f.reachable())
    assert gi.shape == ri.shape, f"reachable cells: gpu {gi.shape[0]} reference {ri.shape[0]}"
    assert np.array_equal(gi, ri)
    bad = np.nonzero(gG.view(np.int32) != rG.view(np.int32))[0]
    assert bad.size == 0, f"{bad.size} costs differ, first {gi[bad[:4]].tolist()} gpu {gG[bad[:4]]} ref {rG[bad[:4]]}"
    assert st["reachable"] == ri.shape[0] and st["traversable"] == f.tidx.shape[0] and st["start_ok"] == f.start_ok, st
    assert st["sweeps"] >= 1
    return st, f


def check_paths(h, f, targets, max_len=4096, submap=0):
    cells, ln = h.travel_path(np.asarray(targets, F32), submap=submap, max_len=max_len)
    for q, t in enumerate(np.asarray(targets, F32)):
        p = f.path(t)
        assert ln[q] == p.shape[0], (q, ln[q], p.shape[0])
        k = min(p.shape[0], max_len)
        assert np.array_equal(cells[q, :k], p[:k]), q
    return cells, ln


def free_cells(h, submap=0):
    idx, L = h.gather(submap)
    return idx[L <= LO["l_occ"]]


SCENES = {"S1": lambda: syn.scene_plane(3.0), "S2": lambda: syn.scene_sphere(4.0), "S4": lambda: syn.scene_noise(4),
          "room": lambda: syn.scene_room()}


@pytest.mark.parametrize("scene", list(SCENES))
def test_fields_match_reference(scene):
    h = handle()
    d = SCENES[scene]()
    Rs, Ts = syn.stream_poses(2, start=40)
    for q in range(2):
        h.integrate_depth(d, Rs[q], Ts[q])
    h.esdf_update(0, D)
    rng = np.random.default_rng(len(scene))
    free = free_cells(h)
    starts = [np.asarray(Ts[1], F32)] + [(free[rng.integers(len(free))].astype(F32) * F32(VS)) for _ in range(2)]
    for q, s in enumerate(starts):
        st, f = check_field(h, s)
        assert st["start_ok"] and (q > 0 or st["reachable"] > 1000), st
        st2, f2 = check_field(h, s, clearance=0.2)
        assert st2["traversable"] < st["traversable"]
    # paths to random reachable cells of the last field (clearance 0.2)
    ri, _ = f2.reachable()
    tg = ri[rng.choice(len(ri), min(64, len(ri)), replace=False)].astype(F32) * F32(VS)
    check_paths(h, f2, tg)


def two_rooms(h):
    """Room A around the origin, room B behind a wall at x = 1 m (cells i = 20, |j|, |k| <= 20), joined by a 5 x 5 cell
    doorway at |j|, |k| <= 2; built from point rays: from A to the wall and through the doorway to B's back wall at
    x = 2 m, and from B (1.5 m) to the back of the wall and to its back wall."""
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
    """hits on the 25 doorway cells until they are OCC"""
    g = np.arange(-2, 3)
    J, K = np.meshgrid(g, g, indexing="ij")
    dcell = np.stack([np.full(J.size, 20), J.ravel(), K.ravel()], 1).astype(F32) * F32(VS)
    for _ in range(4):
        h.integrate_points(dcell, np.eye(3), np.zeros(3))


def test_two_rooms_doorway():
    h = handle(128, 128, min_ray_length=0.0)
    two_rooms(h)
    st, f = check_field(h, np.zeros(3, F32))
    target = np.array([1.25, 0.5, 0.5], F32)                # cell (25,10,10): on B's ray to the wall cell (20,20,20)
    g = h.travel_query(target[None])[0]
    assert np.isfinite(g) and g > np.linalg.norm(target)
    c = np.array([25, 10, 10])                               # the 26-neighbour chamfer distance without the wall
    s = np.sort(np.abs(c))[::-1]
    chamfer = s[2] * math.sqrt(3) * VS + (s[1] - s[2]) * math.sqrt(2) * VS + (s[0] - s[1]) * VS
    assert g > chamfer
    cells, ln = check_paths(h, f, target[None])
    p = cells[0, :ln[0]]
    at_wall = p[p[:, 0] == 20]
    assert at_wall.shape[0] >= 1 and (np.abs(at_wall[:, 1:]) <= 2).all()
    assert (p[-1] == 0).all() and (p[0] == np.array([25, 10, 10])).all()
    # close the doorway: the far room is unreachable
    close_door(h)
    st2, f2 = check_field(h, np.zeros(3, F32))
    assert np.isinf(h.travel_query(target[None])[0]) and st2["reachable"] < st["reachable"]
    assert h.travel_path(target[None])[1][0] == 0


def test_block_seams_and_a_start_on_a_block_corner():
    h = handle(64, 64, min_ray_length=0.0)
    rng = np.random.default_rng(3)
    T = np.array([-0.05, -0.05, -0.05])                       # cell (-1,-1,-1): the high corner of block (-1,-1,-1)
    for q in range(3):
        d = rng.normal(size=(400, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        pts = (d * rng.uniform(0.4, 1.4, (400, 1))).astype(F32)
        h.integrate_points(pts, np.eye(3), T)
    g = np.argwhere(np.ones((4, 4, 4), bool)) * 8 - 9         # a shell of OCC points on the seams i & 7 == 7
    g = g[~(g == -1).all(1)]                                  # (but not on the start)
    h.integrate_points((g.astype(F32) * F32(VS) - T.astype(F32)).astype(F32), np.eye(3), T)
    st, f = check_field(h, T.astype(F32))
    assert st["start_ok"]
    ri, _ = f.reachable()
    blocks = np.unique(ri >> 3, axis=0)
    assert blocks.shape[0] >= 27
    tg = ri[rng.choice(len(ri), 128, replace=False)].astype(F32) * F32(VS)
    cells, ln = check_paths(h, f, tg)
    crossings = sum(int((np.diff(cells[q, :ln[q]] >> 3, axis=0) != 0).any(1).sum()) for q in range(len(tg)))
    assert crossings > 100


def test_queries_and_paths():
    h = handle()
    d = syn.scene_room()
    h.integrate_depth(d, np.eye(3), np.zeros(3))
    h.integrate_depth(d, rot_xyz(0.0, 0.3, 0.1), np.array([0.1, 0.0, 0.05]))
    st, f = check_field(h, np.zeros(3, F32), max_cost=2.0)
    rng = np.random.default_rng(9)
    ri, rG = f.reachable()
    idx, L = h.gather(0)
    n = 1 << 16
    a = ri[rng.integers(len(ri), size=n // 2)].astype(F32) * F32(VS) + rng.uniform(-0.45, 0.45, (n // 2, 3)).astype(F32) * F32(VS)
    b = idx[rng.integers(len(idx), size=n // 4)].astype(F32) * F32(VS)          # known cells, many unreachable
    c = rng.uniform(-8.0, 8.0, (n // 4, 3)).astype(F32)                         # mostly unknown or outside the volume
    c[:64, 0] = np.nan
    c[64:128, 1] = np.inf
    xyz = np.concatenate([a, b, c]).astype(F32)
    g = h.travel_query(xyz)
    want = f.query(xyz, h.N, h.Nz)
    assert np.array_equal(g.view(np.int32), want.view(np.int32))
    assert np.isfinite(g).mean() > 0.5 and np.isinf(g).sum() > 1000
    # torch in -> torch out
    import torch
    tg = h.travel_query(torch.from_numpy(xyz).cuda())
    assert isinstance(tg, torch.Tensor) and np.array_equal(tg.cpu().numpy().view(np.int32), g.view(np.int32))
    # 256 paths, full and truncated, and to unreachable targets
    targets = np.concatenate([ri[rng.choice(len(ri), 240, replace=False)].astype(F32) * F32(VS), b[:16]]).astype(F32)
    cells, ln = check_paths(h, f, targets)
    assert (ln[:240] > 0).all()
    short, sl = check_paths(h, f, targets, max_len=5)
    assert np.array_equal(sl, ln) and (ln > 5).any()
    # more integration changes nothing the readers return; blocks allocated since read +inf
    before = {tuple(x) for x in (idx >> 3).tolist()}
    h.integrate_depth(d, rot_xyz(0.0, 2.5, 0.0), np.array([0.0, 0.2, 0.0]))
    assert np.array_equal(h.travel_query(xyz).view(np.int32), g.view(np.int32))
    c2, l2 = h.travel_path(targets)
    assert np.array_equal(l2, ln) and all(np.array_equal(c2[q, :ln[q]], cells[q, :ln[q]]) for q in range(len(targets)))
    i2, _ = h.gather(0)
    new = np.array([x for x in i2.tolist() if tuple(np.array(x) >> 3) not in before])
    assert len(new) > 0
    assert np.isinf(h.travel_query(new[:4096].astype(F32) * F32(VS))).all()
    gi, gG = as_dict_rows(*h.travel_gather(0))
    assert np.array_equal(gi, as_dict_rows(*f.reachable())[0])


def test_stale_esdf_two_submaps_reset_fusion_and_recycled_slots():
    h = handle(128, 128, max_submaps=2)
    d = syn.scene_room()
    h.integrate_depth(d, np.eye(3), np.zeros(3))
    h.esdf_update(0, D)
    esdf = h.esdf_gather(0)
    h.integrate_depth(d, rot_xyz(0.0, 0.8, 0.0), np.array([0.1, 0.0, 0.0]))      # after the ESDF update: stale
    st, f = check_field(h, np.zeros(3, F32), clearance=0.15, esdf=esdf)
    assert st["start_ok"] and st["traversable"] < free_cells(h).shape[0]
    # two submaps
    h.integrate_depth(syn.scene_sphere(3.0), np.eye(3), np.zeros(3), submap=1)
    refused(h.travel_update, 1, np.zeros(3), clearance=0.1)                    # no ESDF of submap 1
    check_field(h, np.zeros(3, F32), submap=1)
    refused(h.travel_gather, 0)
    refused(h.travel_query, np.zeros((4, 3), F32), 0)
    refused(h.travel_path, np.zeros((4, 3), F32), 0)
    check_field(h, np.zeros(3, F32), submap=0)
    # reset: readers refuse until the next update; recycled pool slots leak nothing
    h.reset()
    refused(h.travel_gather, 0)
    refused(h.travel_query, np.zeros((4, 3), F32), 0)
    h.integrate_points(np.array([[1.0, 0.2, 0.3], [0.1, 1.2, 0.0]], F32), np.eye(3), np.zeros(3))
    st, f = check_field(h, np.zeros(3, F32))
    assert st["start_ok"] and 0 < st["reachable"] < 200
    h.integrate_depth(d, rot_xyz(0.0, 0.2, 0.0), np.zeros(3))
    check_field(h, np.zeros(3, F32))
    # fusion
    src = handle(128, 128)
    src.integrate_depth(d, np.eye(3), np.zeros(3))
    h.set_submap_pose(0, np.eye(3), np.zeros(3))
    h.fuse_from(src)
    refused(h.travel_gather, 0)
    refused(h.travel_path, np.zeros((1, 3), F32), 0)
    check_field(h, np.zeros(3, F32))


def test_invalid_starts_are_not_errors():
    h = handle(128, 128)
    h.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    h.esdf_update(0, D)
    idx, L = h.gather(0)
    occ = idx[L > LO["l_occ"]][0].astype(F32) * F32(VS)
    e_i, e_E = h.esdf_gather(0)
    near = e_i[(e_E > 0) & (e_E < 0.1)][0].astype(F32) * F32(VS)
    for s, cl in [(occ, 0.0), (np.array([3.1, 3.1, 3.1], F32), 0.0), (np.array([100.0, 0, 0], F32), 0.0), (near, 0.2),
                  (np.array([-3.2, 0.0, 0.0], F32), 0.0)]:
        st, _ = check_field(h, s, clearance=cl)
        assert not st["start_ok"] and st["reachable"] == 0 and st["sweeps"] == 1, (s, st)
        assert np.isinf(h.travel_query(np.zeros((1, 3), F32))[0])


def test_no_side_effects():
    a, b = handle(128, 128), handle(128, 128)
    d = syn.scene_room()
    for h in (a, b):
        h.integrate_depth(d, np.eye(3), np.zeros(3))
        h.esdf_update(0, D)
        h.frontier_update(0)
    a.travel_update(0, np.zeros(3), clearance=0.1)
    a.travel_query(np.zeros((8, 3), F32))
    a.travel_path(np.full((8, 3), 0.3, F32))
    a.travel_gather(0)
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
    fo = torch.zeros(4, dtype=torch.float32, device=dev)
    ci = torch.zeros((4, 8, 3), dtype=torch.int32, device=dev)
    li = torch.zeros(4, dtype=torch.int32, device=dev)
    X, FO, CI, LI = (capi.tptr(t) for t in (x, fo, ci, li))
    zero = np.zeros(3, F32)
    n64 = C.c_int64(0)

    def upd(h, start=zero, cl=0.0, mc=1.0, sub=0):
        return L.tslam_octo_travel_update(h.h, sub, capi.np_ptr(np.asarray(start, F32)) if start is not None else None, cl, mc, None, None)

    def gat(h, sub=0):
        return L.tslam_octo_travel_gather(h.h, sub, 0, None, None, C.byref(n64), None)

    def qry(h, sub=0, n=4, xyz=X, out=FO):
        return L.tslam_octo_travel_query(h.h, sub, n, xyz, out, None)

    def pth(h, sub=0, n=4, xyz=X, max_len=8, cells=CI, ln=LI):
        return L.tslam_octo_travel_path(h.h, sub, n, xyz, max_len, cells, ln, None)

    hits = OctoHandle(64, 64, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH)
    assert upd(hits) == capi.E_INVALID and gat(hits) == capi.E_INVALID and qry(hits) == capi.E_INVALID and pth(hits) == capi.E_INVALID
    h = handle(64, 64, max_submaps=2)
    h.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    assert gat(h) == capi.E_INVALID and qry(h) == capi.E_INVALID and pth(h) == capi.E_INVALID   # before any update
    assert upd(h, start=None) == capi.E_INVALID
    for s in ((np.nan, 0, 0), (0, np.inf, 0), (0, 0, -np.inf)):
        assert upd(h, start=s) == capi.E_INVALID, s
    limit = h.travel_limit()
    for cl, mc in ((-0.1, 1.0), (np.nan, 1.0), (np.inf, 1.0), (0.0, 0.0), (0.0, -1.0), (0.0, np.nan), (0.0, np.inf),
                   (0.0, float(np.nextafter(F32(limit), F32(np.inf))))):
        assert upd(h, cl=cl, mc=mc) == capi.E_INVALID, (cl, mc)
    assert upd(h, mc=limit) == capi.TSLAM_OK
    assert upd(h, cl=0.1) == capi.E_INVALID                     # clearance without an ESDF
    h.esdf_update(0, 0.5)
    assert upd(h, cl=0.5) == capi.TSLAM_OK and upd(h, cl=float(np.nextafter(F32(0.5), F32(1)))) == capi.E_INVALID
    assert upd(h, cl=0.1, sub=1) == capi.E_INVALID              # the ESDF is of submap 0
    assert upd(h, sub=2) == capi.E_INVALID and upd(h, sub=-1) == capi.E_INVALID
    assert upd(h) == capi.TSLAM_OK
    for sub in (1, 2, -1):
        assert gat(h, sub) == capi.E_INVALID and qry(h, sub) == capi.E_INVALID and pth(h, sub) == capi.E_INVALID
    assert qry(h, n=-1) == capi.E_INVALID and qry(h, xyz=None) == capi.E_INVALID and qry(h, out=None) == capi.E_INVALID
    assert pth(h, n=-1) == capi.E_INVALID and pth(h, xyz=None) == capi.E_INVALID and pth(h, cells=None) == capi.E_INVALID
    assert pth(h, ln=None) == capi.E_INVALID and pth(h, max_len=0) == capi.E_INVALID and pth(h, max_len=-3) == capi.E_INVALID
    assert qry(h, n=0, xyz=None, out=None) == capi.TSLAM_OK and pth(h, n=0, xyz=None, cells=None, ln=None) == capi.TSLAM_OK
    assert L.tslam_octo_travel_gather(h.h, 0, 4, None, None, C.byref(n64), None) == capi.E_INVALID
    assert L.tslam_octo_travel_gather(h.h, 0, -1, None, None, C.byref(n64), None) == capi.E_INVALID
    n = h.travel_update(0, zero)["reachable"]
    assert n > 1 and L.tslam_octo_travel_gather(h.h, 0, 1, CI, FO, C.byref(n64), None) == capi.E_CAPACITY and n64.value == n
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
    st = o.travel_update(np.zeros(3), clearance=0.1)            # runs esdf_update(max_ray_length) first
    assert st["start_ok"] and o.esdf_max_dist == 3.0
    f = reference(o._h, np.zeros(3, F32), 0.1)
    gi, gG = as_dict_rows(*o._h.travel_gather(0))
    ri, rG = as_dict_rows(*f.reachable())
    assert np.array_equal(gi, ri) and np.array_equal(gG.view(np.int32), rG.view(np.int32))
    rng = np.random.default_rng(2)
    pts = ri[rng.choice(len(ri), 100, replace=False)].astype(F32) * F32(VS)
    c = o.travel_cost(pts)
    assert isinstance(c, np.ndarray) and np.array_equal(c.view(np.int32), f.query(pts, o.N, o.Nz).view(np.int32))
    ct = o.travel_cost(torch.from_numpy(pts).cuda())
    assert isinstance(ct, torch.Tensor) and ct.is_cuda and np.array_equal(ct.cpu().numpy(), c)
    far = pts[np.argmax(c)]
    path = o.travel_path(far, max_len=4)                        # retried with the reported length
    want = f.path(far)[::-1]
    assert path.shape == (want.shape[0], 3) and want.shape[0] > 4
    assert np.array_equal(path, want.astype(np.float64) * float(F32(VS)))
    assert np.array_equal(o.travel_path(torch.from_numpy(far).cuda()), path)
    assert o.travel_path(np.array([6.0, 6.0, 6.0])) is None
    with pytest.raises(ValueError):
        o.travel_update(np.zeros(3), clearance=3.5)
    o.esdf_update(1.0)
    with pytest.raises(ValueError):
        o.travel_update(np.zeros(3), clearance=1.5)
    assert "start_ok" in o.travel_update(np.zeros(3), clearance=0.5)
    hits = Octomap(map_scale=[3.2, 3.2], voxel_scale=VS, max_disp_particles=16)
    for call in (lambda: hits.travel_update(np.zeros(3)), lambda: hits.travel_cost(np.zeros((1, 3))),
                 lambda: hits.travel_path(np.zeros(3))):
        with pytest.raises(ValueError):
            call()
