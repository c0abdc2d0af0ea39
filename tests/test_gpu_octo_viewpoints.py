"""Frontier viewpoints of the log-odds Octomap on the GPU against the numpy reference (octo_viewpoint_reference.py): counts,
samples, scores and poses bit for bit, scores equal to the frontier gain of the returned poses, and plan_exploration
equal to the public calls it composes."""
import ctypes as C

import numpy as np
import pytest

import octo_frontier_reference as fr
import octo_logodds_reference as ref
import octo_viewpoint_reference as vp
from taichislam_b200 import synthetic as syn
from taichislam_b200.mapping.taichi_octomap import Octomap
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu

VS = 0.05
LO = ref.params()
F32 = np.float32
D = 1.0
CAM_S = dict(fx=syn.FX / 4, fy=syn.FY / 4, cx=syn.CX / 4, cy=syn.CY / 4, width=160, height=120, step=2, max_range=3.0)
OFFS = Octomap.viewpoint_offsets(radii=(0.5, 1.0, 1.5), angles=16, heights=(0.0, 0.3))
SCENES = {"S1": lambda: syn.scene_plane(3.0), "S2": lambda: syn.scene_sphere(4.0), "S4": lambda: syn.scene_noise(4),
          "room": lambda: syn.scene_room()}


def handle(N=256, Nz=256, **kw):
    from taichislam_b200.octo_handle import OctoHandle
    kw.setdefault("Kcam", syn.K_DEPTH)
    kw.setdefault("max_ray_length", 5.0)
    return OctoHandle(N, Nz, K=2, voxel_scale=VS, logodds=LO, **kw)


def mapped(scene, N=256, frames=2, **kw):
    h = handle(N, N, **kw)
    d = SCENES[scene]()
    Rs, Ts = syn.stream_poses(frames, start=40)
    for q in range(frames):
        h.integrate_depth(d, Rs[q], Ts[q])
    return h


def check(h, offsets=OFFS, cam=CAM_S, clearance=0.0, min_visible=1, top_k=1, submap=0, frontier=None):
    """the GPU outputs against the reference; frontier = (fidx, fcl, rec) of the last update when the map changed since"""
    count, sample, visible, pos, R = h.frontier_viewpoints(offsets, cam, clearance, min_visible, top_k, submap=submap)
    idx, L = h.gather(submap)
    if frontier is None:
        fidx, fcl = h.frontier_gather(submap)
        ri, rc, rr = fr.frontiers(idx, L, LO["l_occ"], h.N, h.Nz)
        gi, gc = as_dict_rows(fidx, fcl)
        assert np.array_equal(gi, ri) and np.array_equal(gc, rc)
        assert np.array_equal(h.frontier_clusters(submap), rr)
        frontier = (fidx, fcl, rr)
    esdf = h.esdf_gather(submap) if clearance > 0 else None
    r = vp.viewpoints(idx, L, LO["l_occ"], h.N, h.Nz, VS, offsets, cam, clearance, esdf, min_visible, top_k, frontier)
    assert np.array_equal(count, r["count"]), (count, r["count"])
    bad = np.nonzero((sample != r["sample"]).any(1) | (visible != r["visible"]).any(1))[0]
    assert bad.size == 0, f"{bad.size} clusters differ, first {bad[:3].tolist()}: gpu {sample[bad[:3]].tolist()} / " \
                          f"{visible[bad[:3]].tolist()} ref {r['sample'][bad[:3]].tolist()} / {r['visible'][bad[:3]].tolist()}"
    assert np.array_equal(pos.view(np.int32), r["pos"].view(np.int32)) and np.array_equal(R.view(np.int32), r["R"].view(np.int32))
    return count, sample, visible, pos, R, r


def check_against_view_gain(h, out, cam=CAM_S, submap=0):
    """visible[c, j] = per_cluster[v, c] of view_gain_frontier for the returned pose v"""
    count, sample, visible, pos, R = out[:5]
    c, j = np.nonzero(np.arange(sample.shape[1])[None, :] < count[:, None])
    if c.size == 0:
        return 0
    v, _, per = h.view_gain_frontier(pos[c, j], R[c, j], cam, submap=submap)
    assert v.all()
    assert np.array_equal(per[np.arange(c.size), c], visible[c, j])
    return c.size


@pytest.mark.parametrize("clearance", [0.0, 0.2])
@pytest.mark.parametrize("scene", list(SCENES))
def test_matches_reference(scene, clearance):
    h = mapped(scene)
    if clearance > 0:
        h.esdf_update(0, D)
    st = h.frontier_update(0)
    out = check(h, clearance=clearance, top_k=1 if scene != "room" else 4)
    r = out[5]
    assert st["clusters"] == out[0].shape[0]
    assert scene == "S1" or clearance > 0 or out[0].sum() > 0
    assert not r["valid"].all()                                      # some samples land in OCC / UNKNOWN cells
    n = check_against_view_gain(h, out)
    assert scene == "S1" or clearance > 0 or n > 0
    if scene == "room":
        check(h, clearance=clearance, min_visible=20, top_k=3)
        check(h, offsets=OFFS[:1], clearance=clearance, top_k=2)


def test_full_camera_and_many_samples():
    h = mapped("room")
    h.frontier_update(0)
    cam = dict(fx=syn.FX, fy=syn.FY, cx=syn.CX, cy=syn.CY, width=640, height=480, step=2, max_range=5.0)
    offs = Octomap.viewpoint_offsets(radii=(0.5, 1.0, 1.5, 2.0), angles=32, heights=(0.0, 0.2, -0.2, 0.4, -0.4, 0.6, 0.8, -0.6))
    assert offs.shape[0] == 1024
    out = check(h, offsets=offs, cam=cam, top_k=2)
    check_against_view_gain(h, out, cam)


def test_two_submaps():
    h = handle(max_submaps=2)
    h.integrate_depth(syn.scene_sphere(3.0), np.eye(3), np.zeros(3), submap=0)
    h.integrate_depth(syn.scene_room(), rot_xyz(0.0, 0.0, 1.0), np.array([0.4, 0.0, 0.0]), submap=1)
    h.frontier_update(1)
    refused(h.frontier_viewpoints, OFFS, CAM_S, submap=0)
    a = check(h, submap=1, top_k=2)
    h.frontier_update(0)
    refused(h.frontier_viewpoints, OFFS, CAM_S, submap=1)
    b = check(h, submap=0, top_k=2)
    assert a[0].sum() > 0 and b[0].sum() > 0


def refused(fn, *a, **kw):
    from taichislam_b200 import _capi as capi
    with pytest.raises(capi.TslamError) as e:
        fn(*a, **kw)
    assert e.value.code == capi.E_INVALID


def test_stale_frontier_set_reset_and_fusion():
    h = mapped("room", 128)
    h.frontier_update(0)
    fidx, fcl = h.frontier_gather(0)
    rec = h.frontier_clusters(0)
    h.integrate_depth(syn.scene_room(), rot_xyz(0.0, 0.3, 0.8), np.array([0.3, 0.1, 0.0]))   # no update after it
    out = check(h, top_k=2, frontier=(fidx, fcl, rec))     # the last update's rows, the classes as of the call
    assert out[0].sum() > 0
    h.reset()
    refused(h.frontier_viewpoints, OFFS, CAM_S)
    h.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    h.frontier_update(0)
    check(h)
    src = handle(128, 128)
    src.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    h.set_submap_pose(0, np.eye(3), np.zeros(3))
    h.fuse_from(src)
    refused(h.frontier_viewpoints, OFFS, CAM_S)
    h.sync()


def test_refusals():
    import torch
    from taichislam_b200 import _capi as capi
    from taichislam_b200.octo_handle import OctoHandle
    L = capi.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    off = torch.from_numpy(OFFS).to(dev)
    buf = torch.zeros(1 << 16, dtype=torch.int32, device=dev)
    cam = OctoHandle.view_camera(CAM_S)
    O, B = capi.tptr(off), capi.tptr(buf)

    def call(h, S=OFFS.shape[0], c=cam, o=O, cl=0.0, mv=1, k=2, nc=None, sub=0, outs=(B,) * 5):
        nc = h.frontier_clusters(sub).shape[0] if nc is None else nc
        return L.tslam_octo_frontier_viewpoints(h.h, sub, C.byref(c) if c is not None else None, S, o, cl, mv, k, nc, *outs, None)

    hits = OctoHandle(64, 64, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH)
    assert call(hits, nc=0) == capi.E_INVALID
    h = handle(64, 64, max_submaps=2)
    h.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    assert call(h, nc=0) == capi.E_INVALID                                   # before any frontier update
    h.frontier_update(0)
    nc = h.frontier_clusters(0).shape[0]
    assert nc > 1 and nc * 2 * 13 < buf.numel()
    assert call(h) == capi.TSLAM_OK
    for kw in (dict(c=None), dict(o=None), dict(outs=(None,) + (B,) * 4), dict(outs=(B,) * 4 + (None,)), dict(S=0), dict(S=1025),
               dict(k=0), dict(k=1025), dict(mv=0), dict(mv=-3), dict(cl=float("nan")), dict(cl=-0.1), dict(cl=float("inf")),
               dict(cl=0.1), dict(nc=nc + 1), dict(nc=nc - 1), dict(sub=2, nc=nc), dict(sub=-1, nc=nc), dict(sub=1, nc=nc)):
        assert call(h, **kw) == capi.E_INVALID, kw
    for bad in (dict(fx=0.0), dict(fx=float("nan")), dict(fy=-1.0), dict(max_range=0.0), dict(max_range=float("inf")),
                dict(cx=float("nan")), dict(cy=float("inf")), dict(width=0), dict(height=-1), dict(step=0),
                dict(width=3, step=4), dict(height=1, step=2), dict(fx=1e-30)):
        assert call(h, c=OctoHandle.view_camera(dict(CAM_S, **bad))) == capi.E_INVALID, bad
    h.esdf_update(0, 0.5)
    assert call(h, cl=0.5) == capi.TSLAM_OK and call(h, cl=0.51) == capi.E_INVALID       # clearance above the ESDF's D
    big = torch.from_numpy(np.resize(OFFS, (1024, 3))).to(dev)                # the largest n_samples and top_k
    outs = [torch.empty((nc, 1024, w), dtype=torch.float32, device=dev) for w in (1, 1, 1, 3, 9)]
    assert call(h, S=1024, o=capi.tptr(big), k=1024, outs=tuple(capi.tptr(t) for t in outs)) == capi.TSLAM_OK
    cnt = outs[0].reshape(-1)[:nc].view(torch.int32).cpu().numpy()            # count int32[nc]
    assert 0 < cnt.max() <= 1024
    with pytest.raises(ValueError):                                          # the Octomap surface: a hit counter
        o = Octomap(map_scale=[3.2, 3.2], voxel_scale=VS, max_disp_particles=16)
        o.set_dep_camera_intrinsic(syn.K_DEPTH)
        o.frontier_viewpoints(160, 120)


def test_zero_clusters():
    h = handle(64, 64)
    assert h.frontier_update(0)["clusters"] == 0                             # an empty map
    count, sample, visible, pos, R = h.frontier_viewpoints(OFFS, CAM_S, top_k=3)
    assert count.shape == (0,) and sample.shape == (0, 3) and pos.shape == (0, 3, 3) and R.shape == (0, 3, 3, 3)


def test_no_side_effects():
    a, b = handle(128, 128), handle(128, 128)
    d = syn.scene_room()
    for h in (a, b):
        h.integrate_depth(d, np.eye(3), np.zeros(3))
        h.esdf_update(0, D)
        h.frontier_update(0)
    a.frontier_viewpoints(OFFS, CAM_S, clearance=0.1, top_k=4)
    a.frontier_viewpoints(OFFS, CAM_S)
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
    assert sa == sb and not sa["full"]                  # same re-examined block count as the twin
    assert np.array_equal(a.frontier_clusters(0), b.frontier_clusters(0))


def test_torch_and_numpy():
    import torch
    h = mapped("S2")
    h.frontier_update(0)
    n = h.frontier_viewpoints(OFFS, CAM_S, top_k=3)
    t = h.frontier_viewpoints(torch.from_numpy(OFFS).cuda(), CAM_S, top_k=3)
    for a, b in zip(n, t):
        assert isinstance(b, torch.Tensor) and b.is_cuda
        assert np.array_equal(a, b.cpu().numpy())


def octomap_room():
    o = Octomap(map_scale=[12.8, 12.8], voxel_scale=VS, occupancy_model="logodds", max_ray_length=3.0, max_disp_particles=1024)
    o.set_dep_camera_intrinsic(syn.K_DEPTH)
    o.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    d = syn.scene_room()
    o.recast_depth_to_map(np.eye(3), np.zeros(3), d, None)
    o.recast_depth_to_map(rot_xyz(0.0, 0.0, 0.4), np.array([0.1, 0.0, 0.0]), d, None)
    return o


@pytest.mark.parametrize("clearance", [0.0, 0.1])
def test_plan_exploration_is_the_public_calls_composed(clearance):
    o = octomap_room()
    start = np.array([0.0, 0.0, 0.0])
    kw = dict(radii=(0.5, 1.0), angles=12, heights=(0.0,), clearance=clearance, min_visible=5, top_k=3)
    plan = o.plan_exploration(start, 320, 240, min_voxels=8, restarts=16, seed=3, **kw)
    # by hand
    fv = o.frontier_viewpoints(320, 240, **kw)
    cl = o.get_frontier_clusters()
    cam = dict(fx=syn.FX, fy=syn.FY, cx=syn.CX, cy=syn.CY, width=320, height=240, step=o.recast_step, max_range=3.0)
    offs = Octomap.viewpoint_offsets((0.5, 1.0), 12, (0.0,))
    ref_out = o._h.frontier_viewpoints(offs, cam, clearance, 5, 3)
    assert all(np.array_equal(fv[k], v) for k, v in zip(("count", "sample", "visible", "pos", "R"), ref_out))
    o.travel_update(start, clearance)
    goals, none = [], []                    # (cluster, slot) of each cluster's best reachable viewpoint; clusters without
    for c in range(cl["size"].shape[0]):
        if cl["size"][c] < 8:
            continue
        n = int(fv["count"][c])
        cost = o.travel_cost(fv["pos"][c, :n]) if n else np.zeros(0, F32)
        fin = np.nonzero(np.isfinite(cost))[0]
        if fin.size:
            goals.append((c, int(fin[0])))
        else:
            none.append(c)
    assert len(goals) > 1
    gpos = np.array([fv["pos"][c, j] for c, j in goals], F32)
    tour = o.exploration_tour(start, gpos, clearance, restarts=16, seed=3)
    order = np.array([goals[q][0] for q in tour["order"]])
    assert np.array_equal(plan["clusters"], order)
    assert np.array_equal(plan["unreachable"], np.sort(np.array(none + [goals[q][0] for q in tour["unreachable"]], np.int64)))
    assert np.array_equal(plan["pos"], gpos[tour["order"]])
    assert np.array_equal(plan["yaw"], np.arctan2(plan["R"][:, 0, 0].astype(np.float64), plan["R"][:, 0, 2].astype(np.float64)))
    assert np.array_equal(plan["visible"], np.array([fv["visible"][c, j] for c, j in goals])[tour["order"]])
    assert plan["cost"] == tour["cost"] and np.array_equal(plan["leg_costs"], tour["leg_costs"])
    assert plan["inf_legs"] == tour["inf_legs"] and plan["converged"] == tour["converged"]
    assert np.array_equal(plan["path"], tour["path"])
    # the first path runs from the start's cell to the first viewpoint's cell through FREE cells only
    path = plan["path"]
    occ, unk = o._h.query_points(path.astype(F32))
    assert not occ.any() and not unk.any()
    vs = float(np.float32(VS))
    assert np.array_equal(np.rint(path[-1] / vs), ref.round_half_away(plan["pos"][0] / np.float32(VS)))
    assert np.abs(np.diff(np.rint(path / vs), axis=0)).max() <= 1


def test_plan_exploration_without_qualifying_clusters_and_with_too_many():
    o = octomap_room()
    plan = o.plan_exploration(np.zeros(3), 320, 240, radii=(0.5, 1.0), angles=12, min_voxels=1 << 30)
    assert plan["clusters"].size == 0 and plan["unreachable"].size == 0 and plan["path"] is None
    # 1024 clusters with a reachable viewpoint are more than a tour takes (the start is the 1024th point)
    k = 1024
    o.frontier_viewpoints = lambda *a, **kw: dict(count=np.ones(k, np.int32), pos=np.zeros((k, 1, 3), F32),
                                                  R=np.zeros((k, 1, 3, 3), F32), yaw=np.zeros((k, 1)),
                                                  visible=np.ones((k, 1), np.int32), sample=np.zeros((k, 1), np.int32))
    o.get_frontier_clusters = lambda min_voxels=1: dict(size=np.ones(k, np.int64))
    o.travel_cost = lambda xyz: np.zeros(len(xyz), F32)
    with pytest.raises(ValueError):
        o.plan_exploration(np.zeros(3), 320, 240)
