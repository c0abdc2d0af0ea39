"""Viewpoint gain of the log-odds Octomap on the GPU against the numpy reference (octo_view_gain_reference.py): valid
flags, unknown gains, frontier totals and per-cluster counts, bit for bit."""
import ctypes as C
import math

import numpy as np
import pytest

import octo_frontier_reference as fr
import octo_logodds_reference as ref
import octo_view_gain_reference as vg
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu

VS = 0.05
LO = ref.params()
F32 = np.float32
CAM_S = dict(fx=syn.FX / 4, fy=syn.FY / 4, cx=syn.CX / 4, cy=syn.CY / 4, width=160, height=120, step=2, max_range=3.0)
CAM_F = dict(fx=syn.FX, fy=syn.FY, cx=syn.CX, cy=syn.CY, width=640, height=480, step=2, max_range=5.0)


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


def views(h, n, seed, submap=0, invalid=True):
    """n views on FREE cells (jittered inside the cell) with random rotations, then invalid ones: on OCC cells, outside
    the volume, in unknown space at a volume corner, and with NaN / inf numbers"""
    rng = np.random.default_rng(seed)
    idx, L = h.gather(submap)
    free, occ = idx[L <= LO["l_occ"]], idx[L > LO["l_occ"]]
    pick = free[rng.choice(len(free), n, replace=False)]
    pos = (pick.astype(F32) * F32(VS) + rng.uniform(-0.4, 0.4, (n, 3)).astype(F32) * F32(VS)).astype(F32)
    R = np.stack([rot_xyz(rng.uniform(-0.6, 0.6), rng.uniform(-math.pi, math.pi), rng.uniform(-math.pi, math.pi))
                  for _ in range(n)]).astype(F32)
    if invalid:
        bad = [occ[0] * VS, occ[-1] * VS, (100.0, 0.0, 0.0), (-(h.N // 2 - 1) * VS, -(h.N // 2 - 1) * VS, (h.Nz // 2 - 2) * VS),
               (np.nan, 0.0, 0.0), (0.0, np.inf, 0.0), pick[0] * VS, pick[1] * VS]
        bR = np.repeat(np.eye(3, dtype=F32)[None], len(bad), 0)
        bR[6, 2, 2] = np.nan
        bR[7, 0, 1] = np.inf
        pos = np.concatenate([pos, np.asarray(bad, F32)])
        R = np.concatenate([R, bR])
    return pos.astype(F32), R.astype(F32)


def check_unknown(h, pos, R, cam, submap=0):
    gv, gg = h.view_gain_unknown(pos, R, cam, submap=submap)
    idx, L = h.gather(submap)
    rv, rg = vg.unknown_gain(idx, L, LO["l_occ"], h.N, h.Nz, VS, pos, R, cam)
    assert np.array_equal(gv, rv), f"valid: gpu {gv.astype(int).tolist()} ref {rv.astype(int).tolist()}"
    bad = np.nonzero(gg != rg)[0]
    assert bad.size == 0, f"{bad.size} unknown gains differ, first {bad[:4].tolist()}: gpu {gg[bad[:4]].tolist()} ref {rg[bad[:4]].tolist()}"
    return gv, gg


def check_frontier(h, pos, R, cam, submap=0, stale=None):
    """stale = (fidx, fcl, n_clusters) of the last update when the map changed since; else the update is current and its
    frontier set must equal the reference's"""
    gv, gt, gp = h.view_gain_frontier(pos, R, cam, submap=submap)
    idx, L = h.gather(submap)
    if stale is None:
        fidx, fcl = h.frontier_gather(submap)
        ri, rc, rr = fr.frontiers(idx, L, LO["l_occ"], h.N, h.Nz)
        gi, gc = as_dict_rows(fidx, fcl)
        assert np.array_equal(gi, ri) and np.array_equal(gc, rc)   # cluster ordinals = frontier_gather's
        stale = (fidx, fcl, rr.shape[0])
    rv, rt, rp = vg.frontier_gain(idx, L, LO["l_occ"], h.N, h.Nz, VS, pos, R, cam, *stale)
    assert np.array_equal(gv, rv)
    assert gp.shape == rp.shape
    bad = np.nonzero((gp != rp).any(1))[0]
    assert bad.size == 0, f"{bad.size} views differ, first {bad[:4].tolist()}: gpu {gt[bad[:4]].tolist()} ref {rt[bad[:4]].tolist()}"
    assert np.array_equal(gt, rt) and np.array_equal(gp.sum(1), gt)
    return gv, gt, gp


SCENES = {"S1": lambda: syn.scene_plane(3.0), "S2": lambda: syn.scene_sphere(4.0), "S4": lambda: syn.scene_noise(4),
          "room": lambda: syn.scene_room()}


@pytest.mark.parametrize("scene", list(SCENES))
def test_matches_reference(scene):
    h = handle()
    d = SCENES[scene]()
    Rs, Ts = syn.stream_poses(2, start=40)
    for q in range(2):
        h.integrate_depth(d, Rs[q], Ts[q])
    h.frontier_update(0)
    pos, R = views(h, 96, seed=len(scene))
    gv, gg = check_unknown(h, pos, R, CAM_S)
    assert gv[:96].all() and not gv[96:].any() and (gg[:96] > 0).mean() > 0.5 and (gg[96:] == 0).all()
    gv, gt, gp = check_frontier(h, pos, R, CAM_S)
    assert (gt[96:] == 0).all() and (gp[96:] == 0).all()
    assert scene == "S1" or gt.max() > 0
    # a few views with the full 640 x 480 camera, 5 m
    check_unknown(h, pos[:3], R[:3], CAM_F)
    check_frontier(h, pos[:3], R[:3], CAM_F)


def test_sensor_model_cross_check():
    """On a map without OCC cells the gain is what an all-far frame from the view adds to the known voxels."""
    h = handle()
    far = np.full((syn.H, syn.W), 65535, np.uint16)
    for q in range(3):
        R, T = syn.stream_pose(200 * q)
        h.integrate_depth(far, R, T)
    cam = dict(fx=syn.FX, fy=syn.FY, cx=syn.CX, cy=syn.CY, width=syn.W, height=syn.H, step=2, max_range=5.0)
    rng = np.random.default_rng(7)
    for q in range(5):
        idx, L = h.gather(0)
        assert (L <= LO["l_occ"]).all()
        p = (idx[rng.integers(len(idx))].astype(F32) * F32(VS)).astype(F32)
        R = rot_xyz(rng.uniform(-0.5, 0.5), rng.uniform(-3, 3), rng.uniform(-3, 3)).astype(F32)
        valid, gain = h.view_gain_unknown(p[None], R[None], cam)
        assert valid[0] and gain[0] > 0
        h.integrate_depth(far, R.astype(np.float64), p.astype(np.float64))
        assert h.gather(0)[0].shape[0] - idx.shape[0] == gain[0], q


def view_bytes(h, cam):
    """bytes of one view's bitmap (DESIGN.md section 7): window half-extent ceil(r_max / vs) + 2, clipped to the volume"""
    ww, hh, step = cam["width"] // cam["step"], cam["height"] // cam["step"], cam["step"]
    dep = float(F32(cam["max_range"]))
    fx, fy, cx, cy = (float(F32(cam[k])) for k in ("fx", "fy", "cx", "cy"))
    r2 = max((((i - cx) * dep / fx) ** 2 + ((j - cy) * dep / fy) ** 2 + dep * dep) for i in (0, (ww - 1) * step) for j in (0, (hh - 1) * step))
    half = math.ceil(math.sqrt(r2) / float(F32(VS))) + 2
    e = 2 * half + 1
    return ((min(e, h.N) ** 2 * min(e, h.Nz) + 31) // 32) * 4


def test_chunk_boundaries(monkeypatch):
    h = handle()
    d = syn.scene_room()
    h.integrate_depth(d, np.eye(3), np.zeros(3))
    h.integrate_depth(d, rot_xyz(0.0, 0.5, 0.2), np.array([0.2, 0.0, 0.1]))
    pos, R = views(h, 13, seed=11)
    one = h.view_gain_unknown(pos, R, CAM_S)
    for budget in (1, 3 * view_bytes(h, CAM_S), 3 * view_bytes(h, CAM_S) + 5):
        monkeypatch.setenv("TSLAM_VIEW_SCRATCH", str(budget))
        got = h.view_gain_unknown(pos, R, CAM_S)
        assert np.array_equal(got[0], one[0]) and np.array_equal(got[1], one[1]), budget
    monkeypatch.delenv("TSLAM_VIEW_SCRATCH")
    check_unknown(h, pos, R, CAM_S)


def test_views_next_to_the_volume_boundary():
    h = handle(64, 64)                      # 3.2 m box: 3 m views reach out of the volume in every direction
    d = syn.scene_room()
    for q in range(3):
        R, T = syn.stream_pose(60 * q)
        h.integrate_depth(d, R, T)
    h.frontier_update(0)
    idx, L = h.gather(0)
    free = idx[L <= LO["l_occ"]]
    edge = free[(np.abs(free + 0.5).max(1) >= 29)]
    assert len(edge) > 0
    rng = np.random.default_rng(5)
    pick = edge[rng.choice(len(edge), min(48, len(edge)), replace=False)]
    pos = (pick.astype(F32) * F32(VS)).astype(F32)
    R = np.stack([rot_xyz(0.0, rng.uniform(-3, 3), rng.uniform(-3, 3)) for _ in range(len(pick))]).astype(F32)
    gv, gg = check_unknown(h, pos, R, CAM_S)
    assert gv.all()
    check_frontier(h, pos, R, CAM_S)


def test_two_submaps():
    h = handle(max_submaps=2)
    d = syn.scene_sphere(3.0)
    h.integrate_depth(d, np.eye(3), np.zeros(3), submap=0)
    h.integrate_depth(syn.scene_room(), rot_xyz(0.0, 0.0, 1.0), np.array([0.4, 0.0, 0.0]), submap=1)
    p0, R0 = views(h, 32, seed=1, submap=0)
    p1, R1 = views(h, 32, seed=2, submap=1)
    g0 = check_unknown(h, p0, R0, CAM_S, submap=0)[1]
    g1 = check_unknown(h, p1, R1, CAM_S, submap=1)[1]
    assert not np.array_equal(h.view_gain_unknown(p0, R0, CAM_S, submap=1)[1], g0)
    h.frontier_update(1)
    refused(h.view_gain_frontier, p0, R0, CAM_S, submap=0)
    check_frontier(h, p1, R1, CAM_S, submap=1)
    h.frontier_update(0)
    refused(h.view_gain_frontier, p1, R1, CAM_S, submap=1)
    check_frontier(h, p0, R0, CAM_S, submap=0)
    assert g1.sum() > 0


def test_stale_frontier_set_with_current_classes():
    h = handle()
    d = syn.scene_room()
    h.integrate_depth(d, np.eye(3), np.zeros(3))
    h.frontier_update(0)
    fidx, fcl = h.frontier_gather(0)
    nc = h.frontier_clusters(0).shape[0]
    h.integrate_depth(d, rot_xyz(0.0, 0.3, 0.8), np.array([0.3, 0.1, 0.0]))   # no update after it
    pos, R = views(h, 64, seed=3)
    _, gt, _ = check_frontier(h, pos, R, CAM_S, stale=(fidx, fcl, nc))
    assert gt.max() > 0


def test_no_side_effects():
    a, b = handle(128, 128), handle(128, 128)
    d = syn.scene_room()
    for h in (a, b):
        h.integrate_depth(d, np.eye(3), np.zeros(3))
        h.esdf_update(0, 1.0)
        h.frontier_update(0)
    pos, R = views(a, 32, seed=4)
    a.view_gain_unknown(pos, R, CAM_S)
    a.view_gain_frontier(pos, R, CAM_S)
    a.view_gain_unknown(pos[:2], R[:2], CAM_F)
    for h in (a, b):
        h.integrate_depth(d, rot_xyz(0.0, 0.4, 0.6), np.array([0.2, -0.1, 0.0]))
    assert a.stats() == b.stats()
    ai, aL = as_dict_rows(*a.gather(0))
    bi, bL = as_dict_rows(*b.gather(0))
    assert np.array_equal(ai, bi) and np.array_equal(aL, bL)
    assert a.esdf_update(0, 1.0) == b.esdf_update(0, 1.0)
    ae, be = as_dict_rows(*a.esdf_gather(0)), as_dict_rows(*b.esdf_gather(0))
    assert np.array_equal(ae[0], be[0]) and np.array_equal(ae[1].view(np.int32), be[1].view(np.int32))
    sa, sb = a.frontier_update(0), b.frontier_update(0)
    assert sa == sb and not sa["full"]          # same re-examined block count as the twin
    af, bf = as_dict_rows(*a.frontier_gather(0)), as_dict_rows(*b.frontier_gather(0))
    assert np.array_equal(af[0], bf[0]) and np.array_equal(af[1], bf[1])
    assert np.array_equal(a.frontier_clusters(0), b.frontier_clusters(0))


def test_refusals():
    import torch
    from taichislam_b200 import _capi as capi
    from taichislam_b200.octo_handle import OctoHandle
    L = capi.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    p = torch.zeros((4, 3), dtype=torch.float32, device=dev)
    r = torch.eye(3, device=dev).repeat(4, 1, 1).contiguous()
    u8 = torch.zeros(4, dtype=torch.uint8, device=dev)
    i64 = torch.zeros(4, dtype=torch.int64, device=dev)
    i32 = torch.zeros(64, dtype=torch.int32, device=dev)
    cam = OctoHandle.view_camera(CAM_S)
    P, Rp, V, G, T = (capi.tptr(x) for x in (p, r, u8, i64, i32))

    def unk(h, n=4, c=cam, sub=0, pos=P, rot=Rp, valid=V, gain=G):
        return L.tslam_octo_view_gain_unknown(h.h, sub, n, pos, rot, C.byref(c) if c is not None else None, valid, gain, None)

    def fro(h, n=4, c=cam, nc=None, sub=0, pos=P, rot=Rp, valid=V, tot=T, per=T):
        nc = h.frontier_clusters(sub).shape[0] if nc is None else nc
        return L.tslam_octo_view_gain_frontier(h.h, sub, n, pos, rot, C.byref(c) if c is not None else None, nc, valid, tot, per, None)

    hits = OctoHandle(64, 64, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH)
    assert unk(hits) == capi.E_INVALID
    assert fro(hits, nc=0) == capi.E_INVALID
    h = handle(64, 64, max_submaps=2)
    h.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    assert fro(h, nc=0) == capi.E_INVALID                      # before any frontier update
    h.frontier_update(0)
    assert unk(h) == capi.TSLAM_OK and fro(h) == capi.TSLAM_OK
    nc = h.frontier_clusters(0).shape[0]
    assert nc > 1
    for kw in (dict(n=-1), dict(c=None), dict(pos=None), dict(rot=None), dict(valid=None), dict(sub=2), dict(sub=-1)):
        assert unk(h, **kw) == capi.E_INVALID, kw
        assert fro(h, nc=nc, **kw) == capi.E_INVALID, kw
    assert unk(h, gain=None) == capi.E_INVALID and fro(h, tot=None) == capi.E_INVALID
    assert fro(h, per=None) == capi.TSLAM_OK                   # per-cluster counts are optional
    assert unk(h, n=0, pos=None, rot=None, valid=None, gain=None) == capi.TSLAM_OK   # n == 0: a no-op
    for bad in (dict(fx=0.0), dict(fx=float("nan")), dict(fy=-1.0), dict(max_range=0.0), dict(max_range=float("inf")),
                dict(cx=float("nan")), dict(cy=float("inf")), dict(width=0), dict(height=-1), dict(step=0),
                dict(width=3, step=4), dict(height=1, step=2), dict(fx=1e-30)):
        c = OctoHandle.view_camera(dict(CAM_S, **bad))
        assert unk(h, c=c) == capi.E_INVALID, bad
        assert fro(h, c=c, nc=nc) == capi.E_INVALID, bad
    assert fro(h, nc=nc + 1) == capi.E_INVALID and fro(h, nc=nc - 1) == capi.E_INVALID
    assert fro(h, nc=nc, sub=1) == capi.E_INVALID               # another submap than the last update's
    h.reset()
    assert fro(h, nc=nc) == capi.E_INVALID                     # after a reset until the next update
    h.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    h.frontier_update(0)
    src = handle(64, 64)
    src.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    h.set_submap_pose(0, np.eye(3), np.zeros(3))
    h.fuse_from(src)
    assert fro(h, nc=nc) == capi.E_INVALID                     # after a fusion until the next update
    h.sync()
    # a rotation scaled by 2 sends the rays twice as far as the window allows: reported by the next sync, not dropped
    big = handle(256, 256)
    big.integrate_points(np.array([[0.0, 0.3, 0.35]], np.float32), np.eye(3), np.zeros(3))   # the origin cell FREE
    big.view_gain_unknown(torch.zeros((1, 3), device=dev), 2.0 * torch.eye(3, device=dev)[None], CAM_S)
    refused(big.sync)
    big.sync()
    # the Octomap surface
    from taichislam_b200.mapping.taichi_octomap import Octomap
    o = Octomap(map_scale=[3.2, 3.2], voxel_scale=VS, max_disp_particles=16)
    o.set_dep_camera_intrinsic(syn.K_DEPTH)
    with pytest.raises(ValueError):
        o.view_gain(np.zeros((1, 3)), np.eye(3)[None], 160, 120)
    o = Octomap(map_scale=[3.2, 3.2], voxel_scale=VS, occupancy_model="logodds", max_disp_particles=16)
    with pytest.raises(ValueError):
        o.view_gain(np.zeros((1, 3)), np.eye(3)[None], 160, 120)


def test_octomap_class_flow():
    import torch
    from taichislam_b200.mapping.taichi_octomap import Octomap
    o = Octomap(map_scale=[12.8, 12.8], voxel_scale=VS, occupancy_model="logodds", max_ray_length=3.0, max_disp_particles=1024)
    o.set_dep_camera_intrinsic(syn.K_DEPTH)
    o.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    d = syn.scene_room()
    o.recast_depth_to_map(np.eye(3), np.zeros(3), d, None)
    o.frontier_update()
    o.recast_depth_to_map(rot_xyz(0.0, 0.0, 0.4), np.array([0.1, 0.0, 0.0]), d, None)
    pos, R = views(o._h, 24, seed=9)
    out = o.view_gain(pos, R, 320, 240)           # update=True: frontier_update first, so frontiers and classes agree
    cam = dict(fx=syn.FX, fy=syn.FY, cx=syn.CX, cy=syn.CY, width=320, height=240, step=2, max_range=3.0)
    gv, gg = check_unknown(o._h, pos, R, cam)
    _, gt, gp = check_frontier(o._h, pos, R, cam)
    assert np.array_equal(out["valid"], gv) and np.array_equal(out["unknown"], gg)
    assert np.array_equal(out["frontier"], gt) and np.array_equal(out["frontier_per_cluster"], gp)
    assert gp.shape[1] == o.get_frontier_clusters()["size"].shape[0]
    dev = torch.device("cuda", torch.cuda.current_device())
    tout = o.view_gain(torch.from_numpy(pos).to(dev), torch.from_numpy(R).to(dev), 320, 240, update=False)
    for k in ("valid", "unknown", "frontier", "frontier_per_cluster"):
        assert isinstance(tout[k], torch.Tensor) and tout[k].is_cuda
        assert np.array_equal(tout[k].cpu().numpy(), out[k]), k
    only = o.view_gain(pos, R, 320, 240, step=4, max_range=2.0, frontier=False)
    assert only["frontier"] is None and only["frontier_per_cluster"] is None
    assert np.array_equal(only["unknown"], check_unknown(o._h, pos, R, dict(cam, step=4, max_range=2.0))[1])
