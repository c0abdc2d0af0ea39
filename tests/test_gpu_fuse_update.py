"""Incremental global fusion (tslam_tsdf_fuse_update, TsdfHandle.fuse_update, DenseTSDF.update_fused_submaps and
SubmapMapping(global_fusion="incremental")): bit for bit against the numpy reference of the contract
(tests/fuse_update_reference.py), independent of the history of calls, close to the existing fuse_from, and with the
incremental mesh and ESDF following it."""
import gc

import numpy as np
import pytest

import track_world as tw
from fuse_update_reference import fuse_reference, same_rows, same_values
from taichislam_b200 import _capi as capi
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu

TOL = 1e-4  # test_gpu_tsdf.py::test_submap_fusion
K_HALF = [syn.FX / 2, 0, syn.CX / 2, 0, syn.FY / 2, syn.CY / 2, 0, 0, 1]
M = 16      # submap table of these tests


@pytest.fixture(autouse=True)
def release_maps():
    gc.collect()
    yield
    gc.collect()


def handle(N, is_global, tex=False, max_submaps=M, max_blocks=8192, vs=0.05, K=None):
    from taichislam_b200.tsdf_handle import TsdfHandle
    h = TsdfHandle(N, N, voxel_scale=vs, K=K or K_HALF, max_ray_length=3.0, is_global_map=is_global, max_submaps=max_submaps,
                   max_blocks=max_blocks, texture_enabled=tex)
    if tex:
        h.set_color_intrinsics(K or K_HALF, True)
    return h


def sphere_frame(s, tex):
    d = syn.scene_sphere(2.0 + 0.1 * (s % 3), 240, 320)
    t = None
    if tex:
        rng = np.random.default_rng(s)
        t = rng.integers(0, 256, (1, 240, 320, 3), dtype=np.uint8)
    return d, t


def add_sphere(src, s, tex=False, R=None, T=None):
    d, t = sphere_frame(s, tex)
    R = np.eye(3) if R is None else R
    T = np.zeros(3) if T is None else T
    src.integrate_depth(d, R[None], np.asarray(T)[None], submaps=[s], texture=t)


def pose_of(s, jitter=0.0):
    return rot_xyz(0.1 * s + jitter, -0.05 * s, 0.2 * s - jitter), np.array([0.3 * s - 0.5 + jitter, 0.1 * s, -0.2 + 0.05 * s])


def set_poses(dst, poses):
    for s, (R, T) in poses.items():
        dst.set_submap_pose(s, R, T)


def rows(h, tex=False):
    return as_dict_rows(*h.gather(0, color=tex))


def same(a, b):
    return len(a) == len(b) and all(same_values(x, y) for x, y in zip(a, b))


def reference(src, poses, include, N, tex=False, vs=0.05):
    parts = []
    for s, (R, T) in poses.items():
        if include is not None and not include[s]:
            continue
        g = src.gather(s, color=tex)
        p = dict(idx=g[0], tsdf=g[1], w=g[2], occ=g[3], R=np.float32(R), T=np.float32(T))
        if tex:
            p["color"] = g[4]
        parts.append(p)
    return fuse_reference(parts, N, N, np.float32(vs))


def fresh(src, poses, include, N, tex=False):
    g = handle(N, True, tex)
    set_poses(g, poses)
    st = g.fuse_update(src, include=include)
    assert st["full"] and st["reason"] == "first call"
    out = rows(g, tex)
    g.close()
    return out


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tex", [False, True])
def test_sphere_submaps_match_reference_bit_for_bit(tex):
    src, dst = handle(128, False, tex), handle(256, True, tex)
    poses = {0: (rot_xyz(0.1, 0.2, 0.3), np.array([0.5, 0.1, -0.2])), 1: (rot_xyz(-0.3, 0.1, 1.0), np.array([-0.4, 0.6, 0.3]))}
    for s in poses:
        add_sphere(src, s, tex)
    set_poses(dst, poses)
    st = dst.fuse_update(src)
    assert st["full"] and st["added"] == 2 and st["voxels_skipped"] == 0
    ref = reference(src, poses, None, 256, tex)
    assert st["voxels_splatted"] == ref["splatted"] > 0
    assert same_rows(dst.gather(0, color=tex), ref)


@pytest.mark.parametrize("tex", [False, True])
def test_box_room_submaps_match_reference_bit_for_bit(tex):
    src = handle(256, False, tex, K=syn.K_DEPTH)
    dst = handle(256, True, tex, K=syn.K_DEPTH)
    poses = {}
    for s in range(4):
        for k in range(3):
            R, t = tw.pose(10 * s + 3 * k)
            d = tw.render(R, t, seed=k)
            tex_img = np.random.default_rng(k).integers(0, 256, d.shape + (3,), dtype=np.uint8)[None] if tex else None
            src.integrate_depth(d, R[None], t[None], submaps=[s], texture=tex_img)
        poses[s] = pose_of(s, 0.01)
    set_poses(dst, poses)
    dst.fuse_update(src)
    assert same_rows(dst.gather(0, color=tex), reference(src, poses, None, 256, tex))


def test_history_independence_over_a_seeded_sequence():
    """Pose changes, include changes, new content, new submaps and a remote-style scatter: after every call the map
    equals a fresh handle's single update bit for bit, and the plan rules pick the incremental path where they should."""
    rng = np.random.default_rng(7)
    N = 256
    src, dst = handle(128, False), handle(N, True)
    poses = {s: pose_of(s) for s in range(M)}
    present = [0, 1, 2, 3, 4, 5]
    for s in present:
        add_sphere(src, s)
    include = np.zeros(M, bool)
    include[present] = True
    set_poses(dst, poses)
    assert dst.fuse_update(src, include=include)["reason"] == "first call"
    assert same(rows(dst), fresh(src, poses, include, N))
    steps = ["move1", "move2", "exclude", "include", "new_submap", "content_excluded", "scatter_new", "move1", "content"]
    for step in steps:
        expect = "incremental"
        if step == "move1":
            s = int(rng.choice(np.flatnonzero(include)))
            poses[s] = pose_of(s, float(rng.uniform(0.01, 0.05)))
        elif step == "move2":
            for s in rng.choice(np.flatnonzero(include), 2, replace=False):
                poses[int(s)] = pose_of(int(s), float(rng.uniform(0.01, 0.05)))
        elif step == "exclude":
            include[int(rng.choice(np.flatnonzero(include)))] = False
        elif step == "include":
            include[int(rng.choice([s for s in present if not include[s]]))] = True
        elif step == "new_submap":
            s = len(present)
            add_sphere(src, s)
            present.append(s)
            include[s] = True
        elif step == "content_excluded":
            s = int(rng.choice(np.flatnonzero(include)))
            include[s] = False
            st = dst.fuse_update(src, include=include)
            assert st["reason"] == "incremental" and st["removed"] == 1
            add_sphere(src, s, R=rot_xyz(0.0, 0.1, 0.0), T=np.array([0.05, 0.0, 0.0]))  # not fused now: nothing to subtract
        elif step == "scatter_new":
            s = M - 1  # remote submaps fill the table from the top
            g = src.gather(0)
            src.scatter(s, g[0], g[1], g[2], g[3])
            include[s] = True
            present.append(s)
        elif step == "content":
            s = int(rng.choice(np.flatnonzero(include)))
            add_sphere(src, s, T=np.array([0.0, 0.02, 0.0]))  # its old content is gone: a full update
            expect = "content changed"
        set_poses(dst, poses)
        st = dst.fuse_update(src, include=include)
        assert st["reason"] == expect, (step, st)
        assert same(rows(dst), fresh(src, poses, include, N)), step


def test_same_voxels_as_fuse_from_and_values_within_tol():
    src, g_new, g_old = handle(128, False), handle(256, True), handle(256, True)
    poses = {s: pose_of(s) for s in range(4)}
    for s in poses:
        add_sphere(src, s)
    set_poses(g_new, poses)
    set_poses(g_old, poses)
    g_new.fuse_update(src)
    g_old.fuse_from(src)
    ni, nt, nw, no = rows(g_new)
    oi, ot, ow, oo = rows(g_old)
    assert np.array_equal(ni, oi)
    fin = np.isfinite(ot)
    heavy = fin & (ow >= 1e-3)  # lighter voxels carry the 2^-24 quantisation of each term (see the CPU reference test)
    assert heavy.mean() > 0.9
    assert np.abs(nt[heavy] - ot[heavy]).max() <= TOL
    assert np.all(np.abs(nw[fin] - ow[fin]) <= TOL * np.maximum(1.0, ow[fin]))
    # occ: equal wherever no running sum can saturate, i.e. the sum of |occ| over the voxel's contributions is < 128
    parts = []
    for s, (R, T) in poses.items():
        g = src.gather(s)
        parts.append(dict(idx=g[0], tsdf=g[1], w=g[2], occ=np.abs(g[3].astype(np.int64)), R=np.float32(R), T=np.float32(T)))
    absref = fuse_reference(parts, 256, 256, np.float32(0.05))
    assert np.array_equal(absref["idx"], ni)
    safe = absref["occ"] < 127
    assert safe.mean() > 0.5 and np.array_equal(no[safe], oo[safe])


def test_tolerance_leaves_small_moves_in_place():
    src, dst = handle(128, False), handle(256, True)
    poses = {s: pose_of(s) for s in range(3)}
    for s in poses:
        add_sphere(src, s)
    set_poses(dst, poses)
    dst.fuse_update(src, tolerance=0.01)
    before = rows(dst)
    R, T = poses[1]
    poses[1] = (R, T + np.array([0.004, 0.0, 0.0]))
    set_poses(dst, poses)
    st = dst.fuse_update(src, tolerance=0.01)
    assert st["reason"] == "incremental" and st["within_tolerance"] == 1 and st["moved"] == 0 and st["blocks_committed"] == 0
    assert same(rows(dst), before)
    poses[1] = (R, T + np.array([0.03, 0.0, 0.0]))
    set_poses(dst, poses)
    st = dst.fuse_update(src, tolerance=0.01)
    assert st["moved"] == 1 and st["within_tolerance"] == 0
    assert same(rows(dst), fresh(src, poses, None, 256))
    # a rotation counts with the submap's radius: 0.2 degrees over a ~3 m radius is ~1 cm
    poses[2] = (rot_xyz(0.0, 0.0, np.deg2rad(0.2)) @ poses[2][0], poses[2][1])
    set_poses(dst, poses)
    assert dst.fuse_update(src, tolerance=0.05)["within_tolerance"] == 1
    assert dst.fuse_update(src, tolerance=0.001)["moved"] == 1
    assert same(rows(dst), fresh(src, poses, None, 256))


def test_every_full_update_trigger_gives_the_incremental_bits():
    N = 256
    src, dst = handle(128, False), handle(N, True)
    poses = {s: pose_of(s) for s in range(8)}
    for s in poses:
        add_sphere(src, s)
    set_poses(dst, poses)
    assert dst.fuse_update(src)["reason"] == "first call"
    ref = fresh(src, poses, None, N)
    assert same(rows(dst), ref)
    st = dst.fuse_update(src, full=True)
    assert st["reason"] == "full requested" and same(rows(dst), ref)
    assert dst.fuse_update(src)["reason"] == "incremental"
    src2 = handle(128, False)
    for s in poses:
        add_sphere(src2, s)
    assert dst.fuse_update(src2)["reason"] == "other source" and same(rows(dst), fresh(src2, poses, None, N))
    assert dst.fuse_update(src)["reason"] == "other source" and same(rows(dst), ref)
    # dst written in between: integrate, scatter, reset, fuse_from
    writes = [lambda: dst.integrate_depth(syn.scene_sphere(2.0, 240, 320), np.eye(3)[None], np.zeros((1, 3))),
              lambda: dst.scatter(0, np.zeros((1, 3), np.int32), np.zeros(1, np.float32), np.ones(1, np.float32), np.zeros(1, np.int8)),
              lambda: dst.reset(),
              lambda: dst.fuse_from(src)]
    for wr in writes:
        wr()
        st = dst.fuse_update(src)
        assert st["reason"] == "destination written" and same(rows(dst), ref)
    # new content in a contributing submap
    add_sphere(src, 3, T=np.array([0.0, 0.0, 0.05]))
    st = dst.fuse_update(src)
    assert st["reason"] == "content changed"
    ref = fresh(src, poses, None, N)
    assert same(rows(dst), ref)
    # every submap moves: subtracting and re-adding costs twice a rebuild
    poses = {s: pose_of(s, 0.02) for s in poses}
    set_poses(dst, poses)
    st = dst.fuse_update(src)
    assert st["reason"] == "cheaper than subtract and re-add" and st["added"] == 8
    assert same(rows(dst), fresh(src, poses, None, N))
    # and one submap moving is incremental
    poses[5] = pose_of(5, 0.04)
    set_poses(dst, poses)
    st = dst.fuse_update(src)
    assert st["reason"] == "incremental" and st["moved"] == 1
    assert same(rows(dst), fresh(src, poses, None, N))


def one_shot_mesh(g, thres=0.1, cap=1 << 20):
    r = g.marching_cubes(step=1, thres=thres, cap_tri=cap)
    return (r[0],) + tuple(np.ascontiguousarray(a).view(np.int32) for a in r[1:])


def cached_mesh(c, thres=0.1, cap=1 << 20):
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    v = torch.empty((3 * cap, 3), dtype=torch.float32, device=dev)
    n = torch.empty((3 * cap, 3), dtype=torch.float32, device=dev)
    demand, rc = c.update_into(thres, cap, v, n)
    k = 3 * min(demand, cap)
    return (demand, v[:k].cpu().numpy().view(np.int32), n[:k].cpu().numpy().view(np.int32))


def test_mesh_and_esdf_follow_the_updates():
    from taichislam_b200.mesh_handle import MeshCache
    src, dst = handle(128, False), handle(256, True)
    poses = {s: (np.eye(3), np.array([1.2 * (s % 4) - 1.8, 1.2 * (s // 4) - 0.6, 0.0])) for s in range(8)}
    for s in poses:
        add_sphere(src, s, T=np.array([0.0, 0.0, -1.6]))
    set_poses(dst, poses)
    dst.fuse_update(src)
    mc = MeshCache(dst)
    a = cached_mesh(mc)
    assert a[0] > 100 and same(a, one_shot_mesh(dst))
    dst.esdf_update()
    # one submap of eight moves: the mesh follows it and remeshes only near its old and new footprint
    s = 5
    old = dst.gather(0)[0]
    R, T = poses[s]
    poses[s] = (R, T + np.array([0.0, 0.0, 0.3]))
    set_poses(dst, poses)
    st = dst.fuse_update(src)
    assert st["reason"] == "incremental" and st["moved"] == 1
    b = cached_mesh(mc)
    assert same(b, one_shot_mesh(dst))
    ub = mc.updated_blocks()
    assert not ub["full"]
    listed = ub["blocks"].cpu().numpy()[:, 1:]
    one = handle(256, True)
    set_poses(one, {s: poses[s]})
    one.fuse_update(src, include=np.arange(M) == s)
    new_blocks = {tuple(x) for x in np.floor_divide(one.gather(0)[0], 16)}
    set_poses(one, {s: (R, T)})
    one.fuse_update(src, include=np.arange(M) == s)
    old_blocks = {tuple(x) for x in np.floor_divide(one.gather(0)[0], 16)}
    foot = old_blocks | new_blocks
    near = [min(max(abs(int(a) - int(b)) for a, b in zip(blk, f)) for f in foot) <= 1 for blk in listed]
    assert len(listed) > 0 and all(near)
    assert len(listed) < len({tuple(x) for x in np.floor_divide(old, 16)})
    # ESDF: the incremental update after a fusion update equals a full recompute on the same handle
    dst.esdf_update()
    i1, e1 = dst.esdf_gather()
    dst.esdf_update2(full=True)
    i2, e2 = dst.esdf_gather()
    o1, o2 = np.lexsort(i1.T[::-1]), np.lexsort(i2.T[::-1])
    assert np.array_equal(i1[o1], i2[o2]) and same_values(e1[o1], e2[o2])
    # an update that only adds keeps the ESDF incremental
    add_sphere(src, 9, T=np.array([0.0, 0.0, -1.6]))
    poses[9] = (np.eye(3), np.array([0.0, 1.5, 0.5]))
    set_poses(dst, poses)
    assert dst.fuse_update(src)["added"] == 1
    assert same(cached_mesh(mc), one_shot_mesh(dst))
    st = dst.esdf_update2()
    assert st["raise_sweeps"] != -1
    i1, e1 = dst.esdf_gather()
    dst.esdf_update2(full=True)
    i2, e2 = dst.esdf_gather()
    o1, o2 = np.lexsort(i1.T[::-1]), np.lexsort(i2.T[::-1])
    assert np.array_equal(i1[o1], i2[o2]) and same_values(e1[o1], e2[o2])
    mc.close()


def test_no_side_effects_on_src_and_queued_frames_are_flushed():
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    sub = DenseTSDF(map_scale=[6.4, 6.4], max_submap_num=M, max_ray_length=3.0, max_blocks=8192)
    glob = DenseTSDF(map_scale=[12.8, 12.8], max_submap_num=M, is_global_map=True, max_blocks=8192)
    sub.set_dep_camera_intrinsic(np.array(K_HALF, np.float64).reshape(3, 3))
    sub.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    d = syn.scene_sphere(2.0, 240, 320)
    sub.recast_depth_to_map(np.eye(3), np.zeros(3), d, None)       # queued, not yet integrated
    glob.set_base_pose_submap(0, rot_xyz(0.1, 0.0, 0.2), np.array([0.2, 0.0, 0.0]))
    st = glob.update_fused_submaps(sub)
    assert st["added"] == 1 and st["voxels_splatted"] > 0
    before = as_dict_rows(*sub._h.gather(0))
    glob.set_base_pose_submap(0, rot_xyz(0.1, 0.0, 0.25), np.array([0.2, 0.0, 0.0]))
    st = glob.update_fused_submaps(sub)
    assert st["added"] + st["moved"] == 1  # (the only submap moved: the cost rule picks the rebuild)
    after = as_dict_rows(*sub._h.gather(0))
    assert same(before, after)


def test_pool_exhaustion_is_reported():
    src, dst = handle(128, False), handle(256, True, max_blocks=2)
    add_sphere(src, 0)
    set_poses(dst, {0: (np.eye(3), np.zeros(3))})  # (a zero pose table would fold the submap onto one voxel)
    with pytest.raises(capi.TslamError) as e:
        dst.fuse_update(src)
    assert e.value.code == capi.E_POOL_FULL


def test_submap_table_outside_the_limit_sizes_include_like_the_c_side():
    """max_submaps = 0 gives the C side's 1024-entry table, so include masks take 1024 entries, as on a 1024 pair."""
    include = [True, False, True]
    out = []
    for m in (0, 1024):
        src, dst = handle(128, False, max_submaps=m), handle(256, True, max_submaps=m)
        for s in range(3):
            add_sphere(src, s)
        set_poses(dst, {s: pose_of(s) for s in range(3)})
        out.append((dst.fuse_update(src, include=include), rows(dst)))
        src.close()
        dst.close()
    assert out[0][0] == out[1][0] and out[0][0]["added"] == 2
    assert same(out[0][1], out[1][1]) and out[0][1][0].shape[0] > 0


def test_refusals_that_need_handles():
    import torch
    src, dst = handle(128, False), handle(256, True)
    add_sphere(src, 0)
    for d, msg in ((handle(256, False), "global map"), (handle(256, True, max_submaps=M + 1), "max_submaps"),
                   (handle(256, True, vs=0.04), "voxel size"), (handle(256, True, tex=True), "texture")):
        with pytest.raises(capi.TslamError) as e:
            d.fuse_update(src)
        assert e.value.code == capi.E_INVALID and msg in str(e.value)
    # a dst holding ghost blocks (the tiled multi-GPU global map)
    keys = torch.tensor([(0 << 30) | (512 << 20) | (512 << 10) | 512], dtype=torch.int64, device="cuda")
    twp = torch.zeros((1, 4096, 2), dtype=torch.float32, device="cuda")
    obs = torch.zeros((1, 4096), dtype=torch.uint8, device="cuda")
    capi.check(dst.L.tslam_tsdf_ghost_unpack(dst.h, 1, capi.tptr(keys), capi.tptr(twp), capi.tptr(obs), capi.stream_ptr()))
    with pytest.raises(capi.TslamError) as e:
        dst.fuse_update(src)
    assert e.value.code == capi.E_INVALID and "ghost" in str(e.value)


def test_submap_mapping_incremental_flow():
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    opts = dict(max_submap_num=M, max_blocks=16384, max_ray_length=3.0)
    K = np.array(K_HALF, np.float64).reshape(3, 3)
    maps = {}
    for mode in ("incremental", "rebuild"):
        sm = SubmapMapping(keyframe_step=2, sub_opts=dict(map_scale=[6.4, 6.4], **opts), global_opts=dict(map_scale=[12.8, 12.8], **opts),
                           global_fusion=mode)
        sm.set_dep_camera_intrinsic(K)
        maps[mode] = sm
    d = syn.scene_sphere(2.0, 240, 320)

    def check(sm, rb):
        sc = sm.submap_collection
        act = sc.get_active_submap_id()
        inc = np.arange(M) != act
        g = sm.global_map._h
        g2 = handle(g.N, True, max_blocks=16384)
        for s in range(M):
            g2.set_submap_pose(s, sm.global_map.submaps_base_R_np[s], sm.global_map.submaps_base_T_np[s])
        sc._flush()
        g2.fuse_update(sc._h, include=inc)
        assert same(rows(g), rows(g2))
        g2.close()
        if rb is not None:  # the rebuild mode at the same point: it fused at the switch, when the active submap was empty
            ni, nt, nw, _ = rows(g)
            oi, ot, ow, _ = rows(rb.global_map._h)
            assert np.array_equal(ni, oi)
            heavy = np.isfinite(ot) & (ow >= 1e-3)
            assert np.abs(nt[heavy] - ot[heavy]).max() <= TOL

    for f in range(8):
        R, T = rot_xyz(0.0, 0.05 * f, 0.0), np.array([0.1 * f, 0.0, 0.0])
        for sm in maps.values():
            sm.recast_depth_to_map_by_frame(f, True, (R, T), (np.eye(3), np.zeros(3)), d, None)
        inc = maps["incremental"]
        if f % 2 == 0 and f > 0:  # a submap switch just happened: both modes fused with the active submap empty
            check(inc, maps["rebuild"])
            if f > 2:
                assert not inc.last_fusion_stats["full"], inc.last_fusion_stats
    inc = maps["incremental"]
    fids = sorted(inc.submaps)
    inc.set_frame_poses({fids[1]: (rot_xyz(0.0, 0.1, 0.02), np.array([0.25, 0.01, 0.0]))})
    assert not inc.last_fusion_stats["full"] and inc.last_fusion_stats["moved"] == 1
    check(inc, None)
    res = inc.align_submap(fids[2], apply=True, band=0.2)
    if res["status"] == 0:
        assert not inc.last_fusion_stats["full"]
    check(inc, None)
