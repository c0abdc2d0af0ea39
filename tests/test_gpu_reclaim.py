"""Reclaim of TSDF pool blocks (tslam_tsdf_reclaim, TsdfHandle.reclaim / block_keys, DenseTSDF.reclaim and
SubmapMapping(reclaim_empty=True)): the pool against the numpy statement (tests/reclaim_reference.py) slot for slot,
kept blocks bit for bit, freed slots reused, the incremental global fusion kept exact and incremental, the mesh and the
ESDF following, slot-order readers unchanged, and the refusals."""
import gc

import numpy as np
import pytest

import loop_world as lw
import reclaim_reference as rr
from fuse_update_reference import same_values
from taichislam_b200 import _capi as capi
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu

K_HALF = [syn.FX / 2, 0, syn.CX / 2, 0, syn.FY / 2, syn.CY / 2, 0, 0, 1]
M = 16
VS = 0.05


@pytest.fixture(autouse=True)
def release_maps():
    gc.collect()
    yield
    gc.collect()


def handle(N, is_global, tex=False, max_blocks=8192, K=None):
    from taichislam_b200.tsdf_handle import TsdfHandle
    h = TsdfHandle(N, N, voxel_scale=VS, K=K or K_HALF, max_ray_length=3.0, is_global_map=is_global, max_submaps=M,
                   max_blocks=max_blocks, texture_enabled=tex)
    if tex:
        h.set_color_intrinsics(K or K_HALF, True)
    return h


def add_sphere(h, s, tex=False, R=None, T=None, radius=None, commit=True):
    d = syn.scene_sphere(radius or (2.0 + 0.1 * (s % 3)), 240, 320)
    t = np.random.default_rng(s).integers(0, 256, (1, 240, 320, 3), dtype=np.uint8) if tex else None
    R = np.eye(3) if R is None else R
    T = np.zeros(3) if T is None else np.asarray(T)
    h.integrate_depth(d, R[None], T[None], submaps=[s], texture=t, commit=commit)


def pose_of(s, jitter=0.0):
    return rot_xyz(0.1 * s + jitter, -0.05 * s, 0.2 * s - jitter), np.array([0.3 * s - 0.5 + jitter, 0.1 * s, -0.2 + 0.05 * s])


def half_sphere(keys):
    """a sphere around the block with the lowest x that reaches about half of the blocks (metres, the map's frame)"""
    c = (np.asarray(keys, np.float64)[:, 1:] * 16 + 7.5) * VS
    centre = c[np.argmin(c[:, 0])]
    return centre.tolist(), float(np.median(np.linalg.norm(c - centre, axis=1)))


def key_tuples(keys):
    return [tuple(int(v) for v in k) for k in keys]


def voxels(h, s, tex=False):
    """gather rows of submap s in key order"""
    return as_dict_rows(*h.gather(s, color=tex))


def block_of_rows(s, idx):
    return [(s,) + tuple(int(v) for v in b) for b in np.floor_divide(idx, 16)]


def empty_flags(h, keys, tex=False):
    """per pool slot: no observed voxel in the block"""
    observed = set()
    for s in sorted(set(int(k[0]) for k in keys)):
        observed |= set(block_of_rows(s, h.gather(s, color=tex)[0]))
    return np.array([k not in observed for k in key_tuples(keys)], bool)


def snapshot(h, tex=False, esdf=False):
    keys = h.block_keys()
    subs = sorted(set(int(k[0]) for k in keys))
    snap = dict(keys=keys, vox={s: voxels(h, s, tex) for s in subs})
    if esdf:
        snap["esdf"] = {s: as_dict_rows(*h.esdf_gather(s)) for s in subs}
    return snap


def restrict(rows, s, kept):
    """the rows of voxels that lie in kept blocks"""
    m = np.array([b in kept for b in block_of_rows(s, rows[0])], bool)
    return tuple(a[m] for a in rows)


def same_tuple(a, b):
    return len(a) == len(b) and all(same_values(x, y) for x, y in zip(a, b))


def same_integration(a, b):
    """gather rows of two maps that integrated the same frames: the same voxels and occupancy, TSDF and weight equal up
    to the order-dependent f32 reductions of the ray march (two runs of the same integration differ there too)"""
    assert np.array_equal(a[0], b[0]), "voxel sets differ"
    assert np.array_equal(a[3], b[3]), "occupancy differs"
    dt = np.abs(a[1].astype(np.float64) - b[1])
    assert np.array_equal(np.isnan(a[1]), np.isnan(b[1])) and np.nanmax(dt, initial=0.0) <= 1e-5, ("tsdf", np.nanmax(dt, initial=0.0))
    assert np.allclose(a[2], b[2], rtol=1e-5, atol=1e-6, equal_nan=True), ("weight", np.nanmax(np.abs(a[2] - b[2]), initial=0.0))
    return True


def check_reclaim(h, kw, tex=False, esdf=False, mask=None):
    """reclaim(**kw) on h against the reference: stats, slot order, kept voxels (and ESDF values) bit for bit"""
    before = snapshot(h, tex, esdf)
    keys = before["keys"]
    empty = empty_flags(h, keys, tex)
    rules = (rr.ALL if kw.get("all_blocks") else 0) | (rr.EMPTY if kw.get("empty") else 0) | (rr.OUTSIDE if "center" in kw else 0)
    keep, order, st_ref = rr.reclaim(keys, empty, rules, mask=mask, center=kw.get("center"), radius=kw.get("radius"), vs=VS)
    st = h.reclaim(**kw)
    assert [st[k] for k in ("blocks_before", "candidates", "dropped", "dropped_nonempty", "moved", "blocks_after")] == st_ref.tolist()
    after = h.block_keys()
    assert np.array_equal(after, keys[order])
    assert after.shape[0] == int(keep.sum())
    kept = set(key_tuples(keys[keep]))
    for s, rows in before["vox"].items():
        assert same_tuple(voxels(h, s, tex), restrict(rows, s, kept)), s
        if esdf:
            assert same_tuple(as_dict_rows(*h.esdf_gather(s)), restrict(before["esdf"][s], s, kept)), s
    return st, keep


def mask_of(ids):
    m = np.zeros(M, bool)
    m[list(ids)] = True
    return m


def collection(tex=False, n=4):
    h = handle(128, False, tex)
    for s in range(n):
        R, T = pose_of(s)
        add_sphere(h, s, tex, R=R, T=T)
    return h


def moved_dst(tex=False):
    """a global map after an incremental update that moved a submap: blocks its old pose covered are empty"""
    src, dst = handle(128, False, tex), handle(256, True, tex)
    poses = {s: pose_of(s) for s in range(4)}
    for s in poses:
        add_sphere(src, s, tex)
    for s, (R, T) in poses.items():
        dst.set_submap_pose(s, R, T)
    dst.fuse_update(src)
    R, T = poses[2]
    dst.set_submap_pose(2, R, T + np.array([0.6, -0.4, 0.3]))
    st = dst.fuse_update(src)
    assert st["reason"] == "incremental" and st["moved"] == 1
    return src, dst


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tex", [False, True])
def test_pool_state_after_each_rule(tex):
    h = collection(tex)
    st, _ = check_reclaim(h, dict(submaps=[1], all_blocks=True), tex, mask=mask_of([1]))
    assert st["moved"] > 0
    c, r = half_sphere(h.block_keys())
    st, _ = check_reclaim(h, dict(center=c, radius=r), tex)
    assert 0 < st["dropped"] < st["blocks_before"] and st["moved"] > 0
    c, r = half_sphere(h.block_keys())
    check_reclaim(h, dict(submaps=[0, 3], center=c, radius=r, all_blocks=False), tex, mask=mask_of([0, 3]))
    src, dst = moved_dst(tex)
    st, _ = check_reclaim(dst, dict(empty=True), tex)
    assert st["dropped"] > 0 and st["dropped_nonempty"] == 0 and st["moved"] > 0
    dst.set_submap_pose(1, *pose_of(1, 0.4))
    assert dst.fuse_update(src)["reason"] == "incremental"                                   # empty blocks again
    c, r = half_sphere(dst.block_keys())
    st, _ = check_reclaim(dst, dict(empty=True, center=c, radius=r), tex)                   # mixed rules
    assert st["dropped"] > 0
    st, _ = check_reclaim(dst, dict(empty=True), tex)                                        # nothing left to drop
    assert st["dropped"] == 0 and st["moved"] == 0


def test_pool_state_with_esdf_allocated():
    h = collection(False, n=3)
    h.esdf_update(1)
    st, _ = check_reclaim(h, dict(submaps=[0], all_blocks=True), esdf=True, mask=mask_of([0]))
    assert st["moved"] > 0
    # the next ESDF update is a full one, and equals a full recompute
    assert h.esdf_update2(1)["raise_sweeps"] == -1


def test_reclaim_between_integrate_and_commit():
    a, b = handle(128, False), handle(128, False)
    for h in (a, b):
        for s in range(3):
            R, T = pose_of(s)
            add_sphere(h, s, R=R, T=T, commit=(s < 2))   # submap 2's sums are still pending
    st = a.reclaim(submaps=[0], all_blocks=True)
    assert st["dropped"] > 0 and st["moved"] > 0
    a.commit()
    b.commit()
    for s in (1, 2):
        assert same_integration(voxels(a, s), voxels(b, s)), s
    assert a.count_active(0) == 0


def test_freed_slots_are_reused_after_dropping_a_submap():
    h = handle(128, False)
    add_sphere(h, 0)
    R, T = pose_of(1)
    add_sphere(h, 1, R=R, T=T)
    keep0 = voxels(h, 0)
    nb = h.block_keys().shape[0]
    st = h.reclaim(submaps=[1], all_blocks=True)
    assert st["dropped"] > 0 and st["blocks_after"] == nb - st["dropped"]
    R2, T2 = pose_of(5)
    add_sphere(h, 1, R=R2, T=T2, radius=2.5)
    fresh = handle(128, False)
    add_sphere(fresh, 1, R=R2, T=T2, radius=2.5)
    assert same_integration(voxels(h, 1), voxels(fresh, 1))
    assert same_tuple(voxels(h, 0), keep0)
    n1 = fresh.block_keys().shape[0]
    assert h.block_keys().shape[0] == st["blocks_after"] + n1    # the new blocks took the slots from blocks_after on


def test_pool_full_then_outside_then_integrate_again():
    R1, T1 = np.eye(3), np.array([0.0, 0.0, 0.0])
    R2, T2 = rot_xyz(0.0, 1.2, 0.0), np.array([0.4, 0.0, 0.3])
    probe = handle(128, False)
    add_sphere(probe, 0, R=R1, T=T1)
    nA = probe.block_keys().shape[0]
    probe.close()
    probe = handle(128, False)
    add_sphere(probe, 1, R=R2, T=T2)
    nB = probe.block_keys().shape[0]
    probe.close()
    cap = nA + nB - 8
    h = handle(128, False, max_blocks=cap)
    add_sphere(h, 0, R=R1, T=T1)
    with pytest.raises(capi.TslamError) as e:
        add_sphere(h, 1, R=R2, T=T2)
        h.sync()
    assert e.value.code == capi.E_POOL_FULL
    h.reclaim(submaps=[1], all_blocks=True)
    # keep about half of submap 0, give the rest back
    before0 = voxels(h, 0)
    keys = h.block_keys()
    c, r = half_sphere(keys)
    st = h.reclaim(submaps=[0], center=c, radius=r)
    assert st["dropped"] >= 8
    kept = set(key_tuples(keys[~rr.outside(keys, c, r, VS)]))
    add_sphere(h, 1, R=R2, T=T2)
    h.sync()                                                       # no pool error: the overflowed keys allocate again
    fresh = handle(128, False)
    add_sphere(fresh, 1, R=R2, T=T2)
    assert same_integration(voxels(h, 1), voxels(fresh, 1))
    assert same_tuple(voxels(h, 0), restrict(before0, 0, kept))


def test_incremental_fusion_with_empty_reclaim_after_every_call():
    rng = np.random.default_rng(11)
    N = 256
    src, dst, ctl = handle(128, False), handle(N, True), handle(N, True)
    poses = {s: pose_of(s) for s in range(M)}
    present = [0, 1, 2, 3, 4]
    for s in present:
        add_sphere(src, s)
    include = np.zeros(M, bool)
    include[present] = True

    def update(step):
        for g in (dst, ctl):
            for s, (R, T) in poses.items():
                g.set_submap_pose(s, R, T)
        st = dst.fuse_update(src, include=include)
        sc = ctl.fuse_update(src, include=include)
        if step != "first":
            assert st["reason"] == "incremental", (step, st)     # no reclaim forced a full update
        assert sc["reason"] == st["reason"]
        rc = dst.reclaim(empty=True)
        assert rc["dropped_nonempty"] == 0
        # the fused map is the control's, bit for bit, and the pool holds exactly the blocks with an observed voxel
        a, b = voxels(dst, 0), voxels(ctl, 0)
        assert same_tuple(a, b), step
        keys = dst.block_keys()
        assert sorted(key_tuples(keys)) == sorted(set(block_of_rows(0, a[0]))), step
        assert ctl.block_keys().shape[0] >= keys.shape[0]
        fresh = handle(N, True)
        for s, (R, T) in poses.items():
            fresh.set_submap_pose(s, R, T)
        fresh.fuse_update(src, include=include)
        assert same_tuple(a, voxels(fresh, 0)), step
        fresh.close()
        return rc

    update("first")
    dropped = 0
    for step in ["move1", "move2", "exclude", "include", "new_submap", "move1", "exclude", "move2"]:
        if step == "move1":
            s = int(rng.choice(np.flatnonzero(include)))
            poses[s] = pose_of(s, float(rng.uniform(0.2, 0.6)))
        elif step == "move2":
            for s in rng.choice(np.flatnonzero(include), 2, replace=False):
                poses[int(s)] = pose_of(int(s), float(rng.uniform(0.2, 0.6)))
        elif step == "exclude":
            include[int(rng.choice(np.flatnonzero(include)))] = False
        elif step == "include":
            include[int(rng.choice([s for s in present if not include[s]]))] = True
        elif step == "new_submap":
            s = len(present)
            add_sphere(src, s)
            present.append(s)
            include[s] = True
        dropped += update(step)["dropped"]
    assert dropped > 0
    assert ctl.block_keys().shape[0] > dst.block_keys().shape[0]


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


def triangle_multiset(mesh):
    ntri = mesh[0]
    t = np.concatenate([a.reshape(ntri, -1) for a in mesh[1:]], 1)
    return t[np.lexsort(t.T[::-1])]


def esdf_rows(h):
    i, e = h.esdf_gather()
    o = np.lexsort(i.T[::-1])
    return i[o], e[o]


def test_mesh_and_esdf_after_reclaim():
    from taichislam_b200.mesh_handle import MeshCache
    _, dst = moved_dst()
    mc = MeshCache(dst)
    cached_mesh(mc)
    dst.esdf_update()
    before = one_shot_mesh(dst)
    st = dst.reclaim(empty=True)
    assert st["moved"] > 0
    after = one_shot_mesh(dst)
    assert before[0] == after[0] > 100
    assert np.array_equal(triangle_multiset(before), triangle_multiset(after))
    assert same_tuple(cached_mesh(mc), after)
    assert mc.updated_blocks()["full"]
    assert dst.esdf_update2()["raise_sweeps"] == -1
    i1, e1 = esdf_rows(dst)
    dst.esdf_update2(full=True)
    i2, e2 = esdf_rows(dst)
    assert np.array_equal(i1, i2) and same_values(e1, e2)
    # an OUTSIDE reclaim that drops observed blocks: the mesh and ESDF still follow
    c, r = half_sphere(dst.block_keys())
    st = dst.reclaim(center=c, radius=r)
    assert st["dropped_nonempty"] > 0
    assert same_tuple(cached_mesh(mc), one_shot_mesh(dst))
    dst.esdf_update()
    i1, e1 = esdf_rows(dst)
    dst.esdf_update2(full=True)
    i2, e2 = esdf_rows(dst)
    assert np.array_equal(i1, i2) and same_values(e1, e2)
    # a reclaim that drops nothing leaves both incremental
    assert dst.reclaim(empty=True)["dropped"] == 0
    cached_mesh(mc)
    assert not mc.updated_blocks()["full"]
    assert dst.esdf_update2()["raise_sweeps"] != -1
    mc.close()


def describe(h, subs, band):
    d = h.place_describe(subs, np.tile(np.eye(3), (len(subs), 1, 1)), 4.0, 0.3, band)
    return [d["sc"].cpu().numpy(), d["ring"].cpu().numpy(), d["bev"].cpu().numpy(), d["n_points"]]


def test_slot_order_readers():
    h = collection(False, n=5)
    band = 0.2
    R0, T0 = np.eye(3)[None], np.zeros(3)[None]
    ref01 = h.register(h, [0], [1], R0, T0, band)
    ref23 = h.register(h, [2], [3], R0, T0, band)
    d0 = describe(h, [1, 2, 3], band)
    # submap 4 was integrated last: its blocks lie at the top of the pool, so dropping it moves nothing
    st = h.reclaim(submaps=[4], all_blocks=True)
    assert st["dropped"] > 0 and st["moved"] == 0
    for a, b in ((h.register(h, [0], [1], R0, T0, band), ref01), (h.register(h, [2], [3], R0, T0, band), ref23)):
        for k in ("R", "T", "H", "b", "cost", "n_points"):
            assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    # dropping submap 0 moves blocks of submaps 2 and 3 into its slots: the same within f64 rounding
    st = h.reclaim(submaps=[0], all_blocks=True)
    assert st["moved"] > 0
    r = h.register(h, [2], [3], R0, T0, band)
    assert np.array_equal(np.asarray(r["n_points"]), np.asarray(ref23["n_points"]))
    for k in ("R", "T", "H"):
        assert np.allclose(np.asarray(r[k]), np.asarray(ref23[k]), rtol=1e-9, atol=1e-12), k
    for a, b in zip(d0, describe(h, [1, 2, 3], band)):
        assert same_values(a, b), "place descriptors changed"


def test_queued_frames_are_integrated_first():
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    maps = []
    for _ in range(2):
        sub = DenseTSDF(map_scale=[6.4, 6.4], max_submap_num=M, max_ray_length=3.0, max_blocks=8192)
        sub.set_dep_camera_intrinsic(np.array(K_HALF, np.float64).reshape(3, 3))
        sub.set_base_pose_submap(0, np.eye(3), np.zeros(3))
        sub.recast_depth_to_map(np.eye(3), np.zeros(3), syn.scene_sphere(2.0, 240, 320), None)   # queued
        maps.append(sub)
    st = maps[0].reclaim(empty=True)
    assert st["blocks_before"] > 0                                   # the queued frame had been integrated
    maps[1]._flush()
    assert same_integration(voxels(maps[0]._h, 0), voxels(maps[1]._h, 0))


def test_refusals_leave_the_map_unchanged():
    import ctypes as C
    import torch
    h = collection(False, n=2)
    keys = h.block_keys()

    def refused(msg):
        with pytest.raises(capi.TslamError) as e:
            h.reclaim(all_blocks=True)
        assert e.value.code == capi.E_INVALID and msg in str(e.value)
        assert np.array_equal(h.block_keys(), keys)

    # tile cuts
    t = (C.c_int32 * 3)(2, 1, 1)
    cx, cy, cz = (C.c_int32 * 3)(-32, 0, 32), (C.c_int32 * 2)(-32, 32), (C.c_int32 * 2)(-32, 32)
    capi.check(h.L.tslam_tiling_set_cuts(h.h, t, cx, cy, cz))
    refused("tiled map")
    capi.check(h.L.tslam_tiling_set_cuts(h.h, None, None, None, None))
    # an open tiled ESDF exchange
    h.esdf_tiled_begin(0)
    refused("tiled ESDF")
    h.esdf_tiled_end()
    # a tiled fusion update in progress
    g = handle(256, True)
    g.fuse_update_tiled_plan(h, (1, 1, 1), 0, 1)
    gkeys = g.block_keys()
    with pytest.raises(capi.TslamError) as e:
        g.reclaim(empty=True)
    assert e.value.code == capi.E_INVALID and "tiled fusion" in str(e.value)
    assert np.array_equal(g.block_keys(), gkeys)
    # ghost blocks
    key = torch.tensor([(5 << 30) | (514 << 20) | (512 << 10) | 512], dtype=torch.int64, device="cuda")
    twp = torch.zeros((1, 4096, 2), dtype=torch.float32, device="cuda")
    obs = torch.zeros((1, 4096), dtype=torch.uint8, device="cuda")
    capi.check(h.L.tslam_tsdf_ghost_unpack(h.h, 1, capi.tptr(key), capi.tptr(twp), capi.tptr(obs), capi.stream_ptr()))
    keys = h.block_keys()
    refused("ghost")


def test_submap_mapping_option_needs_incremental_fusion():
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    with pytest.raises(ValueError):
        SubmapMapping(global_fusion="rebuild", reclaim_empty=True)


def test_submap_mapping_loop_closure_with_reclaim():
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    sub = dict(map_scale=[12.8, 12.8], voxel_scale=VS, max_ray_length=6.0, max_submap_num=16, max_disp_particles=1 << 16)
    glo = dict(map_scale=[25.6, 12.8], voxel_scale=VS, max_ray_length=6.0, max_submap_num=16, max_disp_particles=1 << 16)
    maps = {}
    for rec in (False, True):
        sm = SubmapMapping(DenseTSDF, sub_opts=sub, global_opts=glo, keyframe_step=lw.FRAMES, global_fusion="incremental",
                           reclaim_empty=rec)
        sm.set_dep_camera_intrinsic(syn.K_DEPTH)
        maps[rec] = sm
    ext = (np.eye(3), np.zeros(3))
    fid = 0
    for s in range(lw.N_LOOP):
        for f in range(lw.FRAMES):
            for sm in maps.values():
                sm.recast_depth_to_map_by_frame(fid, True, lw.odometry_pose(s, f), ext, lw.render(s, f), np.array([]))
            fid += 1
    # one more submap (room B): the loop submap is no longer the active one, so it is in the global map
    s = lw.N_LOOP
    for f in range(lw.FRAMES):
        for sm in maps.values():
            sm.recast_depth_to_map_by_frame(fid, True, lw.odometry_pose(s, f), ext, lw.render(s, f), np.array([]))
        fid += 1
    last = lw.FRAMES * (lw.N_LOOP - 1)
    sm, other = maps[True], maps[False]
    out = sm.detect_loops(last, min_gap=2)
    c = out[(last, 0)]
    assert c["accepted"]
    sm.set_frame_poses({last: (c["world_R"], c["world_T"])})              # the loop closure moves the submap by metres
    st = sm.last_fusion_stats
    assert st["moved"] == 1 and not st["full"], st
    res = sm.align_submap(last, reference_frame_id=0, apply=True, band=0.2)  # refined from there (applied when it converges)
    # the flow without the option gets the same pose bits (the two collections were integrated apart, so their own
    # registrations could differ in the last bits)
    other.set_frame_poses({last: (c["world_R"], c["world_T"])})
    if res["status"] == 0:
        other.set_frame_poses({last: (res["world_R"], res["world_T"])})
    rc = maps[True].last_reclaim_stats
    assert rc is not None and rc["dropped"] > 0 and rc["dropped_nonempty"] == 0
    a, b = maps[True].global_map._h, maps[False].global_map._h
    assert same_integration(voxels(a, 0), voxels(b, 0))               # (two collections, integrated apart)
    assert a.block_keys().shape[0] <= b.block_keys().shape[0]
    assert maps[False].last_reclaim_stats is None
