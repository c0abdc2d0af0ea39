"""Incremental marching cubes (tslam_mesh_*, MeshCache, MarchingCubeMesher step 1): after every update the mesh is
bit-identical to a fresh tslam_mc_generate2(step=1) of the same map - n_tri, vertices, normals and colours compared as
int32 views, so NaN normals compare too - and it remeshes only what a commit since the last update could change."""
import gc

import numpy as np
import pytest

from taichislam_b200 import synthetic as syn
from util import rot_xyz

pytestmark = pytest.mark.gpu

THRES = 0.1


@pytest.fixture(autouse=True)
def release_maps():
    gc.collect()
    yield
    gc.collect()


def one_shot(g, thres=THRES, cap=1 << 20, color=False):
    r = g.marching_cubes(step=1, thres=thres, cap_tri=cap, color=color)
    return (r[0],) + tuple(np.ascontiguousarray(a).view(np.int32) for a in r[1:])


def cached(c, thres=THRES, cap=1 << 20, color=False):
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    v = torch.empty((3 * cap, 3), dtype=torch.float32, device=dev)
    n = torch.empty((3 * cap, 3), dtype=torch.float32, device=dev)
    col = torch.empty((3 * cap, 3), dtype=torch.float32, device=dev) if color else None
    demand, rc = c.update_into(thres, cap, v, n, col)
    k = 3 * min(demand, cap)
    out = (demand, v[:k].cpu().numpy().view(np.int32), n[:k].cpu().numpy().view(np.int32))
    if color:
        out += (col[:k].cpu().numpy().view(np.int32),)
    return out, rc


def assert_same(a, b):
    assert a[0] == b[0], (a[0], b[0])
    for x, y in zip(a[1:], b[1:]):
        assert x.shape == y.shape and np.array_equal(x, y)


def per_block(g, thres=THRES):
    """{block key tuple: bytes of its triangles} of the full mesh, through a fresh cache (a full rebuild lists every
    block with its range)."""
    from taichislam_b200.mesh_handle import MeshCache
    c = MeshCache(g)
    (n, v, nrm), _ = cached(c, thres)
    ub = c.updated_blocks()
    assert ub["full"]
    c.close()
    out = {}
    for key, f, k in zip(ub["blocks"].cpu().numpy(), ub["first_tri"].cpu().numpy(), ub["n_tri"].cpu().numpy()):
        if k:
            out[tuple(int(x) for x in key)] = v[3 * f:3 * (f + k)].tobytes() + nrm[3 * f:3 * (f + k)].tobytes()
    return out


def listed(c):
    ub = c.updated_blocks()
    return {tuple(int(x) for x in b) for b in ub["blocks"].cpu().numpy()}, ub


def test_stream_512_single_batched_and_moving_surface():
    from taichislam_b200.mesh_handle import MeshCache
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True, max_ray_length=6.0)
    c = MeshCache(g)
    Rs, Ts = syn.stream_poses(40, start=40)
    steps = [("single", q) for q in range(6)] + [("batch", (6, 14)), ("single", 14), ("batch", (15, 31))] + \
            [("single", q) for q in range(31, 36)]
    prev = None
    for i, (kind, q) in enumerate(steps):
        if kind == "single":
            g.integrate_depth(syn.scene_sphere(3.0 if q < 12 else 3.6), Rs[q][None], Ts[q][None])
        else:
            a, b = q
            d = np.stack([syn.scene_sphere(3.0 if k < 12 else 3.6) for k in range(a, b)])
            g.integrate_depth(d, Rs[a:b], Ts[a:b])
        got, rc = cached(c)
        assert rc == 0
        assert_same(got, one_shot(g))
        blocks, stamped, touched, remeshed = c.stats
        if i > 0:
            assert remeshed < blocks and stamped <= touched, c.stats
        lst, ub = listed(c)
        assert ub["full"] == (i == 0)
        cur = per_block(g)
        if prev is not None:
            changed = {k for k in set(prev) | set(cur) if prev.get(k) != cur.get(k)}
            assert changed, "the stream must change the mesh"
            assert changed <= lst, sorted(changed - lst)[:5]
        prev = cur
    assert got[0] > 10000


def test_textured_colours_equal():
    from taichislam_b200.mesh_handle import MeshCache
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True, max_ray_length=5.0, texture_enabled=True)
    g.set_color_intrinsics([1, 0, 0, 0, 1, 0, 0, 0, 1], True)
    c = MeshCache(g)
    Rs, Ts = syn.stream_poses(6, start=10)
    for q in range(6):
        tex = syn.texture_gradient(60 + q)
        g.integrate_depth(syn.scene_sphere(3.0 if q < 3 else 3.3), Rs[q][None], Ts[q][None], texture=tex[None])
        got, rc = cached(c, color=True)
        assert rc == 0 and got[0] > 1000
        assert_same(got, one_shot(g, color=True))
    # the colour mode is part of the cache: without colours it rebuilds, and equals the uncoloured one-shot
    got, _ = cached(c)
    assert listed(c)[1]["full"]
    assert_same(got, one_shot(g))


def test_change_at_a_block_corner_remeshes_the_lower_neighbours():
    """Only voxel (0,0,0) of blocks (bx, by, 3) and voxels above it change; their lower neighbours (bx-1, by-1, 2) are
    not written (their voxels keep their bits), so they can enter the update only through the 27-neighbourhood of the
    stamped blocks - and their mesh does change, because voxel (0,0,0) of the block above is a corner of their cell
    (15,15,15)."""
    from taichislam_b200.mesh_handle import MeshCache
    from taichislam_b200.tsdf_handle import TsdfHandle
    vs = 0.05
    g = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True, max_ray_length=5.0, internal_voxels=0)
    # a plane between voxel z = 47 (block layer 2) and z = 48 (layer 3): every cell of the z = 47 layer holds triangles
    x, y, z = np.meshgrid(np.arange(-40, 40), np.arange(-40, 40), np.arange(40, 56), indexing="ij")
    idx = np.stack([x, y, z], -1).reshape(-1, 3).astype(np.int32)
    t = ((idx[:, 2] - 47.5) * vs).astype(np.float32)
    g.scatter(0, idx, t, np.ones(len(idx), np.float32), np.zeros(len(idx), np.int8))
    c = MeshCache(g)
    cached(c)
    before = per_block(g)

    def layer(lo, hi):  # observed voxels with lo <= z < hi, sorted by index (gather's row order is unspecified)
        gi, gt, gw, _ = g.gather()
        sel = (gi[:, 2] >= lo) & (gi[:, 2] < hi)
        gi, gt, gw = gi[sel], gt[sel], gw[sel]
        o = np.lexsort((gi[:, 2], gi[:, 1], gi[:, 0]))
        return gi[o], gt[o].view(np.int32), gw[o].view(np.int32)

    layer2 = layer(32, 48)
    top = layer(48, 49)
    # one vertical ray per target, from 1.02 m above voxel (16 bx, 16 by, 48): samples j = 1 .. (int)(L / vs + 0) = 20
    # (dense_tsdf.py:249-253), the last one 1.0 m below the sensor, 0.4 voxel above the target's centre, so the ray writes
    # voxels z >= 48 only
    targets = [(bx, by, 3) for bx in (-1, 0, 1) for by in (-1, 0, 1)]
    down = np.diag([1.0, -1.0, -1.0]).astype(np.float32)
    for bx, by, bz in targets:
        g.integrate_points(np.array([[0.0, 0.0, 1.02]], np.float32), down, np.array([16 * bx * vs, 16 * by * vs, 48 * vs + 1.02], np.float32))
    assert all(np.array_equal(x, y) for x, y in zip(layer(32, 48), layer2))   # layer 2 not written: not stamped
    top2 = layer(48, 49)
    assert np.array_equal(top2[0], top[0])
    corner = (top[0][:, 0] % 16 == 0) & (top[0][:, 1] % 16 == 0) & (np.abs(top[0][:, 0]) <= 16) & (np.abs(top[0][:, 1]) <= 16)
    assert corner.sum() == 9 and (top2[1][corner] != top[1][corner]).all()         # every target voxel was written
    got, rc = cached(c)
    assert rc == 0
    assert_same(got, one_shot(g))
    lst, ub = listed(c)
    assert not ub["full"]
    after = per_block(g)
    below = {(0, bx - 1, by - 1, bz - 1) for bx, by, bz in targets}
    assert below <= lst, sorted(below - lst)
    assert all(before.get(b) != after.get(b) for b in below), "the corner change must reach the lower neighbours' mesh"


def test_every_epoch_path_rebuilds_fully():
    from taichislam_b200.mesh_handle import MeshCache
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True, max_ray_length=5.0)
    c = MeshCache(g)
    g.integrate_depth(syn.scene_room(seed=5), rot_xyz(0.0, 0.4, 0.0)[None], np.zeros((1, 3)))
    cached(c)
    # reset, then a smaller scene: recycled pool slots
    g.reset()
    g.integrate_depth(syn.scene_plane(2.5), np.eye(3)[None], np.zeros((1, 3)))
    got, _ = cached(c)
    assert listed(c)[1]["full"]
    assert_same(got, one_shot(g))
    # load_numpy (scatter) of a different state
    idx, t, w, occ = g.gather()
    t = t.copy()
    t[::7] = -np.abs(t[::7])
    g.scatter(0, idx, t, w, occ)
    got, _ = cached(c)
    assert listed(c)[1]["full"]
    assert_same(got, one_shot(g))
    # fuse_submaps
    s = TsdfHandle(128, 128, K=syn.K_DEPTH, is_global_map=False, max_ray_length=3.0, max_submaps=4)
    for k in range(2):
        R, T = rot_xyz(0.0, 0.0, 0.3 * k), np.array([0.4 * k, 0.0, 0.0], np.float32)
        g.set_submap_pose(k, R, T)
        s.set_submap_pose(k, np.eye(3), np.zeros(3))
        s.integrate_depth(syn.scene_sphere(2.0), np.eye(3)[None], np.zeros((1, 3)), submaps=[k])
    g.fuse_from(s)
    got, _ = cached(c)
    assert listed(c)[1]["full"]
    assert_same(got, one_shot(g))
    assert got[0] > 1000
    # ... and the next plain integrate is incremental again
    g.integrate_depth(syn.scene_plane(2.2), np.eye(3)[None], np.zeros((1, 3)))
    got, _ = cached(c)
    assert not listed(c)[1]["full"]
    assert_same(got, one_shot(g))


def test_nothing_changed_remeshes_nothing():
    from taichislam_b200.mesh_handle import MeshCache
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True, max_ray_length=5.0)
    g.integrate_depth(syn.scene_room(), np.eye(3)[None], np.zeros((1, 3)))
    c = MeshCache(g)
    a, _ = cached(c)
    b, _ = cached(c)
    assert c.stats[1] == c.stats[2] == c.stats[3] == 0 and c.stats[0] > 0
    assert_same(a, b)
    lst, ub = listed(c)
    assert not lst and not ub["full"]
    assert_same(b, one_shot(g))


def test_local_group_second_mesh_remeshes_only_around_ghosts():
    from taichi_slam.mapping import DenseTSDF, MarchingCubeMesher
    from taichislam_b200.distributed import LocalGroup, TiledGlobalMap, run_local_fusion, run_local_mesh, submap_owner
    world = 4
    d = syn.scene_sphere(2.5, 240, 320)
    K = [syn.FX / 2, 0, syn.CX / 2, 0, syn.FY / 2, syn.CY / 2, 0, 0, 1]
    poses = {s: (rot_xyz(0.05 * s, 0.03 * s, 0.7 * s + 0.1), np.array([2.2 * (s % 3) - 2.0, 2.0 * (s // 3) - 1.5, 0.1 * (s % 2)])) for s in range(6)}
    grp = LocalGroup(world)
    subs, glos, tiled = [], [], []
    for r in range(world):
        sub = DenseTSDF(map_scale=[6.4, 6.4], voxel_scale=0.05, max_ray_length=3.0, max_submap_num=8, max_disp_particles=1024,
                        max_image_pixels=240 * 320)
        sub.set_dep_camera_intrinsic(K)
        glo = DenseTSDF(map_scale=[12.8, 12.8], voxel_scale=0.05, is_global_map=True, max_submap_num=8, max_disp_particles=1024)
        for s, (R, T) in poses.items():
            glo.set_base_pose_submap(s, R, T)
            if submap_owner(s, world) != r:
                continue
            sub.active_submap_id[None] = s
            sub.set_base_pose_submap(s, np.eye(3), np.zeros(3))
            sub.recast_depth_to_map(np.eye(3), np.zeros(3), d, np.array([]))
        subs.append(sub); glos.append(glo)
        tiled.append(TiledGlobalMap(glo, grp, r, world))
    run_local_fusion(tiled, subs)
    meshers = [MarchingCubeMesher(g_, 400000, tsdf_surface_thres=0.25) for g_ in glos]
    run_local_mesh(tiled, meshers)
    assert all(m_.updated_blocks()["full"] for m_ in meshers)
    mv, mn, counts = run_local_mesh(tiled, meshers)   # halo re-exchanged, no new fusion
    off = 0
    for r, (t, glo, m_) in enumerate(zip(tiled, glos, meshers)):
        ref = one_shot(glo._h, thres=0.25, cap=400000)
        k = counts[r]
        assert k == ref[0]
        assert np.array_equal(mv[3 * off:3 * (off + k)].cpu().numpy().view(np.int32), ref[1])
        assert np.array_equal(mn[3 * off:3 * (off + k)].cpu().numpy().view(np.int32), ref[2])
        off += k
        ub = m_.updated_blocks()
        assert not ub["full"]
        for s, bx, by, bz in ub["blocks"].cpu().numpy():
            near_ghost = any(t.owner_of_block(bx + dx, by + dy, bz + dz) != r
                             for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1))
            assert near_ghost, (r, bx, by, bz)
    assert sum(counts) > 1000


def test_settings_and_capacity():
    from taichislam_b200.mesh_handle import MeshCache
    from taichislam_b200 import _capi as capi
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True, max_ray_length=5.0)
    g.integrate_depth(syn.scene_room(), np.eye(3)[None], np.zeros((1, 3)))
    c = MeshCache(g)
    cached(c)
    got, _ = cached(c, thres=0.2)
    assert listed(c)[1]["full"]
    assert_same(got, one_shot(g, thres=0.2))
    # capacity below the demand: the same saturated prefix, demand and error code; then the full mesh again
    n = got[0]
    g.integrate_depth(syn.scene_room(seed=4), rot_xyz(0.0, 0.2, 0.0)[None], np.zeros((1, 3)))
    small, rc = cached(c, thres=0.2, cap=n // 3)
    assert rc == capi.E_CAPACITY
    ref = g.marching_cubes(step=1, thres=0.2, cap_tri=n // 3)
    assert small[0] == ref[0] and np.array_equal(small[1], ref[1].view(np.int32)) and np.array_equal(small[2], ref[2].view(np.int32))
    big, rc = cached(c, thres=0.2)
    assert rc == 0
    assert_same(big, one_shot(g, thres=0.2))


def _dense(tex=False):
    from taichislam_b200.mapping import DenseTSDF
    m = DenseTSDF(map_scale=[12.8, 12.8], is_global_map=True, max_ray_length=5.0, texture_enabled=tex)
    m.set_dep_camera_intrinsic(np.array(syn.K_DEPTH).reshape(3, 3))
    m.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    return m


def _mesher_equals_one_shot(mesher, m):
    n = int(mesher.num_facelets[None])
    ref = one_shot(m._h, thres=mesher.tsdf_surface_thres, cap=mesher.max_triangles, color=mesher.enable_texture)
    assert n == ref[0]
    k = 3 * min(n, mesher.max_triangles)
    assert np.array_equal(mesher.mesh_vertices.t[:k].cpu().numpy().view(np.int32), ref[1])
    assert np.array_equal(mesher.mesh_normals.t[:k].cpu().numpy().view(np.int32), ref[2])
    if mesher.enable_texture:
        assert np.array_equal(mesher.mesh_colors.t[:k].cpu().numpy().view(np.int32), ref[3])
    assert int(mesher.num_vertices[None]) == k


def test_mesher_step_2_then_1_and_dense_tsdf_flow():
    from taichislam_b200.mapping import MarchingCubeMesher
    m = _dense()
    mesher = MarchingCubeMesher(m, max_triangles=400000, tsdf_surface_thres=0.1)
    Rs, Ts = syn.stream_poses(8, start=5)
    for q in range(8):  # the DenseTSDF frame queue, meshed after every frame
        m.recast_depth_to_map(Rs[q], Ts[q], syn.scene_sphere(3.0 if q < 4 else 3.6), np.array([]))
        mesher.generate_mesh(1)
        _mesher_equals_one_shot(mesher, m)
        if q:
            ub = mesher.updated_blocks()
            assert not ub["full"] and int(ub["blocks"].shape[0]) < mesher._cache.stats[0]
    assert int(mesher.num_facelets[None]) > 10000
    mesher.generate_mesh(2)
    assert mesher._cache is None
    ref2 = m._h.marching_cubes(step=2, thres=0.1, cap_tri=400000)
    assert int(mesher.num_facelets[None]) == ref2[0]
    mesher.generate_mesh(1)
    assert mesher.updated_blocks()["full"]
    _mesher_equals_one_shot(mesher, m)


def test_mesher_textured_dense_tsdf():
    from taichislam_b200.mapping import MarchingCubeMesher
    m = _dense(tex=True)
    mesher = MarchingCubeMesher(m, max_triangles=400000, tsdf_surface_thres=0.1)
    Rs, Ts = syn.stream_poses(4, start=5)
    for q in range(4):
        m.recast_depth_to_map(Rs[q], Ts[q], syn.scene_sphere(3.0), syn.texture_gradient(70 + q))
        mesher.generate_mesh(1)
        _mesher_equals_one_shot(mesher, m)
    assert int(mesher.num_facelets[None]) > 10000
