"""Log-odds Octomap on the GPU against the numpy reference (octo_logodds_reference.py): every (ijk, L) pair and every
counter of tslam_octo_get_stats bit-exact."""
import numpy as np
import pytest

import octo_logodds_reference as ref
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu

VS = 0.05
LO = ref.params()


def handle(N=256, Nz=256, **kw):
    from taichislam_b200.octo_handle import OctoHandle
    kw.setdefault("Kcam", syn.K_DEPTH)
    return OctoHandle(N, Nz, K=2, voxel_scale=VS, logodds=LO, **kw)


def refmap(N=256, Nz=256, min_ray_length=0.3, max_ray_length=3.0, recast_step=2, K=syn.K_DEPTH):
    return ref.LogoddsMap(N, Nz, VS, min_ray_length=min_ray_length, max_ray_length=max_ray_length, recast_step=recast_step, K=K)


def assert_state(h, m, submap=0):
    gi, gl = as_dict_rows(*h.gather(submap))
    ri, rl = m.gather(submap)
    ri, rl = as_dict_rows(ri, rl)
    assert gi.shape == ri.shape, f"known voxels: gpu {gi.shape[0]} reference {ri.shape[0]}"
    assert np.array_equal(gi, ri) and np.array_equal(gl, rl)
    return gi.shape[0]


def assert_stats(h, m):
    st = h.stats(clear=True)
    assert [st["rays"], st["miss_visits"], st["hit_voxels"], st["updated_voxels"]] == m.stats.tolist()
    m.stats[:] = 0


SCENES = {"S1": lambda: syn.scene_plane(3.0), "S2": lambda: syn.scene_sphere(4.0), "S4": lambda: syn.scene_noise(4),
          "room": lambda: syn.scene_room()}


@pytest.mark.parametrize("scene", list(SCENES))
def test_depth_stream_bit_exact(scene):
    h = handle(max_ray_length=5.0)
    m = refmap(max_ray_length=5.0)
    d = SCENES[scene]()
    Rs, Ts = syn.stream_poses(3, start=40)
    poses = [(Rs[q], Ts[q]) for q in range(3)] + [(rot_xyz(0.3, -0.2, 0.5), np.array([0.1, -0.2, 0.05]))]
    for R, T in poses:
        h.integrate_depth(d, R, T)
        m.integrate_depth(d, R, T)
        assert assert_state(h, m) > 1000
        assert_stats(h, m)


def test_rays_leave_the_volume():
    # a 64^3 map (+-1.6 m) and rays up to 5 m: most paths run out of the volume and the walk goes on through
    h = handle(64, 64, max_ray_length=5.0)
    m = refmap(64, 64, max_ray_length=5.0)
    d = syn.scene_room()
    for R, T in [(rot_xyz(0.1, 0.2, -0.3), np.array([0.4, -1.2, 0.3])), (rot_xyz(0.0, 1.2, 0.0), np.array([-1.7, 0.0, 0.0]))]:
        h.integrate_depth(d, R, T)
        m.integrate_depth(d, R, T)
        assert_state(h, m)
        assert_stats(h, m)


def test_octomap_class_two_submaps():
    from taichislam_b200.mapping.taichi_octomap import Octomap
    o = Octomap(map_scale=[12.8, 12.8], voxel_scale=VS, occupancy_model="logodds", max_ray_length=4.0, max_submap_num=4,
                max_disp_particles=1 << 20)
    assert (o.l_hit, o.l_miss, o.l_min, o.l_max, o.l_occ) == (868, -415, -2048, 3595, 0)
    o.set_dep_camera_intrinsic(syn.K_DEPTH)
    m = refmap(o.N, o.Nz, max_ray_length=4.0)
    bases = [(rot_xyz(0.0, 0.0, 0.4), np.array([0.5, 0.2, 0.0])), (rot_xyz(0.1, 0.0, -0.3), np.array([-1.0, 0.4, 0.2]))]
    d = syn.scene_sphere(3.5)
    for s, (Rb, Tb) in enumerate(bases):
        if s:
            o.switch_to_next_submap()
        o.set_base_pose_submap(s, Rb, Tb)
        for q in range(2):
            R, T = syn.stream_pose(10 * s + q)
            o.recast_depth_to_map(R, T, d, None)
            m.integrate_depth(d, o.input_R_np, o.input_T_np, submap=s)
    for s in range(2):
        assert_state(o._h, m, s)
    idx, p = o.occupy
    ri, rl = m.gather(1)
    assert idx.shape[0] == ri.shape[0] and p.dtype == np.float32
    assert np.array_equal(np.sort(p), np.sort((rl / 1024.0).astype(np.float32)))


def test_hand_checked_point_rays():
    h = handle(min_ray_length=0.0)
    m = refmap(min_ray_length=0.0)
    ends = np.array([[3, 3, 0], [5, 0, 0], [0, -4, 0], [-2, -5, 3], [2, 2, 2], [0, 0, 0]], np.float32) * np.float32(VS)
    for e in ends:   # one ray per frame: the frame's known cells are exactly its path
        h.integrate_points(e[None], np.eye(3), np.zeros(3))
        m.integrate_points(e[None], np.eye(3), np.zeros(3))
        assert_state(h, m)
        assert_stats(h, m)
    diag = {(0, 0, 0), (1, 0, 0), (1, 1, 0), (2, 1, 0), (2, 2, 0), (3, 2, 0), (3, 3, 0)}
    h2 = handle(min_ray_length=0.0)
    h2.integrate_points(ends[:1], np.eye(3), np.zeros(3))
    idx, L = h2.gather()
    got = {tuple(int(v) for v in c): int(x) for c, x in zip(idx, L)}
    assert set(got) == diag and got[(3, 3, 0)] == 868 and all(got[c] == -415 for c in diag - {(3, 3, 0)})
    # many rays at once, random origin and rotation, some cut at max_ray_length
    rng = np.random.default_rng(3)
    pts = rng.uniform(-4, 4, (20000, 3)).astype(np.float32)
    R, T = rot_xyz(0.4, -0.1, 0.9), np.array([0.31, -0.17, 0.05])
    h.integrate_points(pts, R, T)
    m.integrate_points(pts, R, T)
    assert_state(h, m)
    assert_stats(h, m)


def test_dynamic_clearing_points_and_planes():
    from taichislam_b200.mapping.taichi_octomap import Octomap
    o = Octomap(map_scale=[12.8, 12.8], voxel_scale=VS, occupancy_model="logodds", min_ray_length=0.0, max_ray_length=5.0,
                max_disp_particles=1024)
    o.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    m = refmap(o.N, o.Nz, min_ray_length=0.0, max_ray_length=5.0)
    cell = np.array([[40 * VS, 0.0, 0.0]], np.float32)
    for f in range(5):
        o.recast_pcl_to_map(np.eye(3), np.zeros(3), np.array([[2.0, 0, 0]], np.float32), None)
        m.integrate_points(np.array([[2.0, 0, 0]], np.float32), np.eye(3), np.zeros(3))
    for f in range(1, 11):
        o.recast_pcl_to_map(np.eye(3), np.zeros(3), np.array([[4.0, 0, 0]], np.float32), None)
        m.integrate_points(np.array([[4.0, 0, 0]], np.float32), np.eye(3), np.zeros(3))
        assert o.is_pos_occupy(cell[0]) is (f <= 8), f
        assert o.is_pos_unobserved(cell[0]) is False
        assert_state(o._h, m)
    # a plane at 2 m, then at 4 m: the near wall is carved away
    h = handle(max_ray_length=5.0)
    mp = refmap(max_ray_length=5.0)
    for z in [2.0] * 4 + [4.0] * 10:
        d = syn.scene_plane(z)
        h.integrate_depth(d, np.eye(3), np.zeros(3))
        mp.integrate_depth(d, np.eye(3), np.zeros(3))
        assert_state(h, mp)
        assert_stats(h, mp)
    occ, unk = h.query_points(np.array([[0.0, 0.0, 2.0], [0.0, 0.0, 4.0], [0.0, 0.0, 4.5]], np.float32))
    assert occ.tolist() == [False, True, False] and unk.tolist() == [False, False, True]


def room_map():
    h = handle(max_ray_length=5.0, max_submaps=2)
    m = refmap(max_ray_length=5.0)
    d = syn.scene_room()
    for R, T in [(np.eye(3), np.zeros(3)), (rot_xyz(0.0, 0.0, 0.7), np.array([0.2, 0.1, 0.0]))]:
        h.integrate_depth(d, R, T)
        m.integrate_depth(d, R, T)
    return h, m


def test_queries_match_reference():
    from taichislam_b200.mapping.taichi_octomap import Octomap
    h, m = room_map()
    rng = np.random.default_rng(7)
    pts = rng.uniform(-5.5, 5.5, (20000, 3)).astype(np.float32)
    occ, unk = h.query_points(pts)
    rocc, runk = m.query_points(pts)
    assert np.array_equal(occ, rocc) and np.array_equal(unk, runk) and occ.any() and unk.any() and (~unk & ~occ).any()
    few = pts[:1500]
    for voxel in (0, 1, 3, 8):
        assert np.array_equal(h.query_near(few, voxel), m.query_near(few, voxel)), voxel
    dirs = rng.normal(size=(4000, 3)).astype(np.float32)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    start = np.tile(np.array([[0.1, 0.0, 0.3]], np.float32), (4000, 1))
    gh, gx, gl = h.raycast(start, dirs, 4.0)
    rh, rx, rl = m.raycast(start, dirs, 4.0)
    assert np.array_equal(gh, rh) and np.array_equal(gx, rx) and np.array_equal(gl, rl) and gh.mean() > 0.03
    # the class surface answers the same
    o = Octomap(map_scale=[12.8, 12.8], voxel_scale=VS, occupancy_model="logodds", max_ray_length=5.0, max_disp_particles=1024)
    o.set_dep_camera_intrinsic(syn.K_DEPTH)
    o.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    o.recast_depth_to_map(np.eye(3), np.zeros(3), syn.scene_room(), None)
    o.recast_depth_to_map(rot_xyz(0.0, 0.0, 0.7), np.array([0.2, 0.1, 0.0]), syn.scene_room(), None)
    assert np.array_equal(o.is_pos_occupy(pts), rocc) and np.array_equal(o.is_pos_unobserved(pts), runk)
    assert np.array_equal(o.is_near_pos_occupy(few, 3), m.query_near(few, 3))


def test_hits_mode_near_occupy_matches_oracle_counts():
    from oracle.oracle import OracleOctomap
    from taichislam_b200.octo_handle import OctoHandle
    oo = OracleOctomap(map_scale=[12.8, 12.8], voxel_scale=VS, K=2, min_occupy_thres=1, max_ray_length=6.0, Kcam=syn.K_DEPTH)
    g = OctoHandle(oo.N, oo.Nz, K=2, voxel_scale=VS, min_occupy_thres=1, max_ray_length=6.0, Kcam=syn.K_DEPTH)
    d = syn.scene_room()
    g.integrate_depth(d, np.eye(3), np.zeros(3))
    oo.integrate_depth(np.eye(3), np.zeros(3), d)
    idx, cnt = oo.gather()
    occ = {tuple(c) for c, n in zip(idx.tolist(), cnt.tolist()) if float(n) > 1.0}
    pts = np.random.default_rng(2).uniform(-5, 5, (600, 3)).astype(np.float32)
    c0 = ref.cells(pts, VS)
    for voxel in (1, 3, 8):
        r = range(-voxel, voxel)
        want = [any((c[0] + a, c[1] + b, c[2] + e) in occ for a in r for b in r for e in r) for c in c0.tolist()]
        assert g.query_near(pts, voxel).tolist() == want


def test_lod_export_and_gather():
    import torch
    h, m = room_map()
    Rs, Ts = rot_xyz(0.05, 0.1, -0.2), np.array([0.4, -0.3, 0.2])
    h.set_submap_pose(0, Rs, Ts)
    for level in (1, 2, 4):
        n, xyz = h.export(level)
        want = m.export(level, R=Rs, T=Ts)
        assert n == want.shape[0] > 0, level
        assert np.array_equal(xyz[np.lexsort(xyz.T[::-1])], want[np.lexsort(want.T[::-1])])
    idx, L = h.gather_logodds_device()
    assert idx.dtype == torch.int32 and L.dtype == torch.int32
    assert_state(h, m)


def test_texture_only_on_hit_cells():
    from taichislam_b200.octo_handle import OctoHandle
    hits = OctoHandle(256, 256, K=2, voxel_scale=VS, min_occupy_thres=0, max_ray_length=5.0, Kcam=syn.K_DEPTH, texture_enabled=True)
    lo = handle(max_ray_length=5.0, texture_enabled=True)
    m = refmap(max_ray_length=5.0)
    for h in (hits, lo):
        h.set_color_intrinsics(syn.K_DEPTH, color_same_proj=True)
    d = syn.scene_room()
    for q, (R, T) in enumerate([(np.eye(3), np.zeros(3)), (rot_xyz(0.0, 0.0, 0.3), np.array([0.1, 0.0, 0.0]))]):
        tex = syn.texture_gradient(q)
        hits.integrate_depth(d, R, T, texture=tex)
        lo.integrate_depth(d, R, T, texture=tex)
        m.integrate_depth(d, R, T)
    assert_state(lo, m)
    hi, hc, hcol = hits.gather(color=True)
    li, lL, lcol = lo.gather(color=True)
    hk, lk = ref.pack(hi), ref.pack(li)
    pos = np.searchsorted(lk, hk, sorter=np.argsort(lk))
    order = np.argsort(lk)[pos]
    assert np.array_equal(lk[order], hk)                                   # every hit cell is known
    assert np.array_equal(lcol[order], hcol)                               # with the hits-mode colour
    rest = np.setdiff1d(np.arange(len(lk)), order)
    assert (lcol[rest] == 0).all() and len(rest) > 0                       # misses never touch colour


def test_submap_mapping_logodds_fusion():
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    from taichislam_b200.mapping.taichi_octomap import Octomap
    from taichislam_b200.octo_handle import OctoHandle
    sm = SubmapMapping(Octomap, keyframe_step=2,
                       sub_opts=dict(occupancy_model="logodds", map_scale=[12.8, 12.8], max_ray_length=4.0, max_submap_num=8),
                       global_opts=dict(occupancy_model="logodds", map_scale=[25.6, 25.6], max_ray_length=4.0, max_submap_num=8))
    sm.set_dep_camera_intrinsic(syn.K_DEPTH)
    sub = sm.submap_collection
    m = refmap(sub.N, sub.Nz, max_ray_length=4.0)
    d = syn.scene_sphere(3.0)
    for f in range(6):
        R, T = syn.stream_pose(30 * f, radius=1.0)
        sm.recast_depth_to_map_by_frame(f, True, (R, T), (np.eye(3), np.zeros(3)), d, None)
        m.integrate_depth(d, sub.input_R_np, sub.input_T_np, submap=sub.active_submap_id[None])
    sm.local_to_global()
    g = sm.global_map
    gm = refmap(g.N, g.Nz)
    ns = sub.active_submap_id[None] + 1
    assert ns == 3
    ref.fuse(gm, m, {s: (g.submaps_base_R_np[s], g.submaps_base_T_np[s]) for s in range(ns)})
    assert assert_state(g._h, gm) > 1000
    hits = OctoHandle(64, 64, K=2, voxel_scale=VS)
    from taichislam_b200 import _capi as capi
    with pytest.raises(capi.TslamError) as e:
        g._h.fuse_from(hits)
    assert e.value.code == capi.E_INVALID


class RefBackedMap:
    """BaseMap answering from the reference state (the OracleBackedMap pattern of test_topo_cpu.py)."""

    def __new__(cls, m):
        from taichislam_b200.mapping.mapping_common import BaseMap

        class _M(BaseMap):
            def _query_raycast(self, pos, dir, max_dist):
                return m.raycast(pos, dir, max_dist)

            def _query_points(self, xyz):
                return m.query_points(xyz)

            def _query_near(self, xyz, voxel):
                return m.query_near(xyz, voxel)
        return _M(VS)


def test_topo_graph_on_logodds_octomap():
    from scipy.ndimage import binary_dilation
    from taichislam_b200.mapping.taichi_octomap import Octomap
    from taichislam_b200.mapping.topo_graph import TopoGraphGen
    from topo_world import START_A, two_rooms
    idx, tsdf, _, _ = two_rooms()
    lo = idx.min(0)
    grid = np.zeros(idx.max(0) - lo + 1, bool)
    free = np.zeros_like(grid)
    free[tuple((idx - lo)[tsdf > 0].T)] = True
    grid[tuple((idx - lo)[tsdf <= 0].T)] = True
    shell = grid & binary_dilation(free)             # wall cells next to free space
    pts = ((np.argwhere(shell) + lo).astype(np.float32) * np.float32(VS))
    o = Octomap(map_scale=[12.8, 12.8], voxel_scale=VS, occupancy_model="logodds", min_ray_length=0.0, max_ray_length=3.0,
                max_disp_particles=1024)
    o.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    m = refmap(o.N, o.Nz, min_ray_length=0.0, max_ray_length=3.0)
    for off in ([0, 0, 0], [0.6, 0.5, -0.3], [-0.8, -0.6, 0.4]):   # origins inside room A only
        T = (START_A + np.array(off)).astype(np.float64)
        rel = (pts - T.astype(np.float32)).astype(np.float32)
        o.recast_pcl_to_map(np.eye(3), T, rel, None)
        m.integrate_points(rel, np.eye(3), o.input_T_np)
    assert_state(o._h, m)
    t = TopoGraphGen(o, coll_det_num=64, max_raycast_dist=2.5)
    r = TopoGraphGen(RefBackedMap(m), coll_det_num=64, max_raycast_dist=2.5)
    n = t.generate_topo_graph(START_A, max_nodes=8)
    nr = r.generate_topo_graph(START_A, max_nodes=8)
    assert n == nr >= 1
    nf = t.num_facelets[None]
    assert nf == r.num_facelets[None] > 0
    assert np.array_equal(t.tri_vertices.to_numpy()[:3 * nf], r.tri_vertices.to_numpy()[:3 * nf])
    assert np.array_equal(t.f_is_frontier.a[:nf], r.f_is_frontier.a[:nf])
    centres = t.tri_vertices.to_numpy()[:3 * nf].reshape(nf, 3, 3).mean(1).astype(np.float32)
    unk = o.is_pos_unobserved(centres)
    assert unk.any(), "no facelet centre lies in unknown space"
    assert np.array_equal(unk, m.query_points(centres)[1])


def test_pool_exhaustion_is_reported():
    from taichislam_b200 import _capi as capi
    h = handle(max_ray_length=5.0, max_blocks=16)
    h.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    with pytest.raises(capi.TslamError) as e:
        h.sync()
    assert e.value.code == capi.E_POOL_FULL
