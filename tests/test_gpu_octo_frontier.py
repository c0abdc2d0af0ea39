"""Frontiers of the log-odds Octomap on the GPU against the numpy reference (octo_frontier_reference.py): the frontier
voxels, their cluster ordinals and the int64 cluster records, bit for bit."""
import numpy as np
import pytest

import octo_esdf_reference as oe
import octo_frontier_reference as fr
import octo_logodds_reference as ref
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu

VS = 0.05
LO = ref.params()


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


def expected(h, submap=0):
    idx, L = h.gather(submap)
    return fr.frontiers(idx, L, LO["l_occ"], h.N, h.Nz)


def got(h, submap=0):
    idx, cl = as_dict_rows(*h.frontier_gather(submap))
    return idx, cl, h.frontier_clusters(submap)


def assert_frontiers(h, submap=0):
    gi, gc, gr = got(h, submap)
    ri, rc, rr = expected(h, submap)
    assert gi.shape == ri.shape, f"frontier voxels: gpu {gi.shape[0]} reference {ri.shape[0]}"
    assert np.array_equal(gi, ri)
    assert gr.shape == rr.shape, f"clusters: gpu {gr.shape[0]} reference {rr.shape[0]}"
    bad = np.nonzero((gr != rr).any(1))[0]
    assert bad.size == 0, f"{bad.size} records differ, first gpu {gr[bad[:2]].tolist()} ref {rr[bad[:2]].tolist()}"
    assert np.array_equal(gc, rc)
    return gi, gc, gr


def same_state(a, b, submap=0):
    ai, ac, ar = got(a, submap)
    bi, bc, br = got(b, submap)
    return np.array_equal(ai, bi) and np.array_equal(ac, bc) and np.array_equal(ar, br)


def point_frame(h, origin, ends, submap=0):
    """one frame of point rays from cell `origin` to the cells `ends` (exact cell centres, identity rotation)"""
    o = np.asarray(origin, np.float32) * np.float32(VS)
    e = np.asarray(ends, np.float32).reshape(-1, 3) * np.float32(VS)
    h.integrate_points((e - o).astype(np.float32), np.eye(3), o.astype(np.float64), submap=submap)


SCENES = {"S1": lambda: syn.scene_plane(3.0), "S2": lambda: syn.scene_sphere(4.0), "S4": lambda: syn.scene_noise(4),
          "room": lambda: syn.scene_room()}


@pytest.mark.parametrize("scene", list(SCENES))
def test_full_update_matches_reference(scene):
    h = handle()
    d = SCENES[scene]()
    Rs, Ts = syn.stream_poses(2, start=40)
    for q in range(2):
        h.integrate_depth(d, Rs[q], Ts[q])
    st = h.frontier_update(0, full=True)
    assert st["full"] and st["voxels"] > 100 and st["clusters"] > 0
    gi, gc, gr = assert_frontiers(h)
    assert st["voxels"] == gi.shape[0] and st["clusters"] == gr.shape[0]
    assert (np.diff(gr[:, 0]) > 0).all() and gr[:, 1].sum() == gi.shape[0] and (gr[:, 15] == 0).all()


@pytest.mark.parametrize("scene", ["S2", "room"])
def test_incremental_equals_full_after_every_frame(scene):
    inc, full = handle(), handle()
    d = SCENES[scene]()
    poses = [syn.stream_pose(40 + 60 * q) for q in range(5)] + [(rot_xyz(0.0, 0.4, 0.3), np.array([0.3, -0.2, 0.1]))]
    for q, (R, T) in enumerate(poses):
        inc.integrate_depth(d, R, T)
        full.integrate_depth(d, R, T)
        st = inc.frontier_update(0)
        sf = full.frontier_update(0, full=True)
        assert st["full"] == (q == 0) and sf["full"], st
        assert 0 < st["blocks"] <= sf["blocks"] and (st["voxels"], st["clusters"]) == (sf["voxels"], sf["clusters"])
        assert_frontiers(inc)
        assert same_state(inc, full)


def test_clearing_occupied_cells_incrementally():
    inc, full = handle(), handle()
    for q, z in enumerate([2.0] * 3 + [4.0] * 8):        # the wall at 2 m is carved away, OCC turning FREE
        for h in (inc, full):
            h.integrate_depth(syn.scene_plane(z), np.eye(3), np.zeros(3))
        assert inc.frontier_update(0)["full"] == (q == 0)
        full.frontier_update(0, full=True)
        assert_frontiers(inc)
        assert same_state(inc, full)
    occ, _ = inc.query_points(np.array([[0.0, 0.0, 2.0]], np.float32))
    assert not occ[0]


def test_newly_known_cell_on_a_block_face_clears_the_unflagged_neighbour():
    h = handle(64, 64, min_ray_length=0.0)
    X, Y = (7, 3, 3), (8, 3, 3)                          # X in block (0,0,0), Y across its +x face in block (1,0,0)
    around = [(6, 3, 3), (7, 2, 3), (7, 4, 3), (7, 3, 2), (7, 3, 4)]
    point_frame(h, X, around)                            # X FREE, five neighbours OCC: Y is X's only UNKNOWN neighbour
    assert h.frontier_update(0)["full"]
    gi, _, gr = assert_frontiers(h)
    assert gi.tolist() == [list(X)] and gr[0, 11] == 1 and gr[0, 12:15].tolist() == [1, 0, 0]
    point_frame(h, Y, [(9, 3, 3)])                       # touches block (1,0,0) only
    st = h.frontier_update(0)
    assert not st["full"] and st["blocks"] >= 2          # the flagged block and its face neighbour holding X
    gi, _, _ = assert_frontiers(h)
    assert list(X) not in gi.tolist() and list(Y) in gi.tolist()


def test_cluster_across_a_block_corner():
    h = handle(64, 64, min_ray_length=0.0)
    point_frame(h, (7, 7, 7), [(7, 7, 6)])
    point_frame(h, (8, 8, 8), [(8, 8, 9)])               # FREE cells meeting only at the corner of 8^3 blocks
    point_frame(h, (-1, -1, -1), [(-1, -1, -2)])
    point_frame(h, (0, 0, 0), [(0, 0, 1)])
    assert h.frontier_update(0)["voxels"] == 4
    gi, gc, gr = assert_frontiers(h)
    assert gr.shape[0] == 2 and gr[:, 1].tolist() == [2, 2]
    # a path of cells through the corner of eight blocks, one frame per ray, incremental after each
    cells = [(6, 6, 6), (7, 6, 7), (8, 7, 8), (9, 8, 8), (8, 9, 9), (7, 8, 9)]
    for c in cells:
        point_frame(h, c, [(c[0], c[1], c[2] - 1)])
        assert not h.frontier_update(0)["full"]
        assert_frontiers(h)


def test_rays_reaching_the_volume_edge():
    inc = handle(64, 64)                                  # 3.2 m box, 5 m rays: rays are cut at the volume
    full = handle(64, 64)
    d = syn.scene_room()
    for q in range(4):
        R, T = syn.stream_pose(50 * q)
        for h in (inc, full):
            h.integrate_depth(d, R, T)
        inc.frontier_update(0)
        full.frontier_update(0, full=True)
        gi, _, gr = assert_frontiers(inc)
        assert same_state(inc, full)
    edge = (gi.min(0) == -32) | (gi.max(0) == 31)
    assert edge.any()


def test_two_submaps():
    h = handle(max_submaps=2)
    d = syn.scene_sphere(3.0)
    h.integrate_depth(d, np.eye(3), np.zeros(3), submap=0)
    h.integrate_depth(d, rot_xyz(0.0, 0.0, 1.0), np.array([0.4, 0.0, 0.0]), submap=1)
    h.frontier_update(0)
    f0 = assert_frontiers(h, 0)
    refused(h.frontier_gather, 1)
    refused(h.frontier_clusters, 1)
    assert h.frontier_update(1)["full"]
    assert_frontiers(h, 1)
    refused(h.frontier_gather, 0)
    h.integrate_depth(d, rot_xyz(0.0, 0.2, 1.0), np.array([0.4, 0.1, 0.0]), submap=1)
    h.integrate_depth(d, rot_xyz(0.0, 0.2, 0.0), np.zeros(3), submap=0)
    assert not h.frontier_update(1)["full"]
    assert_frontiers(h, 1)
    assert h.frontier_update(0)["full"]
    g0 = assert_frontiers(h, 0)
    assert not np.array_equal(g0[0], f0[0])


def test_reset_fusion_and_recycled_pool_slots():
    h = handle()
    d = syn.scene_room()
    h.integrate_depth(d, np.eye(3), np.zeros(3))
    h.frontier_update(0)
    h.reset()
    refused(h.frontier_gather, 0)
    refused(h.frontier_clusters, 0)
    # a small frame allocates a few blocks; the update after a reset is full ...
    h.integrate_points(np.array([[1.0, 0.2, 0.3]], np.float32), np.eye(3), np.zeros(3))
    assert h.frontier_update(0)["full"]
    assert_frontiers(h)
    # ... then whole frames land in pool slots that held frontier bits before the reset: incremental == full
    for R, T in [(rot_xyz(0.0, 0.2, 0.0), np.zeros(3)), (rot_xyz(0.0, -0.3, 0.1), np.array([0.0, 0.1, 0.0]))]:
        h.integrate_depth(d, R, T)
        assert not h.frontier_update(0)["full"]
        gi, gc, gr = assert_frontiers(h)
        h.frontier_update(0, full=True)
        fi, fc, fr_ = got(h)
        assert np.array_equal(fi, gi) and np.array_equal(fc, gc) and np.array_equal(fr_, gr)
    # fusion resets the target
    src = handle(max_submaps=2)
    src.integrate_depth(d, np.eye(3), np.zeros(3))
    h.set_submap_pose(0, np.eye(3), np.zeros(3))
    h.fuse_from(src)
    refused(h.frontier_gather, 0)
    assert h.frontier_update(0)["full"]
    assert_frontiers(h)


@pytest.mark.parametrize("esdf_first", [True, False])
def test_interleaved_with_the_esdf(esdf_first):
    h = handle(128, 128)
    d = syn.scene_room()
    D = 1.0
    for q in range(4):
        R, T = syn.stream_pose(45 * q)
        h.integrate_depth(d, R, T)
        if q == 2:      # one frame seen by neither: both trackers must still see its blocks
            continue
        steps = [lambda: h.esdf_update(0, D), lambda: h.frontier_update(0)]
        for s in (steps if esdf_first else steps[::-1]):
            s()
        assert_frontiers(h)
        idx, L = h.gather(0)
        ri, re_ = as_dict_rows(idx, oe.esdf(idx, L, LO["l_occ"], VS, D))
        gi, ge = as_dict_rows(*h.esdf_gather(0))
        assert np.array_equal(gi, ri) and np.array_equal(ge.view(np.int32), re_.view(np.int32))


def test_refusals_and_capacity():
    import ctypes as C
    import torch
    from taichislam_b200 import _capi as capi
    from taichislam_b200.mapping.taichi_octomap import Octomap
    from taichislam_b200.octo_handle import OctoHandle
    hits = OctoHandle(64, 64, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH)
    refused(hits.frontier_update, 0)
    refused(hits.frontier_gather, 0)
    refused(hits.frontier_clusters, 0)
    h = handle(64, 64, max_submaps=2)
    refused(h.frontier_gather, 0)                          # before any update
    refused(h.frontier_clusters, 0)
    L = capi.load()
    assert L.tslam_octo_frontier_update(h.h, 0, 2, None, None) == capi.E_INVALID
    assert L.tslam_octo_frontier_update(h.h, 2, 0, None, None) == capi.E_INVALID
    assert L.tslam_octo_frontier_update(h.h, -1, 0, None, None) == capi.E_INVALID
    refused(h.frontier_gather, 0)                          # a refused update computes nothing
    h.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    st = h.frontier_update(0)
    refused(h.frontier_gather, 1)
    refused(h.frontier_clusters, 1)
    n = C.c_int64(-1)
    dev = torch.device("cuda", torch.cuda.current_device())
    idx = torch.zeros((4, 3), dtype=torch.int32, device=dev)
    cl = torch.zeros(4, dtype=torch.int32, device=dev)
    rec = torch.zeros((1, 16), dtype=torch.int64, device=dev)
    assert L.tslam_octo_frontier_gather(h.h, 0, 4, capi.tptr(idx), capi.tptr(cl), C.byref(n), None) == capi.E_CAPACITY
    assert n.value == st["voxels"] > 4
    n.value = -1
    assert L.tslam_octo_frontier_gather(h.h, 0, 0, None, None, C.byref(n), None) == capi.E_CAPACITY
    assert n.value == st["voxels"]
    n.value = -1
    assert L.tslam_octo_frontier_clusters(h.h, 0, 1, capi.tptr(rec), C.byref(n), None) == capi.E_CAPACITY
    assert n.value == st["clusters"] > 1
    torch.cuda.synchronize()
    full = h.frontier_clusters(0)
    assert np.array_equal(rec.cpu().numpy(), full[:1])
    assert L.tslam_octo_frontier_gather(h.h, 0, 4, None, None, C.byref(n), None) == capi.E_INVALID
    assert L.tslam_octo_frontier_clusters(h.h, 0, 4, None, C.byref(n), None) == capi.E_INVALID
    assert L.tslam_octo_frontier_gather(h.h, 0, 0, None, None, None, None) == capi.E_INVALID
    assert L.tslam_octo_frontier_clusters(h.h, 0, -1, None, C.byref(n), None) == capi.E_INVALID
    o = Octomap(map_scale=[3.2, 3.2], voxel_scale=VS, max_disp_particles=16)
    for fn in (o.frontier_update, o.get_frontiers, o.get_frontier_clusters):
        with pytest.raises(ValueError):
            fn()


def test_octomap_class_flow():
    import torch
    from taichislam_b200.mapping.taichi_octomap import Octomap
    o = Octomap(map_scale=[12.8, 12.8], voxel_scale=VS, occupancy_model="logodds", max_ray_length=3.0, max_disp_particles=1024)
    o.set_dep_camera_intrinsic(syn.K_DEPTH)
    o.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    d = syn.scene_room()
    o.recast_depth_to_map(np.eye(3), np.zeros(3), d, None)
    st = o.frontier_update()
    assert st["full"] and st["voxels"] > 0
    o.recast_depth_to_map(rot_xyz(0.0, 0.0, 0.4), np.array([0.1, 0.0, 0.0]), d, None)
    st = o.frontier_update()
    assert not st["full"]
    gi, gc, gr = assert_frontiers(o._h)
    idx, cl = o.get_frontiers()
    assert np.array_equal(as_dict_rows(idx, cl)[0], gi)
    c = o.get_frontier_clusters()
    assert np.array_equal(c["label"], gr[:, 0]) and np.array_equal(c["size"], gr[:, 1]) and np.array_equal(c["faces"], gr[:, 11])
    vs = float(np.float32(VS))
    assert np.array_equal(c["centroid"], gr[:, 2:5].astype(np.float64) / gr[:, 1:2] * vs)
    assert np.array_equal(c["bbox_min"], gr[:, 5:8] * vs) and np.array_equal(c["bbox_max"], gr[:, 8:11] * vs)
    d3 = gr[:, 12:15].astype(np.float64)
    nz = (d3 != 0).any(1)
    assert nz.any() and np.allclose(np.linalg.norm(c["direction"][nz], axis=1), 1.0) and (c["direction"][~nz] == 0).all()
    big = o.get_frontier_clusters(min_voxels=10)
    assert np.array_equal(big["label"], gr[gr[:, 1] >= 10, 0])
    ti, tc = o._h.frontier_gather(0, as_torch=True)
    assert isinstance(ti, torch.Tensor) and ti.is_cuda
    o.reset()
    with pytest.raises(Exception):
        o.get_frontiers()


def test_submap_mapping_global_map_frontiers():
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    from taichislam_b200.mapping.taichi_octomap import Octomap
    sm = SubmapMapping(Octomap, keyframe_step=2,
                       sub_opts=dict(occupancy_model="logodds", map_scale=[12.8, 12.8], max_ray_length=4.0, max_submap_num=8),
                       global_opts=dict(occupancy_model="logodds", map_scale=[25.6, 25.6], max_ray_length=4.0, max_submap_num=8))
    sm.set_dep_camera_intrinsic(syn.K_DEPTH)
    d = syn.scene_sphere(3.0)
    for f in range(6):
        R, T = syn.stream_pose(30 * f, radius=1.0)
        sm.recast_depth_to_map_by_frame(f, True, (R, T), (np.eye(3), np.zeros(3)), d, None)
    sub = sm.submap_collection
    assert sub.frontier_update()["voxels"] > 0
    assert_frontiers(sub._h, sub._active())
    sm.local_to_global()
    g = sm.global_map
    st = g.frontier_update()
    assert st["full"] and st["clusters"] > 0
    assert_frontiers(g._h, g._active())
    assert g.get_frontier_clusters()["size"].sum() == st["voxels"]
