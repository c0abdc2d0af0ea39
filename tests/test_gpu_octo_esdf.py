"""Occupancy ESDF of the log-odds Octomap on the GPU against the numpy reference (octo_esdf_reference.py), bit for bit
as int32 views, and its queries against tests/esdf_query_reference.py."""
import numpy as np
import pytest

import esdf_query_reference as eq
import octo_esdf_reference as oe
import octo_logodds_reference as ref
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu

VS = 0.05
LO = ref.params()
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


def expected(h, submap=0, d=D):
    """(idx, E) of the reference on the map's current known voxels, rows sorted."""
    idx, L = h.gather(submap)
    return as_dict_rows(idx, oe.esdf(idx, L, LO["l_occ"], VS, d))


def field(h, submap=0):
    return as_dict_rows(*h.esdf_gather(submap))


def assert_field(h, submap=0, d=D):
    gi, ge = field(h, submap)
    ri, re_ = expected(h, submap, d)
    assert gi.shape == ri.shape, f"known voxels: gpu {gi.shape[0]} reference {ri.shape[0]}"
    assert np.array_equal(gi, ri)
    bad = np.nonzero(ge.view(np.int32) != re_.view(np.int32))[0]
    assert bad.size == 0, f"{bad.size} voxels differ, first {gi[bad[:4]].tolist()} gpu {ge[bad[:4]]} ref {re_[bad[:4]]}"
    return gi, ge


SCENES = {"S1": lambda: syn.scene_plane(3.0), "S2": lambda: syn.scene_sphere(4.0), "S4": lambda: syn.scene_noise(4),
          "room": lambda: syn.scene_room()}


@pytest.mark.parametrize("scene", list(SCENES))
def test_full_update_matches_reference(scene):
    h = handle()
    d = SCENES[scene]()
    Rs, Ts = syn.stream_poses(2, start=40)
    for q in range(2):
        h.integrate_depth(d, Rs[q], Ts[q])
    st = h.esdf_update(0, D, full=True)
    assert st["raise_sweeps"] == -1 and st["lower_sweeps"] > 1
    _, e = assert_field(h)
    assert (e == np.float32(D)).any() and (e > 0).any() and (e < 0).any()


@pytest.mark.parametrize("scene", ["S2", "room"])
def test_incremental_equals_full_after_every_frame(scene):
    h = handle()
    d = SCENES[scene]()
    poses = [syn.stream_pose(40 + 60 * q) for q in range(5)] + [(rot_xyz(0.0, 0.4, 0.3), np.array([0.3, -0.2, 0.1]))]
    for q, (R, T) in enumerate(poses):
        h.integrate_depth(d, R, T)
        st = h.esdf_update(0, D)
        if q == 0:
            assert st["raise_sweeps"] == -1
        else:
            assert st["raise_sweeps"] >= 0 and st["changed"] > 0, st
        gi, ge = assert_field(h)
        assert h.esdf_update(0, D, full=True)["raise_sweeps"] == -1
        fi, fe = field(h)
        assert np.array_equal(fi, gi) and np.array_equal(fe.view(np.int32), ge.view(np.int32))


def test_dynamic_clearing_runs_the_raise_wave():
    h = handle()
    suspects, raised = 0, 0
    for q, z in enumerate([2.0] * 3 + [4.0] * 8):
        h.integrate_depth(syn.scene_plane(z), np.eye(3), np.zeros(3))
        st = h.esdf_update(0, D)
        if q:
            assert st["raise_sweeps"] >= 0
        suspects += st["suspect"]
        raised = max(raised, st["raise_sweeps"])
        assert_field(h)
    occ, _ = h.query_points(np.array([[0.0, 0.0, 2.0]], np.float32))
    assert not occ[0]                      # the wall at 2 m is gone
    assert suspects > 0 and raised > 1


def test_block_seams_and_point_rays():
    h = handle(64, 64, min_ray_length=0.0)
    ends = np.array([[7, 7, 7], [15, -1, 7], [-1, -1, -1], [7, 15, -9], [23, 7, 7], [-9, -17, 15], [7, 0, 0], [8, 8, 8]],
                    np.float32) * np.float32(VS)
    for q, e in enumerate(ends):   # one ray per frame: occupied end cells on 8^3 block seams and corners
        h.integrate_points(e[None], np.eye(3), np.zeros(3))
        st = h.esdf_update(0, D)
        assert st["raise_sweeps"] == -1 if q == 0 else (st["raise_sweeps"] >= 0 and st["changed"] > 0), st
        assert_field(h)
    # a shell of points on the seams i & 7 == 7, seen from two origins
    g = np.argwhere(np.ones((4, 4, 4), bool)) * 8 - 9
    pts = g.astype(np.float32) * np.float32(VS)
    for T in (np.zeros(3), np.array([0.12, -0.07, 0.2])):
        h.integrate_points((pts - T.astype(np.float32)).astype(np.float32), np.eye(3), T)
        assert h.esdf_update(0, D)["raise_sweeps"] >= 0
        assert_field(h)


def test_d_change_reset_and_fusion_force_a_full_update():
    h = handle()
    d = syn.scene_room()
    h.integrate_depth(d, np.eye(3), np.zeros(3))
    h.esdf_update(0, D)
    h.integrate_depth(d, rot_xyz(0.0, 0.0, 0.3), np.array([0.1, 0.0, 0.0]))
    assert h.esdf_update(0, 0.5)["raise_sweeps"] == -1
    assert_field(h, d=0.5)
    assert h.esdf_update(0, 0.5)["raise_sweeps"] >= 0   # nothing changed since: incremental, nothing to do
    assert_field(h, d=0.5)
    # reset: readers refuse until the next update, which is full
    h.reset()
    refused(h.esdf_gather, 0)
    refused(h.esdf_query, np.zeros((4, 3), np.float32))
    # a single ray allocates a few blocks; the next update is full ...
    h.integrate_points(np.array([[1.0, 0.2, 0.3]], np.float32), np.eye(3), np.zeros(3))
    assert h.esdf_update(0, D)["raise_sweeps"] == -1
    assert_field(h)
    # ... then whole frames land in pool slots that held the field before the reset: incremental == full
    for R, T in [(rot_xyz(0.0, 0.2, 0.0), np.zeros(3)), (rot_xyz(0.0, -0.3, 0.1), np.array([0.0, 0.1, 0.0]))]:
        h.integrate_depth(d, R, T)
        assert h.esdf_update(0, D)["raise_sweeps"] >= 0
        gi, ge = assert_field(h)
        h.esdf_update(0, D, full=True)
        fi, fe = field(h)
        assert np.array_equal(fi, gi) and np.array_equal(fe.view(np.int32), ge.view(np.int32))
    # fusion resets the target
    src = handle(max_submaps=2)
    src.integrate_depth(d, np.eye(3), np.zeros(3))
    h.set_submap_pose(0, np.eye(3), np.zeros(3))
    h.fuse_from(src)
    refused(h.esdf_gather, 0)
    assert h.esdf_update(0, D)["raise_sweeps"] == -1
    assert_field(h)


def test_two_submaps_have_separate_fields():
    h = handle(max_submaps=2)
    d = syn.scene_sphere(3.0)
    h.integrate_depth(d, np.eye(3), np.zeros(3), submap=0)
    h.integrate_depth(d, rot_xyz(0.0, 0.0, 1.0), np.array([0.4, 0.0, 0.0]), submap=1)
    h.esdf_update(0, D)
    f0 = assert_field(h, 0)
    refused(h.esdf_gather, 1)
    assert h.esdf_update(1, D)["raise_sweeps"] == -1
    assert_field(h, 1)
    refused(h.esdf_query, np.zeros((4, 3), np.float32), submap=0)
    h.integrate_depth(d, rot_xyz(0.0, 0.2, 1.0), np.array([0.4, 0.1, 0.0]), submap=1)
    h.integrate_depth(d, rot_xyz(0.0, 0.2, 0.0), np.zeros(3), submap=0)
    assert h.esdf_update(1, D)["raise_sweeps"] >= 0
    assert_field(h, 1)
    assert h.esdf_update(0, D)["raise_sweeps"] == -1
    g0 = assert_field(h, 0)
    assert g0[0].shape[0] > f0[0].shape[0]


def seam_points(rng, n):
    """points whose interpolation cube straddles 8^3 block seams on one, two or three axes"""
    c = rng.integers(-12, 12, (n, 3)) * 8 - 1          # i0 & 7 == 7
    keep = rng.random((n, 3)) < 0.5
    c = np.where(keep, c, rng.integers(-90, 90, (n, 3)))
    u = c + rng.random((n, 3))
    return (u * VS).astype(np.float32)


def test_queries_bit_exact_and_as_of_the_last_update():
    import torch
    h = handle()
    d = syn.scene_room()
    for R, T in [(np.eye(3), np.zeros(3)), (rot_xyz(0.0, 0.0, 0.7), np.array([0.2, 0.1, 0.0]))]:
        h.integrate_depth(d, R, T)
    h.esdf_update(0, D)
    idx, e = h.esdf_gather(0)
    st = eq.EsdfState(idx, np.zeros(len(e), np.float32), e, 256, 256, VS)
    rng = np.random.default_rng(11)
    pts = np.concatenate([rng.uniform(-6.5, 6.5, (1 << 16, 3)).astype(np.float32), seam_points(rng, 1 << 14),
                          np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [6.35, 0, 0], [-6.4, -6.4, -6.4],
                                    [6.4, 0, 0]], np.float32)])
    want = eq.query(st, pts)

    def same(got):
        dist, grad, valid = got
        assert np.array_equal(valid, want[2])
        assert np.array_equal(dist.view(np.int32), want[0].view(np.int32))
        assert np.array_equal(grad.view(np.int32), want[1].view(np.int32))

    got = h.esdf_query(pts)
    same(got)
    assert got[2].sum() > 1000 and (~got[2]).sum() > 1000
    assert np.isnan(got[0][-6:-3]).all()
    # torch in -> torch out
    tg = h.esdf_query(torch.from_numpy(pts).cuda())
    assert all(isinstance(t, torch.Tensor) and t.is_cuda for t in tg)
    same(tuple(t.cpu().numpy() for t in tg))
    assert h.esdf_query(np.zeros((0, 3), np.float32))[0].shape == (0,)
    # more integration without an update: the answers stay those of the last update; new blocks read invalid
    h.integrate_depth(d, rot_xyz(0.0, 0.0, 2.5), np.array([-0.3, 0.0, 0.0]))
    same(h.esdf_query(pts))
    ni, _ = h.gather(0)
    new = ~np.isin(ref.pack(ni >> 3), ref.pack(idx >> 3))
    assert new.sum() > 1000
    probe = (ni[new][:2000].astype(np.float32) + np.float32(0.25)) * np.float32(VS)
    assert not h.esdf_query(probe)[2].any()
    h.esdf_update(0, D)
    assert h.esdf_query(probe)[2].any()


def test_refusals():
    from taichislam_b200 import _capi as capi
    from taichislam_b200.mapping.taichi_octomap import Octomap
    from taichislam_b200.octo_handle import OctoHandle
    hits = OctoHandle(64, 64, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH)
    refused(hits.esdf_update, 0, D)
    refused(hits.esdf_gather, 0)
    refused(hits.esdf_query, np.zeros((4, 3), np.float32))
    h = handle(64, 64, max_submaps=2)
    refused(h.esdf_gather, 0)                                    # before any update
    refused(h.esdf_query, np.zeros((4, 3), np.float32))
    for bad in (float("nan"), float("inf"), -float("inf"), 0.0, -1.0):
        refused(h.esdf_update, 0, bad)
    refused(h.esdf_gather, 0)                                    # a refused update computes nothing
    h.integrate_depth(syn.scene_room(), np.eye(3), np.zeros(3))
    h.esdf_update(0, D)
    refused(h.esdf_gather, 1)
    refused(h.esdf_query, np.zeros((4, 3), np.float32), submap=1)
    assert h.esdf_query(np.zeros((0, 3), np.float32))[2].shape == (0,)
    with pytest.raises(ValueError):
        Octomap(map_scale=[3.2, 3.2], voxel_scale=VS, max_disp_particles=16).esdf_update()
    assert capi.load().tslam_octo_esdf_update(h.h, 0, D, 2, None, None) == capi.E_INVALID


def test_octomap_class_flow():
    import torch
    from taichislam_b200.mapping.taichi_octomap import Octomap
    o = Octomap(map_scale=[12.8, 12.8], voxel_scale=VS, occupancy_model="logodds", max_ray_length=3.0, max_disp_particles=1024)
    o.set_dep_camera_intrinsic(syn.K_DEPTH)
    o.set_base_pose_submap(0, np.eye(3), np.zeros(3))
    d = syn.scene_room()
    o.recast_depth_to_map(np.eye(3), np.zeros(3), d, None)
    rng = np.random.default_rng(4)
    pts = rng.uniform(-3.5, 3.5, (20000, 3)).astype(np.float32)
    dist, grad, valid = o.esdf_query(pts)                  # update=True: D defaults to max_ray_length
    assert o.esdf_max_dist == 3.0 and valid.any()
    assert_field(o._h, d=3.0)
    hd, hg, hv = o._h.esdf_query(pts)
    assert np.array_equal(valid, hv) and np.array_equal(dist.view(np.int32), hd.view(np.int32))
    assert np.array_equal(grad.view(np.int32), hg.view(np.int32))
    o.recast_depth_to_map(rot_xyz(0.0, 0.0, 0.4), np.array([0.1, 0.0, 0.0]), d, None)
    stale = o.esdf_query(pts, update=False)[0]
    assert np.array_equal(stale.view(np.int32), dist.view(np.int32))
    td, tg, tv = o.esdf_query(torch.from_numpy(pts).cuda())
    assert isinstance(td, torch.Tensor)
    assert_field(o._h, d=3.0)
    gi, ge = as_dict_rows(*o.get_voxels_ESDF())
    fi, fe = field(o._h)
    assert np.array_equal(gi, fi) and np.array_equal(ge, fe)
    st = o.esdf_update(1.0)
    assert st["raise_sweeps"] == -1 and o.esdf_max_dist == 1.0
    assert_field(o._h, d=1.0)
