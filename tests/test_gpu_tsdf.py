"""GPU parity tests of the TSDF path: CUDA kernels (through the C ABI) vs the CPU oracle.

Bar: observed-voxel index sets, occupy flags and all counters bit-exact; TSDF / W within 1e-4
(the only order-dependent arithmetic is the f32 sum of the contributions of different rays to
one voxel, REDG.ADD.F32x2)."""
import json
import os

import numpy as np
import pytest

from taichislam_b200 import synthetic as syn
from util import compare_voxels, as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu
TOL = 1e-4
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "golden.json")))


def make_pair(map_scale, **kw):
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    gpu_only = {k: kw.pop(k) for k in ("max_submaps", "max_blocks", "max_image_pixels", "max_points") if k in kw}
    o = OracleTSDF(map_scale=map_scale, K=syn.K_DEPTH, **kw)
    okw = dict(kw)
    okw.pop("num_voxel_per_blk_axis", None)
    g = TsdfHandle(o.N, o.Nz, K=syn.K_DEPTH, **okw, **gpu_only)
    return g, o


def stats_equal(g, o):
    sg, so = g.stats(), o.stats()
    for k in ("n_px", "n_valid", "n_rays", "n_updates", "n_oob"):
        assert sg[k] == so[k], f"{k}: gpu {sg[k]} oracle {so[k]}"
    assert sg["err_flags"] == 0


def test_c1_single_frame_256():
    """BASELINE config 1: one synthetic 640x480 frame (S1) into a 256^3 TSDF, identity pose."""
    g, o = make_pair([12.8, 12.8], is_global_map=True)
    d = syn.scene_plane(3.0)
    g.integrate_depth(d, np.eye(3)[None], np.zeros((1, 3)))
    o.integrate_depth(np.eye(3), np.zeros(3), d)
    stats_equal(g, o)
    assert g.count_active() == o.count_active() == GOLD["integrate_256"]["S1_plane3m"]["active"]
    compare_voxels(g.gather(), o.gather(), TOL)


@pytest.mark.parametrize("scene", ["sphere4", "room", "noise"])
def test_single_frame_generic_pose_512(scene):
    d = {"sphere4": syn.scene_sphere(4.0), "room": syn.scene_room(), "noise": syn.scene_noise()}[scene]
    R = rot_xyz(0.15, -0.1, 0.4)
    T = np.array([0.31, -0.27, 0.12])
    g, o = make_pair([25.6, 25.6], is_global_map=True)
    g.integrate_depth(d, R[None], T[None])
    o.integrate_depth(R, T, d)
    stats_equal(g, o)
    compare_voxels(g.gather(), o.gather(), TOL)


def test_stream_batch_equals_sequential_frames():
    """12 frames of the bench stream.  (a) one batched call, committed once == oracle accumulating the 12 frames and
    committing once; (b) frame-by-frame calls with a commit each == oracle committing every frame; (c) the two
    granularities agree wherever the Wmax=1000 clamp never bound (W < 1000): the only place commit granularity can
    matter (dense_tsdf.py:267)."""
    n = 12
    d = np.stack([syn.scene_sphere(4.0)] * n)
    Rs, Ts = syn.stream_poses(n, start=5)
    g, o = make_pair([25.6, 25.6], is_global_map=True)
    g.integrate_depth(d, Rs, Ts)
    for q in range(n):
        o.integrate_depth(Rs[q], Ts[q], d[q], commit=(q == n - 1))
    stats_equal(g, o)
    compare_voxels(g.gather(), o.gather(), TOL)
    g2, o2 = make_pair([25.6, 25.6], is_global_map=True)
    for q in range(n):
        g2.integrate_depth(d[q], Rs[q][None], Ts[q][None], commit=True)
        o2.integrate_depth(Rs[q], Ts[q], d[q], commit=True)
    compare_voxels(g2.gather(), o2.gather(), TOL)
    i1, t1, w1, _ = as_dict_rows(*g.gather())
    i2, t2, w2, _ = as_dict_rows(*g2.gather())
    assert np.array_equal(i1, i2)
    free = (w1 < 999.0) & (w2 < 999.0)
    assert free.mean() > 0.9
    assert np.abs(t1[free] - t2[free]).max() <= TOL and np.all(np.abs(w1[free] - w2[free]) <= 1e-4 * np.maximum(1, w1[free]))


def test_device_resident_input_and_uncommitted_reads():
    import torch
    d = syn.scene_room()
    dd = torch.from_numpy(d.view(np.int16)).cuda().view(torch.int16)
    g, o = make_pair([25.6, 25.6], is_global_map=True)
    g.integrate_depth(dd[None].contiguous(), np.eye(3)[None], np.zeros((1, 3)), commit=False)
    o.integrate_depth(np.eye(3), np.zeros(3), d)
    # readers flush pending sums themselves
    assert g.count_active() == o.count_active()
    compare_voxels(g.gather(), o.gather(), TOL)


def test_point_cloud_path():
    rng = np.random.default_rng(7)
    u = rng.normal(size=(20000, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    pts = (u * rng.uniform(0.5, 6.0, size=(20000, 1))).astype(np.float32)
    pts[:50] *= 40.0  # beyond max_ray_length -> filtered (dense_tsdf.py:177)
    R = rot_xyz(-0.2, 0.3, 0.1)
    T = np.array([0.1, 0.2, -0.3])
    g, o = make_pair([25.6, 25.6], is_global_map=True)
    g.integrate_points(pts, R, T)
    o.integrate_points(R, T, pts)
    stats_equal(g, o)
    compare_voxels(g.gather(), o.gather(), TOL)


def test_submaps_and_out_of_volume_rays():
    """Small volume (rays leave it -> skipped, counted) and two submaps in one collection."""
    d = syn.scene_sphere(4.0)
    g, o = make_pair([3.2, 3.2], is_global_map=False, max_submaps=8)
    R = rot_xyz(0.0, 0.5, 0.0)
    g.integrate_depth(np.stack([d, d]), np.stack([np.eye(3), R]), np.zeros((2, 3)), submaps=[0, 3])
    o.integrate_depth(np.eye(3), np.zeros(3), d, submap=0)
    o.integrate_depth(R, np.zeros(3), d, submap=3)
    stats_equal(g, o)
    assert o.stats()["n_oob"] > 0
    for s in (0, 3):
        compare_voxels(g.gather(s), o.gather(s), TOL)
    assert g.count_active(1) == 0


def test_empty_and_ragged_frames():
    g, o = make_pair([12.8, 12.8], is_global_map=True, max_image_pixels=640 * 480)
    z = np.zeros((480, 640), np.uint16)
    g.integrate_depth(z, np.eye(3)[None], np.zeros((1, 3)))
    assert g.count_active() == 0 and g.stats()["n_rays"] == 0
    d = syn.scene_room()[:333, :457].copy()  # odd sizes: range(0, h/step) truncates (dense_tsdf.py:192)
    g.integrate_depth(d, np.eye(3)[None], np.zeros((1, 3)))
    o.integrate_depth(np.eye(3), np.zeros(3), z)
    o.integrate_depth(np.eye(3), np.zeros(3), d)
    stats_equal(g, o)
    compare_voxels(g.gather(), o.gather(), TOL)


def test_scatter_gather_roundtrip_golden_crop():
    """load_numpy -> count_active -> to_numpy on the crop of the reference's shipped map."""
    z = np.load(os.path.join(HERE, "golden", "ri_new_crop.npz"))
    from taichislam_b200.tsdf_handle import TsdfHandle
    from oracle.oracle import tsdf_dims
    N, Nz = tsdf_dims(list(z["map_scale"]), float(z["voxel_size"]), 16)
    g = TsdfHandle(N, Nz, voxel_scale=float(z["voxel_size"]), is_global_map=True)
    g.scatter(0, z["indices"].astype(np.int32), z["TSDF"].astype(np.float32), z["W_TSDF"].astype(np.float32), z["occupy"])
    assert g.count_active() == GOLD["crop"]["voxels"]
    idx, t, w, occ = as_dict_rows(*g.gather())
    ci, ct, cw, co = as_dict_rows(z["indices"].astype(np.int32), z["TSDF"], z["W_TSDF"], z["occupy"])
    assert np.array_equal(idx, ci)
    assert np.array_equal(t.astype(np.float16).view(np.uint16), ct.view(np.uint16))  # NaNs included, bit-exact
    assert np.array_equal(w.astype(np.float16).view(np.uint16), cw.view(np.uint16))
    assert np.array_equal(occ, co)
    g.reset()
    assert g.count_active() == 0


def test_surface_and_slice_export():
    d = syn.scene_room()
    R = rot_xyz(0.0, 0.2, 0.1)
    T = np.array([0.0, 0.0, 0.4])
    g, o = make_pair([25.6, 25.6], is_global_map=True, disp_floor=-2.0, disp_ceiling=6.0)
    g.integrate_depth(d, R[None], T[None])
    o.integrate_depth(R, T, d)
    ng, xg, cg = g.surface()
    no, xo, co = o.surface()
    assert ng == no and ng > 1000
    og, oo = np.lexsort(xg.T[::-1]), np.lexsort(xo.T[::-1])
    # voxels whose |TSDF| sits within 1e-4 of the 1.8*vs threshold could flip; none should on this scene
    assert np.array_equal(xg[og], xo[oo])
    assert np.allclose(cg[og], co[oo], atol=1e-6)
    ng, xg, vg = g.slice(3.0, 0.5)
    no, xo, vo = o.slice(3.0, 0.5)
    assert ng == no and ng > 100
    og, oo = np.lexsort(xg.T[::-1]), np.lexsort(xo.T[::-1])
    assert np.array_equal(xg[og], xo[oo])
    assert np.allclose(vg[og], vo[oo], atol=TOL)
    # capacity saturation: count still reports the demand
    n_full = g.surface()[0]
    n2, x2, _ = g.surface(cap=100)
    assert n2 == n_full and x2.shape[0] == 100


def test_submap_fusion():
    """fuse_submaps (dense_tsdf.py:272-318): two submaps with generic poses splatted into a global map."""
    d = syn.scene_sphere(2.0, 240, 320)
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    K = [syn.FX / 2, 0, syn.CX / 2, 0, syn.FY / 2, syn.CY / 2, 0, 0, 1]
    so = OracleTSDF(map_scale=[6.4, 6.4], K=K, max_ray_length=3.0)
    sg = TsdfHandle(so.N, so.Nz, K=K, max_ray_length=3.0, max_submaps=8)
    go = OracleTSDF(map_scale=[12.8, 12.8], is_global_map=True)
    gg = TsdfHandle(go.N, go.Nz, is_global_map=True, max_submaps=8)
    poses = {0: (rot_xyz(0.1, 0.2, 0.3), np.array([0.5, 0.1, -0.2])), 1: (rot_xyz(-0.3, 0.1, 1.0), np.array([-0.4, 0.6, 0.3]))}
    for s, (R, T) in poses.items():
        sg.integrate_depth(d, np.eye(3)[None], np.zeros((1, 3)), submaps=[s])
        so.integrate_depth(np.eye(3), np.zeros(3), d, submap=s)
        gg.set_submap_pose(s, R, T)
        go.set_submap_pose(s, R, T)
    gg.fuse_from(sg)
    go.fuse_from(so)
    gi, gt, gw, gocc = as_dict_rows(*gg.gather())
    oi, ot, ow, oocc = as_dict_rows(*go.gather())
    assert np.array_equal(gi, oi)
    assert np.array_equal(gocc.astype(np.int32), np.clip(oocc, -128, 127))
    # the reference's sequential RMW poisons a voxel with NaN when a zero-weight corner arrives first
    # (0*NaN, dense_tsdf.py:275); the order-free sum only yields NaN when the TOTAL weight is zero.
    fin = np.isfinite(ot)
    assert fin.mean() > 0.99
    assert np.all(np.isfinite(gt[fin]))
    assert np.abs(gt[fin] - ot[fin]).max() <= TOL
    assert np.all(np.abs(gw[fin] - ow[fin]) <= TOL * np.maximum(1.0, ow[fin]))
    # fusing again after a pose update rebuilds the map from scratch (reset + re-splat)
    gg.fuse_from(sg)
    assert np.array_equal(as_dict_rows(*gg.gather())[0], oi)


def test_pool_exhaustion_is_reported():
    from taichislam_b200.tsdf_handle import TsdfHandle
    from taichislam_b200 import _capi as capi
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True, max_blocks=16)
    g.integrate_depth(syn.scene_sphere(4.0), np.eye(3)[None], np.zeros((1, 3)))
    with pytest.raises(capi.TslamError) as e:
        g.sync()
    assert e.value.code == capi.E_POOL_FULL


def test_bucket_key_range_is_reported():
    """The per-frame bucket index keys a bucket by 13 bits per axis (+-4095 voxels around the sensor origin).  A surface
    point further away than that (9 m at 2 mm voxels) is dropped and reported by the next synchronising call - it must
    not alias into another bucket."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    from taichislam_b200 import _capi as capi
    g = TsdfHandle(512, 512, voxel_scale=0.002, K=syn.K_DEPTH, is_global_map=True)
    g.integrate_depth(syn.scene_sphere(9.0), np.eye(3)[None], np.zeros((1, 3)))
    with pytest.raises(capi.TslamError) as e:
        g.sync()
    assert e.value.code == capi.E_CAPACITY
    g2 = TsdfHandle(512, 512, voxel_scale=0.002, K=syn.K_DEPTH, is_global_map=True)
    g2.integrate_depth(syn.scene_sphere(4.0), np.eye(3)[None], np.zeros((1, 3)))  # 2000 voxels: inside the key range
    g2.sync()
    assert g2.stats()["n_rays"] > 1000


def test_full_size_properties_512():
    """Size-independent properties at the bench configuration (512^3, 64-frame batches):
    integrating the same stream twice doubles every weight and leaves every TSDF value unchanged;
    the sum of weights equals rays*steps*w accounting; reset empties the map."""
    n = 64
    d = np.stack([syn.scene_sphere(4.0)] * n)
    Rs, Ts = syn.stream_poses(n)
    g, _ = make_pair([25.6, 25.6], is_global_map=True)
    g.integrate_depth(d, Rs, Ts)
    i1, t1, w1, _ = as_dict_rows(*g.gather())
    st1 = g.stats()
    assert st1["n_rays"] > 10000 * n // 2 and st1["err_flags"] == 0
    g.integrate_depth(d, Rs, Ts)
    i2, t2, w2, _ = as_dict_rows(*g.gather())
    assert np.array_equal(i1, i2)
    free = w2 < 999.0  # Wmax clamp (dense_tsdf.py:267) binds next to the camera, where thousands of rays overlap
    assert free.mean() > 0.9 and (~free).sum() > 0
    assert np.allclose(w2[free], 2.0 * w1[free], rtol=1e-5)
    assert np.all(w2[~free] <= 1000.0) and np.any(w2 == 1000.0)
    assert np.abs(t2 - t1).max() <= TOL
    assert g.stats()["n_updates"] == 2 * st1["n_updates"]
    g.reset()
    assert g.count_active() == 0


def test_block_axis_10_and_long_range_config():
    """SubmapMapping's default num_voxel_per_blk_axis=10 (N not a multiple of the internal 16^3 block) and a
    max_ray_length >= 60 m configuration (per-pixel reductions instead of the warp-merged ones in the bucket kernel)."""
    d = syn.scene_room()
    R = rot_xyz(0.05, 0.1, -0.2)
    T = np.array([0.1, 0.05, 0.0])
    g, o = make_pair([10, 10], is_global_map=True, num_voxel_per_blk_axis=10)
    assert o.N == 200
    g.integrate_depth(d, R[None], T[None])
    o.integrate_depth(R, T, d)
    stats_equal(g, o)
    assert o.stats()["n_oob"] > 0
    compare_voxels(g.gather(), o.gather(), TOL)
    far = (syn.scene_room().astype(np.float32) * 10).clip(0, 65000).astype(np.uint16)  # up to 50 m
    g2, o2 = make_pair([102.4, 102.4], is_global_map=True, max_ray_length=64.0, voxel_scale=0.2)
    g2.integrate_depth(far, R[None], T[None])
    o2.integrate_depth(R, T, far)
    stats_equal(g2, o2)
    # TSDF values reach 64 m here: the 1e-4 bar of the default configuration (values <= 10 m) scales with the
    # magnitude of the f32 sums (relative 2e-5 observed at the voxels next to the sensor, thousands of contributions)
    compare_voxels(g2.gather(), o2.gather(), 2e-3)


def _march_run(monkeypatch, env, scene="room"):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    d = {"room": syn.scene_room(), "noise": syn.scene_noise()}[scene]
    n = 3
    Rs, Ts = syn.stream_poses(n, start=11)
    g, o = make_pair([25.6, 25.6], is_global_map=True)
    g.integrate_depth(np.stack([d] * n), Rs, Ts)
    for q in range(n):
        o.integrate_depth(Rs[q], Ts[q], d, commit=(q == n - 1))
    return g, o


def test_binned_march_fast_index_is_exact(monkeypatch):
    """The block-binned march takes a voxel index from ONE fused multiply-add per axis when the fraction is at least
    near_eps from .5, and recomputes round((u*j*vs + T)/vs) literally otherwise.  TSLAM_MARCH_VERIFY=1 recomputes
    every index: not one fast-path index may differ (n_verify_bad), and the exact path must be the rare one."""
    g, o = _march_run(monkeypatch, {"TSLAM_MARCH_VERIFY": "1"}, "noise")
    stats_equal(g, o)
    compare_voxels(g.gather(), o.gather(), TOL)
    ms = g.march_stats()
    assert ms["n_verify_bad"] == 0 and ms["n_segs"] > 0
    assert ms["n_slow"] < 0.01 * g.stats()["n_updates"]


def test_binned_march_overflow_path_agrees(monkeypatch):
    """Segment workspace too small -> the rays that do not fit take the exact one-reduction-per-sample path, which must
    build the map of the default path."""
    g0, o = _march_run(monkeypatch, {})
    ref = g0.gather()
    compare_voxels(ref, o.gather(), TOL)
    g1, _ = _march_run(monkeypatch, {"TSLAM_SEG_CAP": "20000"})
    assert g1.march_stats()["n_generic"] > 0
    # here EVERY sample went through the fallback (plain f32 global reductions, arbitrary order): the handful of voxels at
    # the sensor origin sum ~1e5 samples each and carry the f32 accumulation noise (<= 1e-4 relative) that the
    # shared-memory fixed-point sums of the binned path do not have
    compare_voxels(g1.gather(), ref, 2e-3)
    a, b = as_dict_rows(*g1.gather()), as_dict_rows(*ref)
    assert (np.abs(a[1] - b[1]) > TOL).mean() < 1e-4
