"""The integrate launch's kernel chain: the generic path, the seg_count check and the control-block clear run in the tail
of k_march_blocks, the scan in the last CTA of k_seg_class_scan, the dirty-count reset in the last CTA of the commit.
Each must leave the state the next launch starts from exactly as the separate kernels did."""
import numpy as np
import pytest

from taichislam_b200 import synthetic as syn
from util import as_dict_rows, compare_voxels, rot_xyz

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _pair(map_scale, **kw):
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    o = OracleTSDF(map_scale=map_scale, K=syn.K_DEPTH, **kw)
    g = TsdfHandle(o.N, o.Nz, K=syn.K_DEPTH, **kw)
    return g, o


def _stats_equal(g, o):
    sg, so = g.stats(), o.stats()
    for k in ("n_px", "n_valid", "n_rays", "n_updates", "n_oob"):
        assert sg[k] == so[k], f"{k}: gpu {sg[k]} oracle {so[k]}"
    assert sg["err_flags"] == 0


@pytest.mark.parametrize("seg_cap", [None, "20000"])
def test_generic_path_in_the_march_tail(seg_cap, monkeypatch):
    """N = 200 (not a multiple of 16): blocks cut by the volume boundary and segments next to it take the generic path;
    with TSLAM_SEG_CAP the launch overflows and every segment does."""
    if seg_cap:
        monkeypatch.setenv("TSLAM_SEG_CAP", seg_cap)
    d = syn.scene_room()
    R = rot_xyz(0.1, -0.15, 0.3)
    T = np.array([0.21, -0.17, 0.08])
    g, o = _pair([10.0, 10.0], is_global_map=True)
    g.integrate_depth(d, R[None], T[None])
    o.integrate_depth(R, T, d)
    _stats_equal(g, o)
    ms = g.march_stats()
    assert ms["n_generic"] > 0 and ms["n_seg_guard"] == 0
    compare_voxels(g.gather(), o.gather(), 2e-3 if seg_cap else TOL)


def test_march_stats_match_a_reference_run():
    """n_seg_guard stays 0 and n_generic / n_updates are the same on every run of the same launches; n_updates is the
    canonical oracle's."""
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    d = syn.scene_room()  # N = 200: rays reach the volume boundary, the generic path has work
    Rs = np.stack([rot_xyz(0.1, -0.15 + 0.05 * q, 0.3) for q in range(4)])
    Ts = np.stack([np.array([0.21, -0.17, 0.08]) * (1 + q) for q in range(4)])
    runs = []
    for _ in range(2):
        g = TsdfHandle(200, 200, K=syn.K_DEPTH, is_global_map=True)
        g.integrate_depth(np.stack([d] * 4), Rs, Ts)
        g.sync()
        runs.append((g.stats(), g.march_stats()))
    # num_voxel_per_blk_axis = 1 and a map scale half a voxel short of 200 voxels: N = Nz = 200 exactly
    ref = OracleTSDF(map_scale=[199.5 * 0.05, 199.5 * 0.05], num_voxel_per_blk_axis=1, K=syn.K_DEPTH, is_global_map=True)
    assert (ref.N, ref.Nz) == (200, 200)
    for q in range(4):
        ref.integrate_depth(Rs[q], Ts[q], d, commit=(q == 3))
    (s0, m0), (s1, m1) = runs
    assert m0["n_seg_guard"] == 0 and m1["n_seg_guard"] == 0
    assert m0["n_generic"] > 0
    assert (m0["n_generic"], s0["n_updates"]) == (m1["n_generic"], s1["n_updates"])
    assert s0["n_updates"] == ref.stats()["n_updates"] and s0["err_flags"] == 0


def test_back_to_back_launches_equal_one_at_a_time():
    """Two launches of different geometry enqueued back to back must build the map of the same launches with a
    synchronisation after each: the control block, the ray count and the dirty count are cleared on the device."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    a, b = syn.scene_sphere(4.0), syn.scene_room()
    Ra, Ta = syn.stream_poses(8, start=2)
    Rb = np.stack([rot_xyz(0.1 * q, -0.05, 0.2) for q in range(8)])
    Tb = np.stack([np.array([0.3, -0.2, 0.1]) * q / 8 for q in range(8)])
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    g.integrate_depth(np.stack([a] * 8), Ra, Ta)
    g.integrate_depth(np.stack([b] * 8), Rb, Tb)
    g.sync()
    h = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    h.integrate_depth(np.stack([a] * 8), Ra, Ta)
    h.sync()
    sa = h.stats()
    h.integrate_depth(np.stack([b] * 8), Rb, Tb)
    h.sync()
    assert g.stats()["n_rays"] == h.stats()["n_rays"] > sa["n_rays"] > 0
    assert g.stats()["n_updates"] == h.stats()["n_updates"]
    assert g.march_stats()["n_seg_guard"] == 0
    x, y = as_dict_rows(*g.gather()), as_dict_rows(*h.gather())
    assert np.array_equal(x[0], y[0])
    assert np.abs(x[1] - y[1]).max() <= TOL


def test_point_cloud_and_textured_launches():
    """Point clouds take the same chain (one frame); textured maps k_raymarch and the colour commit.  Both against the oracle, twice in
    a row (the second launch starts from what the first one's tail cleared)."""
    rng = np.random.default_rng(11)
    u = rng.normal(size=(20000, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    pts = (u * rng.uniform(0.5, 6.0, size=(20000, 1))).astype(np.float32)
    g, o = _pair([25.6, 25.6], is_global_map=True)
    for q in range(2):
        R = rot_xyz(-0.2 + 0.1 * q, 0.3, 0.1)
        T = np.array([0.1, 0.2 * q, -0.3])
        g.integrate_points(pts, R, T)
        o.integrate_points(R, T, pts)
    _stats_equal(g, o)
    compare_voxels(g.gather(), o.gather(), TOL)

    from taichislam_b200.tsdf_handle import TsdfHandle
    d = syn.scene_sphere(3.0)
    tex = np.zeros(d.shape + (3,), np.uint8)
    tex[..., 0] = 200
    Rs, Ts = syn.stream_poses(4, start=1)
    t = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True, texture_enabled=True)
    u = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True)
    for q in range(2):
        t.integrate_depth(np.stack([d] * 2), Rs[2 * q:2 * q + 2], Ts[2 * q:2 * q + 2], texture=np.stack([tex] * 2))
        u.integrate_depth(np.stack([d] * 2), Rs[2 * q:2 * q + 2], Ts[2 * q:2 * q + 2])
    t.sync()
    u.sync()
    assert t.stats()["n_updates"] == u.stats()["n_updates"] > 0
    compare_voxels(t.gather(), u.gather(), TOL)


def test_kernels_per_depth_launch():
    """An untextured 64-frame depth launch with commit: bucket, counting walk, class + scan, scattering walk, march,
    dirty-list compaction, commit."""
    import torch
    from taichislam_b200.tsdf_handle import TsdfHandle
    d = syn.scene_sphere(4.0)
    Rs, Ts = syn.stream_poses(64, start=0)
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    dev = torch.from_numpy(np.stack([d] * 64).view(np.int16)).cuda()
    g.integrate_depth(dev, Rs, Ts, commit=True)
    l0 = g.launch_count()
    g.integrate_depth(dev, Rs, Ts, commit=True)
    assert g.launch_count() - l0 == 7
    g.sync()
