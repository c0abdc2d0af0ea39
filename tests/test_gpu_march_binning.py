"""The binned march finds each segment twice: a counting walk sizes the blocks' runs, a scattering walk recomputes the
segments from the stored ray records and fills the runs.  Every slot a run was given must be filled by exactly one
segment.  n_seg_guard counts the segments the two walks disagreed about, whether routed to the generic path by a guard
of the scattering walk or counted and never placed.  It must be 0 whatever the scene, pose and configuration."""
import numpy as np
import pytest

from taichislam_b200 import synthetic as syn
from util import as_dict_rows, compare_voxels, rot_xyz

pytestmark = pytest.mark.gpu
TOL = 1e-4

SCENES = {"S1": lambda: syn.scene_plane(3.0), "S2": lambda: syn.scene_sphere(4.0), "S3": lambda: syn.scene_sphere(8.0),
          "S4": lambda: syn.scene_noise()}


def _stream(g, d, n, start=3):
    Rs, Ts = syn.stream_poses(n, start=start)
    g.integrate_depth(np.stack([d] * n), Rs, Ts)
    g.sync()


@pytest.mark.parametrize("scene", sorted(SCENES))
def test_walks_agree_on_bench_scenes(scene):
    """64 frames of the bench stream into a 512^3 map, in one launch; the map must equal the canonical oracle's."""
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    d = SCENES[scene]()
    o = OracleTSDF(map_scale=[25.6, 25.6], K=syn.K_DEPTH, is_global_map=True)
    g = TsdfHandle(o.N, o.Nz, K=syn.K_DEPTH, is_global_map=True)
    _stream(g, d, 64)
    st, ms = g.stats(), g.march_stats()
    assert st["err_flags"] == 0
    assert ms["n_segs"] > 0 and ms["n_items"] > 0
    assert ms["n_seg_guard"] == 0
    Rs, Ts = syn.stream_poses(64, start=3)
    for q in range(64):  # the launch commits once, after its last frame
        o.integrate_depth(Rs[q], Ts[q], d, commit=(q == 63))
    so = o.stats()
    for k in ("n_rays", "n_updates", "n_oob"):
        assert st[k] == so[k], k
    compare_voxels(g.gather(), o.gather(), TOL)


def _same_map(g, g_f32):
    """Same voxels; TSDF within the f32 accumulation noise of g_f32, whose global reductions sum the 10^4-10^5
    contributions of the voxels next to the sensor in arbitrary order (the binned march sums them exactly)."""
    a, b = as_dict_rows(*g.gather()), as_dict_rows(*g_f32.gather())
    assert np.array_equal(a[0], b[0])
    d = np.abs(a[1] - b[1])
    assert d.max() <= 2e-3 and (d > 1e-4).mean() < 1e-4


@pytest.mark.parametrize("scene", ["sphere4", "room", "noise"])
def test_walks_agree_under_generic_poses(scene):
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    d = {"sphere4": syn.scene_sphere(4.0), "room": syn.scene_room(), "noise": syn.scene_noise()}[scene]
    R = rot_xyz(0.15, -0.1, 0.4)
    T = np.array([0.31, -0.27, 0.12])
    o = OracleTSDF(map_scale=[25.6, 25.6], K=syn.K_DEPTH, is_global_map=True)
    g = TsdfHandle(o.N, o.Nz, K=syn.K_DEPTH, is_global_map=True)
    g.integrate_depth(d, R[None], T[None])
    o.integrate_depth(R, T, d)
    st, so, ms = g.stats(), o.stats(), g.march_stats()
    for k in ("n_rays", "n_updates", "n_oob"):
        assert st[k] == so[k], k
    assert st["err_flags"] == 0
    assert ms["n_segs"] > 0 and ms["n_seg_guard"] == 0
    compare_voxels(g.gather(), o.gather(), TOL)


def test_walks_agree_on_long_range_and_cut_blocks():
    """max_ray_length 64 m at 0.2 m voxels (long rays, many block crossings), and N = 200 (blocks cut by the volume
    boundary, segments next to it on the generic path)."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    R = rot_xyz(0.05, 0.1, -0.2)
    T = np.array([0.1, 0.05, 0.0])
    far = (syn.scene_room().astype(np.float32) * 10).clip(0, 65000).astype(np.uint16)  # up to 50 m
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True, max_ray_length=64.0, voxel_scale=0.2)
    g.integrate_depth(far, R[None], T[None])
    ms = g.march_stats()
    assert g.stats()["err_flags"] == 0
    assert ms["n_segs"] > 0 and ms["n_seg_guard"] == 0
    g2 = TsdfHandle(200, 200, K=syn.K_DEPTH, is_global_map=True)
    g2.integrate_depth(syn.scene_room(), R[None], T[None])
    ms2 = g2.march_stats()
    assert g2.stats()["err_flags"] == 0 and g2.stats()["n_oob"] > 0
    assert ms2["n_segs"] > 0 and ms2["n_generic"] > 0 and ms2["n_seg_guard"] == 0


def test_more_segments_than_the_workspace_take_the_generic_path(monkeypatch):
    """The counting walk may count more segments than `seg` holds: the launch overflows, every segment takes the generic
    path, and the map is the one of the binned path."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    d = syn.scene_sphere(4.0)
    g0 = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    _stream(g0, d, 4)
    monkeypatch.setenv("TSLAM_SEG_CAP", "50000")
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    _stream(g, d, 4)
    st, st0, ms = g.stats(), g0.stats(), g.march_stats()
    assert st["err_flags"] == 0
    assert ms["n_segs"] > 50000 and ms["n_items"] == 0 and ms["n_seg_guard"] == 0 and ms["n_generic"] > 0
    assert (st["n_rays"], st["n_updates"], st["n_oob"]) == (st0["n_rays"], st0["n_updates"], st0["n_oob"])
    _same_map(g0, g)
