"""Sample-by-sample audit of the TSDF ray march against the exact f64 reference (tests/march_reference.py).

compare_voxels' 1e-4 bars cannot see a lost or doubled sample where the march is most fragile: voxels with 10^4
samples, or clamped at Wmax.  Here (a) edge-case point clouds are held to the reference within bounds derived per case
(util.march_bounds) and asserted to be well below one sample's effect; (b) every march path conserves samples exactly
on power-of-two weights: W is exact there, W/w is a sample count, and the counts must add up to n_updates."""
import ctypes as C

import numpy as np
import pytest

from march_cases import make_case, reference_of
from util import as_dict_rows, compare_to_reference

pytestmark = pytest.mark.gpu


def gpu_map(case, **kw):
    from taichislam_b200.tsdf_handle import TsdfHandle
    return TsdfHandle(case["N"], case["Nz"], voxel_scale=case["vs"], max_ray_length=case["max_ray_length"],
                      internal_voxels=case["internal_voxels"], is_global_map=True, **kw)


@pytest.mark.parametrize("name", ["hot_bundle", "ties_and_axes", "short_rays", "anisotropic", "tiny_weights", "fine_long", "long_range",
                                  "near_sensor"])
def test_binned_march_matches_reference(name):
    c = make_case(name)
    ref = reference_of(c)
    g = gpu_map(c)
    g.stats(clear=True)
    g.integrate_points(c["pts"], np.eye(3), c["T"])
    st, ms = g.stats(), g.march_stats()
    assert st["err_flags"] == 0 and st["n_rays"] == ref["n_rays"]
    assert st["n_updates"] == ref["n_updates"] and st["n_oob"] == ref["n_oob"]
    assert ms["n_segs"] > 0  # (segments in blocks next to the volume take the generic path: n_generic may be > 0)
    compare_to_reference(g.gather(), ref)
    if name == "hot_bundle":
        assert ms["n_items"] >= 5 and ref["count"].max() >= 20000
    if name == "tiny_weights":
        assert ms["n_fallback"] >= ref["n_tiny"] > 0, "the tiny-weight rays did not take the f32 global path"
    if name == "fine_long":
        assert ms["n_items"] > 0


def test_submap_1023_next_to_submap_0():
    """The top of the 10-bit submap field of the block key, in one collection with submap 0."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    c = make_case("anisotropic")
    ref = reference_of(c)
    g = TsdfHandle(c["N"], c["Nz"], voxel_scale=c["vs"], max_ray_length=c["max_ray_length"], max_submaps=1024)
    g.integrate_points(c["pts"], np.eye(3), c["T"], submap=1023)
    g.integrate_points(c["pts"], np.eye(3), c["T"], submap=0)
    for s in (0, 1023):
        compare_to_reference(g.gather(s), ref)
    assert g.count_active(1) == 0 and g.count_active(1022) == 0
    assert g.stats()["n_updates"] == 2 * ref["n_updates"]


# ---- sample conservation on every march path ------------------------------------------------------------------------
H, W = 48, 64
K = [40.0, 0, 31.5, 0, 40.0, 23.5, 0, 0, 1]
ZS = (2.0, 4.0, 8.0)


def plane_stream(n, seed=1):
    """n fronto-parallel depth planes cycling through z = 2, 4, 8 m (w = 1/z^2 exact for every ray of a frame) under
    seeded generic poses spread over a few metres, so that no voxel comes near Wmax."""
    rng = np.random.default_rng(seed)
    z = np.array([ZS[q % 3] for q in range(n)])
    d = np.stack([np.full((H, W), int(zz * 1000), np.uint16) for zz in z])
    from util import rot_xyz
    Rs = np.stack([rot_xyz(*rng.uniform(-0.6, 0.6, 3)) for _ in range(n)])
    Ts = rng.uniform(-3.0, 3.0, (n, 3))
    Ts[:, 2] *= 0.3
    return d, Rs, Ts, 1.0 / (z * z)


def oracle_counts(d, Rs, Ts):
    """The canonical oracle's map and per-frame in-bounds sample counts."""
    from oracle.oracle import OracleTSDF
    o = OracleTSDF(map_scale=[25.6, 25.6], K=K, is_global_map=True, recast_step=2)
    per = []
    for q in range(d.shape[0]):
        o.clear_stats()
        o.integrate_depth(Rs[q], Ts[q], d[q])
        per.append(o.stats()["n_updates"])
    return o, np.array(per)


def assert_conserved(g, o, per_frame, wf):
    gi, gt, gw = as_dict_rows(*g.gather()[:3])
    oi, ot, ow = as_dict_rows(*o.gather()[:3])
    assert gw.max() < 1000.0, "a voxel reached Wmax: W/w is no longer a count"
    assert np.array_equal(gi, oi), "observed voxel index sets differ"
    assert np.array_equal(gw.view(np.uint32), ow.view(np.uint32)), f"W not bit-equal at {int((gw != ow).sum())} voxels"
    # every W is an exact multiple of 1/64 below 1000: the sum over voxels is exact in f64
    n_upd = g.stats()["n_updates"]
    assert n_upd == per_frame.sum()
    assert gw.astype(np.float64).sum() == float(np.dot(per_frame, wf)), "samples lost or doubled"
    assert np.abs(gt - ot).max() <= 1e-4


def _queue(g, d, Rs, Ts):
    from taichislam_b200 import _capi as capi
    for q in range(d.shape[0]):
        f = np.ascontiguousarray(d[q])
        R9, T3 = capi.f32c(Rs[q]).reshape(9), capi.f32c(Ts[q]).reshape(3)
        capi.check(g.L.tslam_tsdf_queue_depth(g.h, f.ctypes.data_as(C.c_void_p), H, W, capi.np_ptr(R9), capi.np_ptr(T3), 0,
                                              capi.stream_ptr()))
    capi.check(g.L.tslam_tsdf_flush(g.h, capi.stream_ptr()))


PATHS = {"default": {}, "generic": {"TSLAM_SEG_CAP": "3000"},
         "verify": {"TSLAM_MARCH_VERIFY": "1"}, "textured": {}, "queue": {}}


@pytest.fixture(scope="module")
def planes():
    d, Rs, Ts, wf = plane_stream(40)
    o, per = oracle_counts(d, Rs, Ts)
    return d, Rs, Ts, wf, o, per


@pytest.mark.parametrize("path", sorted(PATHS))
def test_sample_conservation(path, planes, monkeypatch):
    from taichislam_b200.tsdf_handle import TsdfHandle
    d, Rs, Ts, wf, o, per = planes
    for k, v in PATHS[path].items():
        monkeypatch.setenv(k, v)
    g = TsdfHandle(o.N, o.Nz, K=K, is_global_map=True, recast_step=2, texture_enabled=(path == "textured"))
    if path == "textured":
        g.set_color_intrinsics(K, True)
        g.integrate_depth(d, Rs, Ts, texture=np.full((d.shape[0], H, W, 3), 77, np.uint8))
    elif path == "queue":
        _queue(g, d, Rs, Ts)
    else:
        g.integrate_depth(d, Rs, Ts)
    g.sync()
    ms = g.march_stats()
    if path == "generic":
        assert ms["n_generic"] > 0
    if path == "verify":
        assert ms["n_verify_bad"] == 0
    if path == "textured":
        assert ms["n_segs"] == 0
    assert_conserved(g, o, per, wf)


def test_sample_conservation_130_frame_call():
    """One integrate_depth call of 130 frames (launches of 64 + 64 + 2) against 130 single-frame calls."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    d, Rs, Ts, wf = plane_stream(130, seed=2)
    o, per = oracle_counts(d, Rs, Ts)
    g = TsdfHandle(o.N, o.Nz, K=K, is_global_map=True, recast_step=2)
    g.integrate_depth(d, Rs, Ts)
    assert_conserved(g, o, per, wf)
    g1 = TsdfHandle(o.N, o.Nz, K=K, is_global_map=True, recast_step=2)
    for q in range(130):
        g1.integrate_depth(d[q], Rs[q][None], Ts[q][None])
    a, b = as_dict_rows(*g.gather()[:3]), as_dict_rows(*g1.gather()[:3])
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])
    assert g1.stats()["n_updates"] == per.sum()
