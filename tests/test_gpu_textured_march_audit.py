"""Sample-by-sample audit of the textured ray march (k_raymarch) against the exact f64 reference (tests/march_reference.py,
path="textured"), colours included.

k_raymarch is its own kernel: one thread per ray, a 16^3 shared-memory window of fixed-point sums around the sensor
origin of each round of 512 rays, f32 reductions for the other samples, a 64-bit colour word raised per sample.  Here
(a) every edge-case cloud of the audit goes through a textured handle and is held to the reference within the textured
bounds, with exact colours; (b) later integrate calls win the colour; (c) samples are conserved exactly when the rays of
one round come from frames of other submaps and other sensor origins than the round's window; (d) the colour word's
frame counter wraps (k_cword_renorm) without changing a colour."""
import ctypes as C

import numpy as np
import pytest

from march_cases import CASES, make_case, reference_of
from test_gpu_march_audit import H, K, W, plane_stream
from util import as_dict_rows, compare_to_reference, key_sort, one_sample_effect, march_bounds

pytestmark = pytest.mark.gpu


def textured_map(case, **kw):
    from taichislam_b200.tsdf_handle import TsdfHandle
    return TsdfHandle(case["N"], case["Nz"], voxel_scale=case["vs"], max_ray_length=case["max_ray_length"],
                      internal_voxels=case["internal_voxels"], is_global_map=True, texture_enabled=True,
                      max_points=max(case["pts"].shape[0], 1 << 16), **kw)


def assert_colors(gi, gc, ref):
    """Colours equal the reference's words exactly, except where its f32 and exact closeness bins disagree."""
    _, gc = as_dict_rows(gi, gc)
    bad = (gc != ref["color"]).any(1)
    assert not (bad & ~ref["color_amb"]).any(), f"{int((bad & ~ref['color_amb']).sum())} of {len(gc)} voxel colours differ"


@pytest.mark.parametrize("name", sorted(CASES))
def test_textured_march_matches_reference(name):
    c = make_case(name)
    ref = reference_of(c, "textured")
    g = textured_map(c)
    g.stats(clear=True)
    g.integrate_points(c["pts"], np.eye(3), c["T"], rgb=c["rgb"])
    st = g.stats()
    assert st["err_flags"] == 0 and st["n_rays"] == ref["n_rays"]
    assert st["n_updates"] == ref["n_updates"] and st["n_oob"] == ref["n_oob"]
    gi, gt, gw, _, gc = g.gather(color=True)
    # hot_bundle: 75 rounds each flush an f32 reduction into the voxels next to the sensor; the worst case of those
    # roundings is about one sample's TSDF spread there, so only W (still well below one sample) is held sharp
    compare_to_reference((gi, gt, gw), ref, sharp=name != "hot_bundle")
    if name == "hot_bundle":
        h = int(np.argmax(ref["count"]))
        assert march_bounds(ref)[0][h] < 0.15 * one_sample_effect(ref)[0][h]
    assert_colors(gi, gc, ref)


def test_textured_later_calls_win():
    """Three integrate_points calls of one cloud with different colours: the colour of every voxel the last call
    reaches is the last call's, as the oracle has it, exactly."""
    from oracle.oracle import OracleTSDF
    c = make_case("anisotropic")
    vs, N, Nz = c["vs"], c["N"], c["Nz"]
    o = OracleTSDF(map_scale=[(N - 0.5) * vs, (Nz - 0.5) * vs], voxel_scale=vs, num_voxel_per_blk_axis=1,
                   max_ray_length=c["max_ray_length"], internal_voxels=c["internal_voxels"], is_global_map=True)
    o.set_color(True, True)
    g = textured_map(c)
    for q in range(3):
        rgb = np.roll(c["rgb"], 7 * q + 1, axis=0) if q else c["rgb"]
        T = c["T"] + np.float32(0.25 * q)
        g.integrate_points(c["pts"], np.eye(3), T, rgb=rgb)
        o.integrate_points_rgb(np.eye(3), T, c["pts"], rgb)
        last = reference_of(dict(c, T=T, rgb=rgb), "textured", seq=q + 1)
    gi, gt, gw, _, gc = g.gather(color=True)
    oi, ot, ow, _ = o.gather()
    oc = o.gather_color()
    assert np.array_equal(gi[key_sort(gi)], oi[key_sort(oi)])
    assert np.array_equal(gc[key_sort(gi)], oc[key_sort(oi)]), "colours differ from the oracle's"
    gi, gc = as_dict_rows(gi, gc)
    sel = np.isin(gi.view([("", gi.dtype)] * 3).ravel(), last["idx"].view([("", gi.dtype)] * 3).ravel())
    assert sel.sum() == last["idx"].shape[0]
    ok = ~last["color_amb"]
    assert np.array_equal(gc[sel][ok], last["color"][ok]), "an earlier call's colour survived the last call"


def test_textured_sample_conservation_across_submaps():
    """One textured depth launch of 40 frames whose submaps alternate 0/1 and whose sensor origin moves every frame:
    rays of a round come from frames outside the round's window or submap.  W stays bit-equal to the oracle per
    submap and the sums of W stay exact."""
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    d, Rs, Ts, wf = plane_stream(40, seed=4)
    sub = np.arange(40) % 2
    o = OracleTSDF(map_scale=[25.6, 25.6], K=K, is_global_map=True, recast_step=2)
    per = []
    for q in range(40):
        o.clear_stats()
        o.integrate_depth(Rs[q], Ts[q], d[q], submap=int(sub[q]))
        per.append(o.stats()["n_updates"])
    per = np.array(per)
    g = TsdfHandle(o.N, o.Nz, K=K, is_global_map=True, recast_step=2, texture_enabled=True, max_submaps=2)
    g.set_color_intrinsics(K, True)
    g.integrate_depth(d, Rs, Ts, submaps=sub, texture=np.full((40, H, W, 3), 77, np.uint8))
    g.sync()
    assert g.stats()["n_updates"] == per.sum()
    total = 0.0
    for s in (0, 1):
        gi, gt, gw = as_dict_rows(*g.gather(s)[:3])
        oi, ot, ow = as_dict_rows(*o.gather(s)[:3])
        assert gw.max() < 1000.0 and np.array_equal(gi, oi)
        assert np.array_equal(gw.view(np.uint32), ow.view(np.uint32)), f"submap {s}: W not bit-equal at {int((gw != ow).sum())} voxels"
        assert np.abs(gt - ot).max() <= 1e-4
        total += gw.astype(np.float64).sum()
    assert total == float(np.dot(per, wf)), "samples lost or doubled"


# ---- the colour word's frame counter across its 22-bit limit -------------------------------------------------------
SEQ_LIMIT = (1 << 22) - 1


def _queue_tex(g, d, tex, Rs, Ts):
    from taichislam_b200 import _capi as capi
    for q in range(d.shape[0]):
        f, t = np.ascontiguousarray(d[q]), np.ascontiguousarray(tex[q])
        R9, T3 = capi.f32c(Rs[q]).reshape(9), capi.f32c(Ts[q]).reshape(3)
        capi.check(g.L.tslam_tsdf_queue_depth_tex(g.h, f.ctypes.data_as(C.c_void_p), t.ctypes.data_as(C.c_void_p), H, W, H, W,
                                                  capi.np_ptr(R9), capi.np_ptr(T3), 0, capi.stream_ptr()))
    capi.check(g.L.tslam_tsdf_flush(g.h, capi.stream_ptr()))


@pytest.mark.parametrize("mode", ["batched", "queue", "points"])
def test_colour_sequence_wrap(mode, monkeypatch):
    """Frames integrated across the frame counter's limit (TSLAM_FRAME_SEQ0 starts it just below): the stored words
    are renormalised and later frames still win, so the colours equal those of the oracle, which never wraps."""
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    n = 64 if mode == "queue" else 40
    d, Rs, Ts, _ = plane_stream(n, seed=5)
    rng = np.random.default_rng(6)
    tex = rng.integers(0, 256, (n, H, W, 3)).astype(np.uint8)
    monkeypatch.setenv("TSLAM_FRAME_SEQ0", str(SEQ_LIMIT - (40 if mode == "queue" else 20)))
    o = OracleTSDF(map_scale=[25.6, 25.6], K=K, is_global_map=True, recast_step=2)
    o.set_color(True, True)
    g = TsdfHandle(o.N, o.Nz, K=K, is_global_map=True, recast_step=2, texture_enabled=True)
    g.set_color_intrinsics(K, True)
    if mode == "points":
        pts = [np.ascontiguousarray(rng.normal(size=(3000, 3)).astype(np.float32) * np.float32(1.5)) for _ in range(n)]
        rgb = [rng.integers(0, 256, (3000, 3)).astype(np.uint8) for _ in range(n)]
        for q in range(n):
            g.integrate_points(pts[q], Rs[q], Ts[q], rgb=rgb[q])
            o.integrate_points_rgb(Rs[q], Ts[q], pts[q], rgb[q])
    else:
        if mode == "batched":
            for b in range(0, n, 8):  # launches of 8 frames: the third starts past the limit
                g.integrate_depth(d[b:b + 8], Rs[b:b + 8], Ts[b:b + 8], texture=tex[b:b + 8])
        else:  # two queue launches of 32 frames: the second starts past the limit
            _queue_tex(g, d, tex, Rs, Ts)
        for q in range(n):
            o.integrate_depth_tex(Rs[q], Ts[q], d[q], tex[q])
    g.sync()
    gi, gt, gw, _, gc = g.gather(color=True)
    oi, ot, ow, _ = o.gather()
    oc = o.gather_color()
    a, b = key_sort(gi), key_sort(oi)
    assert np.array_equal(gi[a], oi[b])
    assert np.abs(gt[a] - ot[b]).max() <= 1e-4
    assert len(np.unique(oc, axis=0)) > 100
    bad = (gc[a] != oc[b]).any(1)
    assert not bad.any(), f"{int(bad.sum())} of {len(gc)} voxel colours differ across the frame counter's wrap"
