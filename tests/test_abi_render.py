"""Argument checks of tslam_tsdf_render that need no GPU: cameras, image size, intrinsics, depth range, sample count and
output arrays are refused before the handle is looked at; the ABI version is unchanged."""
import ctypes as C
import math

from taichislam_b200 import _capi as capi


def _render(n=1, h=48, w=64, K4=(500.0, 500.0, 32.0, 24.0), z_min=0.3, z_max=6.0, step=0.05, null=None, handle=False):
    L = capi.load()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    k4 = (C.c_double * 4)(*K4)
    arrays = dict(K4=C.cast(k4, C.c_void_p), depth=p, status=p)
    if null is not None:
        arrays[null] = None
    m = p if handle else None               # no handle: every check below comes first
    rc = L.tslam_tsdf_render(m, n, h, w, arrays["K4"], None, p, p, z_min, z_max, step, arrays["depth"], None, None, arrays["status"], None)
    return rc, L.tslam_last_error().decode()


def test_camera_count_outside_range_is_refused():
    for n in (0, -1, capi.RENDER_MAX_CAMERAS + 1):
        rc, msg = _render(n=n)
        assert rc == capi.E_INVALID and "outside" in msg, n


def test_image_size_is_refused():
    for kw in (dict(h=0), dict(w=0), dict(h=-3), dict(n=2, h=32768, w=32768), dict(n=1, h=65536, w=32768)):
        rc, msg = _render(**kw)
        assert rc == capi.E_INVALID and "height and width" in msg, kw
    assert "height and width" not in _render(n=1, h=65535, w=32767)[1]     # n h w = 2^31 - 98301 passes this check


def test_bad_intrinsics_are_refused():
    for K4 in ((0.0, 500.0, 32.0, 24.0), (500.0, -1.0, 32.0, 24.0), (math.inf, 500.0, 32.0, 24.0), (500.0, math.nan, 32.0, 24.0),
               (500.0, 500.0, math.nan, 24.0), (500.0, 500.0, 32.0, math.inf), (1e-60, 500.0, 32.0, 24.0), (1e60, 500.0, 32.0, 24.0)):
        rc, msg = _render(K4=K4)
        assert rc == capi.E_INVALID and "fx, fy" in msg, K4


def test_bad_depth_range_and_step_are_refused():
    for kw in (dict(z_min=0.0), dict(z_min=-0.1), dict(z_min=math.nan), dict(z_min=math.inf), dict(z_max=0.3), dict(z_max=0.2),
               dict(z_max=math.inf), dict(z_max=math.nan), dict(step=0.0), dict(step=-0.05), dict(step=math.nan), dict(step=math.inf)):
        rc, msg = _render(**kw)
        assert rc == capi.E_INVALID and "z_min" in msg, kw


def test_too_many_samples_are_refused():
    # K = floor((z_max - z_min) / step) + 1: 65536 samples pass, 65537 do not
    assert "samples" not in _render(z_min=1.0, z_max=1.0 + 65535 * 0.0625, step=0.0625)[1]
    rc, msg = _render(z_min=1.0, z_max=1.0 + 65536 * 0.0625, step=0.0625)
    assert rc == capi.E_INVALID and "samples" in msg


def test_null_outputs_and_handle_are_refused():
    for q in ("K4", "depth", "status"):
        rc, msg = _render(null=q, handle=True)
        assert rc == capi.E_INVALID and "NULL" in msg and "handle" not in msg, q
    rc, msg = _render()
    assert rc == capi.E_INVALID and "NULL handle" in msg


def test_abi_version_is_unchanged():
    assert capi.load().tslam_abi_version() == 6 and capi.ABI_VERSION == 6          # additive entry point
