"""Argument checks of the viewpoint-gain entry points that need no GPU: a NULL handle, camera or arrays are refused."""
import ctypes as C

from taichislam_b200 import _capi as capi


def test_octo_view_gain_calls_refuse_null_handle_camera_and_arrays():
    L = capi.load()
    cam = capi.ViewCamera(100.0, 100.0, 80.0, 60.0, 160, 120, 2, 3.0)
    buf = (C.c_int64 * 32)()
    p = C.cast(buf, C.c_void_p)
    for n in (0, 4):
        assert L.tslam_octo_view_gain_unknown(None, 0, n, p, p, C.byref(cam), p, p, None) == capi.E_INVALID
        assert L.tslam_octo_view_gain_frontier(None, 0, n, p, p, C.byref(cam), 1, p, p, p, None) == capi.E_INVALID
    assert L.tslam_octo_view_gain_unknown(None, 0, 4, p, p, None, p, p, None) == capi.E_INVALID
    assert L.tslam_octo_view_gain_unknown(None, 0, 4, None, None, C.byref(cam), None, None, None) == capi.E_INVALID
    assert L.tslam_octo_view_gain_unknown(None, 0, -1, p, p, C.byref(cam), p, p, None) == capi.E_INVALID
    assert L.tslam_octo_view_gain_frontier(None, 0, 4, p, p, None, 1, p, p, None, None) == capi.E_INVALID
    assert L.tslam_octo_view_gain_frontier(None, 0, 4, None, None, C.byref(cam), 1, None, None, None, None) == capi.E_INVALID
    assert L.tslam_octo_view_gain_frontier(None, 0, -1, p, p, C.byref(cam), 1, p, p, p, None) == capi.E_INVALID
