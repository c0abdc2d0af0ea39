"""Argument checks of tslam_octo_frontier_viewpoints that need no GPU: a NULL handle, camera, offsets or outputs are
refused."""
import ctypes as C

from taichislam_b200 import _capi as capi


def test_octo_frontier_viewpoints_refuses_null_handle_camera_offsets_and_outputs():
    L = capi.load()
    cam = capi.ViewCamera(100.0, 100.0, 80.0, 60.0, 160, 120, 2, 3.0)
    buf = (C.c_int64 * 64)()
    p = C.cast(buf, C.c_void_p)
    f = L.tslam_octo_frontier_viewpoints
    for nc in (0, 3):
        assert f(None, 0, C.byref(cam), 4, p, 0.0, 1, 1, nc, p, p, p, p, p, None) == capi.E_INVALID
        assert f(None, 0, None, 4, p, 0.0, 1, 1, nc, p, p, p, p, p, None) == capi.E_INVALID
        assert f(None, 0, C.byref(cam), 4, None, 0.0, 1, 1, nc, p, p, p, p, p, None) == capi.E_INVALID
    for q in range(5):
        outs = [p] * 5
        outs[q] = None
        assert f(None, 0, C.byref(cam), 4, p, 0.0, 1, 1, 3, *outs, None) == capi.E_INVALID
    assert L.tslam_abi_version() == 6                                  # an additive entry point
