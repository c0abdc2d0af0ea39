"""Argument checks of the travel-cost entry points that need no GPU: a NULL handle or arrays are refused."""
import ctypes as C

from taichislam_b200 import _capi as capi


def test_octo_travel_calls_refuse_null_handle_and_arrays():
    L = capi.load()
    buf = (C.c_int64 * 32)()
    p = C.cast(buf, C.c_void_p)
    n = C.c_int64(0)
    assert L.tslam_octo_travel_update(None, 0, p, 0.0, 1.0, p, None) == capi.E_INVALID
    assert L.tslam_octo_travel_update(None, 0, None, 0.0, 1.0, None, None) == capi.E_INVALID
    assert L.tslam_octo_travel_gather(None, 0, 4, p, p, C.byref(n), None) == capi.E_INVALID
    assert L.tslam_octo_travel_gather(None, 0, 0, None, None, None, None) == capi.E_INVALID
    for k in (0, 4, -1):
        assert L.tslam_octo_travel_query(None, 0, k, p, p, None) == capi.E_INVALID
        assert L.tslam_octo_travel_path(None, 0, k, p, 16, p, p, None) == capi.E_INVALID
    assert L.tslam_octo_travel_query(None, 0, 4, None, None, None) == capi.E_INVALID
    assert L.tslam_octo_travel_path(None, 0, 4, None, 16, None, None, None) == capi.E_INVALID
    assert L.tslam_octo_travel_path(None, 0, 4, p, 0, p, p, None) == capi.E_INVALID
