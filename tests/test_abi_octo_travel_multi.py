"""Argument checks of the many-source travel-cost entry points that need no GPU: a NULL handle or arrays and n_starts out
of range are refused."""
import ctypes as C

from taichislam_b200 import _capi as capi


def test_octo_travel_multi_calls_refuse_null_handle_and_arrays():
    L = capi.load()
    buf = (C.c_int64 * 32)()
    p = C.cast(buf, C.c_void_p)
    for S in (0, 1, 4, 1024, 1025, -1):
        assert L.tslam_octo_travel_multi_update(None, 0, S, p, 0.0, 1.0, p, p, p, None) == capi.E_INVALID
    assert L.tslam_octo_travel_multi_update(None, 0, 4, None, 0.0, 1.0, None, None, None, None) == capi.E_INVALID
    for k in (0, 4, -1):
        assert L.tslam_octo_travel_multi_query(None, 0, k, p, p, None) == capi.E_INVALID
        assert L.tslam_octo_travel_multi_path(None, 0, k, p, p, 16, p, p, None) == capi.E_INVALID
    assert L.tslam_octo_travel_multi_query(None, 0, 4, None, None, None) == capi.E_INVALID
    assert L.tslam_octo_travel_multi_path(None, 0, 4, None, None, 16, None, None, None) == capi.E_INVALID
    assert L.tslam_octo_travel_multi_path(None, 0, 4, p, p, 0, p, p, None) == capi.E_INVALID
