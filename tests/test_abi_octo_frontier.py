"""Argument checks of the frontier entry points that need no GPU: a NULL handle or NULL arrays are refused."""
import ctypes as C

from taichislam_b200 import _capi as capi


def test_octo_frontier_calls_refuse_null_handle_and_arrays():
    L = capi.load()
    n = C.c_int64(0)
    st4 = (C.c_int32 * 4)()
    buf = (C.c_int64 * 32)()
    p = C.cast(buf, C.c_void_p)
    assert L.tslam_octo_frontier_update(None, 0, 0, st4, None) == capi.E_INVALID
    assert L.tslam_octo_frontier_update(None, 0, 1, None, None) == capi.E_INVALID
    assert L.tslam_octo_frontier_gather(None, 0, 0, None, None, C.byref(n), None) == capi.E_INVALID
    assert L.tslam_octo_frontier_gather(None, 0, 4, p, p, C.byref(n), None) == capi.E_INVALID
    assert L.tslam_octo_frontier_gather(None, 0, 4, None, None, None, None) == capi.E_INVALID
    assert L.tslam_octo_frontier_clusters(None, 0, 0, None, C.byref(n), None) == capi.E_INVALID
    assert L.tslam_octo_frontier_clusters(None, 0, 2, p, C.byref(n), None) == capi.E_INVALID
    assert L.tslam_octo_frontier_clusters(None, 0, 2, None, None, None) == capi.E_INVALID
