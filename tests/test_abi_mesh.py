"""Argument checks of the incremental-mesh entry points that need no GPU: a NULL handle is refused by every one."""
import ctypes as C

from taichislam_b200 import _capi as capi


def test_mesh_calls_refuse_a_null_handle():
    L = capi.load()
    out = C.c_void_p()
    n = C.c_int64(0)
    full = C.c_int32(0)
    assert L.tslam_mesh_create(None, C.byref(out)) == capi.E_INVALID and not out.value
    assert L.tslam_mesh_destroy(None) == capi.TSLAM_OK  # like tslam_tsdf_destroy: nothing to free
    assert L.tslam_mesh_update(None, 0.1, 0, None, None, None, C.byref(n), None, None) == capi.E_INVALID
    assert L.tslam_mesh_updated_blocks(None, 0, None, None, None, C.byref(n), C.byref(full), None) == capi.E_INVALID
