"""Argument checks of the tiled-ESDF entry points (ABI 5) that need no GPU: a NULL handle is refused by every one."""
import ctypes as C

import numpy as np

from taichislam_b200 import _capi as capi


def test_tiled_esdf_calls_refuse_a_null_handle():
    L = capi.load()
    tiles = (C.c_int32 * 3)(2, 1, 1)
    cnt = np.zeros(2, np.int32)
    sw = C.c_int32(0)
    assert L.tslam_tiling_owner_points(None, tiles, 2, 0, None, None, None) == capi.E_INVALID
    assert L.tslam_esdf_tiled_begin(None, 0, C.byref(sw), None) == capi.E_INVALID
    assert L.tslam_esdf_halo_count(None, tiles, 0, 2, capi.np_ptr(cnt), None) == capi.E_INVALID
    assert L.tslam_esdf_halo_pack(None, tiles, 0, 2, capi.np_ptr(cnt), 0, None, None, None) == capi.E_INVALID
    assert L.tslam_esdf_ghost_unpack(None, 0, None, None, None) == capi.E_INVALID
    assert L.tslam_esdf_tiled_relax(None, C.byref(sw), None) == capi.E_INVALID
    assert L.tslam_esdf_tiled_end(None) == capi.E_INVALID
