"""Argument checks of the tiled planner-query entry points (ABI 6) that need no GPU: a NULL handle is refused by every
one."""
import ctypes as C

import numpy as np

from taichislam_b200 import _capi as capi


def test_tiled_query_calls_refuse_a_null_handle():
    L = capi.load()
    tiles = (C.c_int32 * 3)(2, 1, 1)
    assert capi.ABI_VERSION == 6
    assert L.tslam_tiling_owner_cells(None, tiles, 2, 0, None, None, None) == capi.E_INVALID
    assert L.tslam_tsdf_raycast_tiled(None, tiles, 0, 2, 0, 0, None, None, None, None, None, None) == capi.E_INVALID
    assert L.tslam_tsdf_query_near_occupy_tiled(None, 0, 0, None, 1, None, None) == capi.E_INVALID
    one = np.zeros(8, np.float32)
    assert L.tslam_tsdf_query_near_occupy_tiled(None, 0, 1, capi.np_ptr(one), 1, capi.np_ptr(one), None) == capi.E_INVALID
