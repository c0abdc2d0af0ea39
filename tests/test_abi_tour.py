"""Argument checks of tslam_tour_open that need no GPU: NULL arrays, n, restarts and max_passes out of range are refused
before the matrix is read."""
import ctypes as C

import numpy as np

from taichislam_b200 import _capi as capi


def test_tour_open_refuses_null_arrays_and_ranges():
    L = capi.load()
    buf = (C.c_int64 * 64)()
    p = C.cast(buf, C.c_void_p)
    info2 = np.zeros(2, np.int32)
    ip = capi.np_ptr(info2)

    def call(n=4, cost=p, R=2, mp=8, tours=p, cost2=p, passes=p, conv=p, best=p, info=ip):
        return L.tslam_tour_open(n, cost, R, 0, mp, tours, cost2, passes, conv, best, info, None)

    for k in ("cost", "tours", "cost2", "passes", "conv", "best", "info"):
        assert call(**{k: None}) == capi.E_INVALID, k
    for n in (0, -1, 1025, 1 << 30):
        assert call(n=n) == capi.E_INVALID, n
    for R in (0, -1, 4097):
        assert call(R=R) == capi.E_INVALID, R
    assert call(mp=-1) == capi.E_INVALID
    assert b"max_passes" in L.tslam_last_error()
    assert info2.tolist() == [0, 0]  # nothing written on a refusal
