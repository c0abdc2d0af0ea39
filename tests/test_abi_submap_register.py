"""Argument checks of tslam_tsdf_register that need no GPU: the pair count and the parameters are refused before the
handles are looked at, then NULL handles and arrays."""
import ctypes as C
import math

from taichislam_b200 import _capi as capi


def _call(P=1, band=0.2, min_weight=0.0, huber=0.05, max_iters=20, min_points=100, null=None):
    L = capi.load()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    arrays = [p] * 12                       # A, B, ref, read, R0, T0, R, T, H, b, cost2, info5
    arrays[0] = arrays[1] = None            # no handle: every check below comes first
    if null is not None:
        arrays = [p] * 12
        arrays[null] = None
    A, B, ra, rb, R0, T0, R, T, H, b, c2, i5 = arrays
    rc = L.tslam_tsdf_register(A, B, P, ra, rb, R0, T0, band, min_weight, huber, max_iters, min_points, R, T, H, b, c2, i5, None)
    return rc, L.tslam_last_error().decode()


def test_pair_count_outside_range_is_refused():
    for P in (0, -1, capi.REG_MAX_PAIRS + 1):
        rc, msg = _call(P=P)
        assert rc == capi.E_INVALID and "n_pairs" in msg


def test_bad_parameters_are_refused():
    for kw in (dict(band=0.0), dict(band=-0.1), dict(band=math.inf), dict(band=math.nan), dict(huber=0.0), dict(huber=math.nan),
               dict(min_weight=math.inf), dict(min_weight=math.nan), dict(max_iters=-1), dict(min_points=-1)):
        rc, msg = _call(**kw)
        assert rc == capi.E_INVALID and "band and huber" in msg, kw


def test_null_handles_and_arrays_are_refused():
    rc, msg = _call()
    assert rc == capi.E_INVALID and "NULL" in msg
    for q in range(12):
        rc, msg = _call(null=q)
        assert rc == capi.E_INVALID and "NULL" in msg, q


def test_abi_version_is_unchanged():
    assert capi.load().tslam_abi_version() == 6                                  # an additive entry point
