"""Argument checks of tslam_tsdf_track_depth / tslam_tsdf_track_points that need no GPU: the frame count and the
parameters are refused before the handle is looked at, then NULL handles and arrays."""
import ctypes as C
import math

from taichislam_b200 import _capi as capi


def _depth(n=1, h=48, w=64, step=2, huber=0.05, max_iters=20, min_points=100, mem=capi.MEM_HOST, null=None):
    L = capi.load()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    arrays = [p] * 10                       # handle, depth, R0, T0, R, T, H, b, cost2, info5
    arrays[0] = None                        # no handle: every check below comes first
    if null is not None:
        arrays = [p] * 10
        arrays[null] = None
    m, d, R0, T0, R, T, H, b, c2, i5 = arrays
    rc = L.tslam_tsdf_track_depth(m, d, mem, n, h, w, None, R0, T0, step, huber, max_iters, min_points, R, T, H, b, c2, i5, None)
    return rc, L.tslam_last_error().decode()


def _points(n=10, huber=0.05, max_iters=20, min_points=100, null=None):
    L = capi.load()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    arrays = [p] * 10                       # handle, xyz, R0, T0, R, T, H, b, cost2, info5
    arrays[0] = None
    if null is not None:
        arrays = [p] * 10
        arrays[null] = None
    m, x, R0, T0, R, T, H, b, c2, i5 = arrays
    rc = L.tslam_tsdf_track_points(m, x, capi.MEM_HOST, n, 0, R0, T0, huber, max_iters, min_points, R, T, H, b, c2, i5, None)
    return rc, L.tslam_last_error().decode()


def test_frame_count_outside_range_is_refused():
    for n in (0, -1, capi.REG_MAX_PAIRS + 1):
        rc, msg = _depth(n=n)
        assert rc == capi.E_INVALID and "outside" in msg, n


def test_bad_parameters_are_refused():
    for kw in (dict(step=0), dict(step=-2), dict(h=0), dict(w=-1), dict(huber=0.0), dict(huber=-0.05), dict(huber=math.inf),
               dict(huber=math.nan), dict(max_iters=-1), dict(min_points=-1), dict(mem=7)):
        rc, msg = _depth(**kw)
        assert rc == capi.E_INVALID and "step >= 1" in msg, kw
    for kw in (dict(n=-1), dict(huber=0.0), dict(huber=math.nan), dict(max_iters=-1), dict(min_points=-1)):
        rc, msg = _points(**kw)
        assert rc == capi.E_INVALID and "n_points >= 0" in msg, kw


def test_null_handles_and_arrays_are_refused():
    for call in (_depth, _points):
        rc, msg = call()
        assert rc == capi.E_INVALID and "NULL" in msg
        for q in range(10):
            rc, msg = call(null=q)
            assert rc == capi.E_INVALID and "NULL" in msg, (call.__name__, q)


def test_abi_version_is_unchanged():
    assert capi.load().tslam_abi_version() == 6                                  # additive entry points
