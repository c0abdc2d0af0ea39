"""Argument checks of tslam_octo_fuse_update that need no GPU: a tolerance that is not finite or negative is refused
first, then a NULL handle, then dst == src, all before either handle is looked at; the ABI version is unchanged."""
import ctypes as C
import math

import numpy as np

from taichislam_b200 import _capi as capi


def _update(dst, src, tolerance=0.0, full=0):
    L = capi.load()
    st = np.full(8, -7, np.int64)
    rc = L.tslam_octo_fuse_update(dst, src, None, tolerance, full, capi.np_ptr(st), None)
    return rc, L.tslam_last_error().decode(), st


def _fake():
    buf = (C.c_double * 64)()
    return buf, C.cast(buf, C.c_void_p)


def test_bad_tolerance_is_refused_first():
    b1, p1 = _fake()
    b2, p2 = _fake()
    for tol in (math.nan, math.inf, -math.inf, -1e-6, -1.0):
        for dst, src in ((None, None), (p1, None), (p1, p2), (p1, p1)):
            rc, msg, st = _update(dst, src, tolerance=tol)
            assert rc == capi.E_INVALID and "tolerance" in msg, (tol, dst, src)
            assert np.all(st == -7)


def test_null_handles_are_refused_before_dst_equals_src():
    b, p = _fake()
    for dst, src in ((None, None), (p, None), (None, p)):
        rc, msg, st = _update(dst, src)
        assert rc == capi.E_INVALID and "NULL handle" in msg
        assert np.all(st == -7)


def test_fusing_a_map_into_itself_is_refused():
    b, p = _fake()
    rc, msg, st = _update(p, p, full=1)
    assert rc == capi.E_INVALID and "dst == src" in msg
    assert np.all(st == -7)


def test_entry_is_declared_and_abi_version_is_unchanged():
    assert capi.SIGNATURES["tslam_octo_fuse_update"][1] == capi.SIGNATURES["tslam_tsdf_fuse_update"][1]
    assert capi.load().tslam_abi_version() == 6 and capi.ABI_VERSION == 6
