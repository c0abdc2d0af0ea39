"""Argument checks of tslam_tsdf_reclaim and tslam_tsdf_block_keys that need no GPU: bad rules, a bad sphere and a
NULL handle are refused before the handle is looked at, with nothing written; the ABI version is unchanged."""
import ctypes as C
import math

import numpy as np

from taichislam_b200 import _capi as capi


def _fake():
    buf = (C.c_double * 64)()
    return buf, C.cast(buf, C.c_void_p)


def _reclaim(m, rules, center=(0.0, 0.0, 0.0), radius=1.0):
    L = capi.load()
    st = np.full(6, -7, np.int64)
    c = None if center is None else np.ascontiguousarray(np.asarray(center, np.float64))
    rc = L.tslam_tsdf_reclaim(m, rules, None, capi.np_ptr(c) if c is not None else None, float(radius), capi.np_ptr(st), None)
    return rc, L.tslam_last_error().decode(), st


def test_bad_rules_are_refused_first():
    b, p = _fake()
    for m in (None, p):
        for rules in (0, 8, 16, 1 | 8, -1, 1 << 30):
            rc, msg, st = _reclaim(m, rules)
            assert rc == capi.E_INVALID and "rules" in msg, (m, rules)
            assert np.all(st == -7)


def test_bad_sphere_is_refused_before_the_handle():
    b, p = _fake()
    for m in (None, p):
        for rules in (capi.RECLAIM_OUTSIDE, capi.RECLAIM_OUTSIDE | capi.RECLAIM_EMPTY, 7):
            for r in (math.nan, math.inf, -math.inf, -1e-9, -1.0):
                rc, msg, st = _reclaim(m, rules, radius=r)
                assert rc == capi.E_INVALID and "radius" in msg, (m, rules, r)
                assert np.all(st == -7)
            rc, msg, st = _reclaim(m, rules, center=None)
            assert rc == capi.E_INVALID and "centre" in msg
            assert np.all(st == -7)
            for c in ((math.nan, 0.0, 0.0), (0.0, math.inf, 0.0), (0.0, 0.0, -math.inf)):
                rc, msg, st = _reclaim(m, rules, center=c)
                assert rc == capi.E_INVALID and "not finite" in msg, c
                assert np.all(st == -7)


def test_sphere_is_not_checked_without_outside():
    # EMPTY / ALL do not read centre or radius: the refusal that follows is the NULL handle
    for rules in (capi.RECLAIM_ALL, capi.RECLAIM_EMPTY, capi.RECLAIM_ALL | capi.RECLAIM_EMPTY):
        rc, msg, st = _reclaim(None, rules, center=None, radius=math.nan)
        assert rc == capi.E_INVALID and "NULL handle" in msg
        assert np.all(st == -7)


def test_null_handle_is_refused():
    rc, msg, st = _reclaim(None, capi.RECLAIM_OUTSIDE, center=(1.0, 2.0, 3.0), radius=0.0)
    assert rc == capi.E_INVALID and "NULL handle" in msg
    assert np.all(st == -7)


def test_block_keys_refuses_a_null_handle():
    L = capi.load()
    n = C.c_int64(-5)
    assert L.tslam_tsdf_block_keys(None, 0, None, C.byref(n), None) == capi.E_INVALID
    assert n.value == -5


def test_entries_are_declared_and_abi_version_is_unchanged():
    assert "tslam_tsdf_reclaim" in capi.SIGNATURES and "tslam_tsdf_block_keys" in capi.SIGNATURES
    assert capi.load().tslam_abi_version() == 6 and capi.ABI_VERSION == 6          # additive entry points
    assert (capi.RECLAIM_ALL, capi.RECLAIM_EMPTY, capi.RECLAIM_OUTSIDE) == (1, 2, 4)
