"""Argument checks of tslam_tsdf_place_describe and tslam_place_match that need no GPU: counts, parameters, the levelled
rotations, top_k, min_gap, NULL arrays and query indices are refused before a handle or a descriptor is looked at."""
import ctypes as C
import math

import numpy as np
import pytest

from taichislam_b200 import _capi as capi
from taichislam_b200 import place


def _describe(n=1, r_max=8.0, h_min=0.3, band=0.2, min_weight=0.0, M=None, null=None, submaps=None):
    L = capi.load()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    sm = np.zeros(max(n, 1), np.int32) if submaps is None else np.asarray(submaps, np.int32)
    M9 = np.tile(np.eye(3, dtype=np.float32).reshape(9), max(n, 1)) if M is None else np.asarray(M, np.float32).reshape(-1)
    params = capi.PlaceParams(r_max, h_min, band, min_weight)
    args = [capi.np_ptr(sm), capi.np_ptr(M9), C.byref(params), p, p, p, p]  # submaps, M9, params, sc, ring, bev, n_points
    if null is not None:
        args[null] = None
    rc = L.tslam_tsdf_place_describe(None, n, *args, None)
    return rc, L.tslam_last_error().decode()


def test_describe_count_outside_range_is_refused():
    for n in (0, -1, 1025):
        rc, msg = _describe(n=n)
        assert rc == capi.E_INVALID and "outside [1, 1024]" in msg


def test_describe_bad_parameters_are_refused():
    for kw in (dict(r_max=0.0), dict(r_max=-1.0), dict(r_max=math.inf), dict(r_max=math.nan), dict(h_min=0.0), dict(h_min=math.nan),
               dict(band=0.0), dict(band=math.inf), dict(min_weight=math.nan), dict(min_weight=-math.inf)):
        rc, msg = _describe(**kw)
        assert rc == capi.E_INVALID and "finite" in msg, kw


def test_describe_non_finite_rotation_is_refused():
    M = np.eye(3).reshape(9).copy()
    M[4] = np.nan
    rc, msg = _describe(M=M)
    assert rc == capi.E_INVALID and "not finite" in msg


def test_describe_null_arrays_then_handle_are_refused():
    for k in range(7):
        rc, msg = _describe(null=k)
        assert rc == capi.E_INVALID and "NULL" in msg, k
    rc, msg = _describe()  # every argument good: the missing handle is named last
    assert rc == capi.E_INVALID and "NULL handle" in msg


def _match(n_db=4, n_q=1, queries=None, top_k=4, min_gap=0, null=None):
    L = capi.load()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    q = np.zeros(max(n_q, 1), np.int32) if queries is None else np.asarray(queries, np.int32)
    args = [p, p, p, p, p]  # sc, ring, bev, n_points, ids: device arrays, never read before the checks pass
    if null is not None and null < 5:
        args[null] = None
    qp = None if null == 5 else capi.np_ptr(q)
    outs = [p, p]
    if null is not None and null >= 6:
        outs[null - 6] = None
    rc = L.tslam_place_match(n_db, *args, n_q, qp, top_k, min_gap, 0, *outs, None)
    return rc, L.tslam_last_error().decode()


def test_match_refusals():
    for kw in (dict(n_db=0), dict(n_db=1025), dict(n_q=0), dict(n_q=1025), dict(top_k=0), dict(top_k=33), dict(min_gap=-1)):
        rc, _ = _match(**kw)
        assert rc == capi.E_INVALID, kw
    for k in range(8):
        rc, msg = _match(null=k)
        assert rc == capi.E_INVALID and "NULL" in msg, k
    for q in (-1, 4):
        rc, msg = _match(queries=[q])
        assert rc == capi.E_INVALID and "out of range" in msg, q


def test_top_k_limit_is_the_header_constant():
    assert capi.load().tslam_place_match is not None
    rc, _ = _match(top_k=32, null=0)  # 32 passes the range check and reaches the NULL check
    assert rc == capi.E_INVALID


def test_level_refuses_bad_up_and_is_minimal():
    for up in ((0.0, 0.0, 0.0), (math.nan, 0.0, 1.0), (0.0, math.inf, 0.0)):
        with pytest.raises(ValueError):
            place.level(up)
    assert np.array_equal(place.level((0.0, 0.0, 1.0)), np.eye(3))
    assert np.array_equal(place.level((0.0, 0.0, 2.0)), np.eye(3))
    for up in ((0.0, -1.0, 0.0), (1.0, 2.0, 0.5), (0.0, 0.0, -1.0), (0.3, 0.0, -1.0)):
        L = place.level(up)
        u = np.asarray(up) / np.linalg.norm(up)
        assert np.allclose(L @ u, [0.0, 0.0, 1.0], atol=1e-15) and np.allclose(L @ L.T, np.eye(3), atol=1e-15)
        assert np.isclose(np.linalg.det(L), 1.0)
        axis = np.cross(u, [0.0, 0.0, 1.0])
        if np.linalg.norm(axis) > 0:  # a rotation about u x z: the axis is fixed
            assert np.allclose(L @ axis, axis, atol=1e-15)
