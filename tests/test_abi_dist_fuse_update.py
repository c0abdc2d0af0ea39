"""Argument checks of the tiled incremental fusion entries (tslam_tsdf_fuse_update_tiled_*) that need no GPU: a bad
tolerance, NULL handles or buffers, dst == src and a bad tiling are refused before a handle is looked at; a phase
called on a map with no update in progress is refused; the entries are declared and the ABI version is unchanged."""
import ctypes as C
import math

import numpy as np

from taichislam_b200 import _capi as capi

S = 16


def _fake():
    buf = (C.c_double * 64)()
    return buf, C.cast(buf, C.c_void_p)


def _plan(dst, src, tiles=(2, 1, 1), rank=0, world=2, tolerance=0.0, bufs=True):
    L = capi.load()
    plan = np.full(3, -7, np.int64)
    present = np.full(S, 7, np.uint8)
    t = None if tiles is None else (C.c_int32 * 3)(*tiles)
    rc = L.tslam_tsdf_fuse_update_tiled_plan(dst, src, t, rank, world, None, tolerance, 0, capi.np_ptr(plan) if bufs else None,
                                             capi.np_ptr(present) if bufs else None, None)
    return rc, L.tslam_last_error().decode(), plan, present


def _untouched(plan, present):
    return np.all(plan == -7) and np.all(present == 7)


def test_bad_tolerance_is_refused_first():
    b1, p1 = _fake()
    b2, p2 = _fake()
    for tol in (math.nan, math.inf, -1e-6):
        for dst, src in ((None, None), (p1, p2), (p1, p1)):
            rc, msg, plan, present = _plan(dst, src, tolerance=tol)
            assert rc == capi.E_INVALID and "tolerance" in msg
            assert _untouched(plan, present)


def test_null_handles_buffers_and_self_fusion_are_refused():
    b, p = _fake()
    b2, p2 = _fake()
    for dst, src in ((None, None), (p, None), (None, p)):
        rc, msg, plan, present = _plan(dst, src)
        assert rc == capi.E_INVALID and "NULL handle" in msg and _untouched(plan, present)
    rc, msg, plan, present = _plan(p, p)
    assert rc == capi.E_INVALID and "dst == src" in msg
    rc, msg, _, _ = _plan(p, p2, bufs=False)
    assert rc == capi.E_INVALID and "NULL plan3 or present" in msg


def test_bad_tilings_are_refused_before_the_handles():
    b1, p1 = _fake()
    b2, p2 = _fake()
    for tiles, rank, world in ((None, 0, 2), ((2, 1, 1), 2, 2), ((2, 1, 1), -1, 2), ((2, 2, 1), 0, 2), ((0, 1, 1), 0, 0),
                               ((17, 1, 1), 0, 17), ((5, 5, 1), 0, 25), ((1, 1, 1), 0, 0)):
        rc, msg, plan, present = _plan(p1, p2, tiles, rank, world)
        assert rc == capi.E_INVALID and "bad tiling" in msg, (tiles, rank, world, msg)
        assert _untouched(plan, present)
    L = capi.load()
    cnt = np.zeros(2, np.int32)
    rc = L.tslam_tsdf_fuse_update_tiled_pack(p1, None, 0, 2, capi.np_ptr(cnt), 0, None, None)
    assert rc == capi.E_INVALID and "bad tiling" in L.tslam_last_error().decode()


def test_later_phases_refuse_null_arguments():
    b, p = _fake()
    L = capi.load()
    t = (C.c_int32 * 3)(2, 1, 1)
    cnt = np.zeros(2, np.int32)
    st = np.full(8, -7, np.int64)
    assert L.tslam_tsdf_fuse_update_tiled_splat(None, p, 0, None) == capi.E_INVALID
    assert L.tslam_tsdf_fuse_update_tiled_splat(p, None, 0, None) == capi.E_INVALID
    assert L.tslam_tsdf_fuse_update_tiled_pack(None, t, 0, 2, capi.np_ptr(cnt), 0, None, None) == capi.E_INVALID
    assert L.tslam_tsdf_fuse_update_tiled_pack(p, t, 0, 2, None, 0, None, None) == capi.E_INVALID
    assert L.tslam_tsdf_fuse_update_tiled_pack(p, t, 0, 2, capi.np_ptr(cnt), -1, None, None) == capi.E_INVALID
    assert L.tslam_tsdf_fuse_update_tiled_pack(p, t, 0, 2, capi.np_ptr(cnt), 4, None, None) == capi.E_INVALID  # cap without rows
    assert L.tslam_tsdf_fuse_update_tiled_unpack(None, 0, None, None) == capi.E_INVALID
    assert L.tslam_tsdf_fuse_update_tiled_unpack(p, -1, None, None) == capi.E_INVALID
    assert L.tslam_tsdf_fuse_update_tiled_unpack(p, 3, None, None) == capi.E_INVALID
    assert L.tslam_tsdf_fuse_update_tiled_finish(None, p, 1, capi.np_ptr(st), None) == capi.E_INVALID
    assert L.tslam_tsdf_fuse_update_tiled_finish(p, None, 1, capi.np_ptr(st), None) == capi.E_INVALID
    assert np.all(st == -7)


def test_entries_are_declared_and_abi_version_is_unchanged():
    for phase in ("plan", "splat", "pack", "unpack", "finish"):
        assert f"tslam_tsdf_fuse_update_tiled_{phase}" in capi.SIGNATURES
        assert f"tslam_tsdf_fuse_update_tiled_{phase}" in open(capi.os.path.join(capi._HERE, "..", "include", "tslam.h")).read()
    assert capi.load().tslam_abi_version() == 6 and capi.ABI_VERSION == 6          # additive entry points
    assert capi.TILED_FUSE_REASONS[:7] == capi.FUSE_REASONS and len(capi.TILED_FUSE_REASONS) == 9
