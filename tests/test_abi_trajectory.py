"""Argument checks of tslam_esdf_trajectory / tslam_octo_esdf_trajectory that need no GPU: every refusal comes before the
handle is looked at; the ABI version is unchanged."""
import ctypes as C
import math

import numpy as np
import pytest

from taichislam_b200 import _capi as capi

GOOD = dict(dt=0.5, v_max=2.0, a_max=2.0, w_smooth=1.0, w_collision=10.0, w_feasibility=1.0, w_unknown=100.0,
            clearance=0.2, g_tol=1e-6, max_iters=10, memory=4, samples=4, check_samples=8)


def _call(entry, n=(8,), ctrl=None, null=None, **kw):
    L = capi.load()
    prm = dict(GOOD, **kw)
    p = capi.TrajParams(*[prm[f] for f, _ in capi.TrajParams._fields_])
    nn = np.asarray(n, np.int32)
    q = np.zeros((max(int(nn.clip(0).sum()), 1), 3)) if ctrl is None else ctrl
    out = np.zeros_like(q)
    cost = np.zeros((max(len(nn), 1), 6))
    info = np.zeros((max(len(nn), 1), 7), np.int32)
    a = dict(n=capi.np_ptr(nn), q=capi.np_ptr(q), p=C.byref(p), out=capi.np_ptr(out), cost=capi.np_ptr(cost),
             info=capi.np_ptr(info))
    if null is not None:
        a[null] = None
    rc = getattr(L, entry)(None, 0, len(nn), a["n"], a["q"], a["p"], a["out"], a["cost"], a["info"], None)
    return rc, L.tslam_last_error().decode()


ENTRIES = ("tslam_esdf_trajectory", "tslam_octo_esdf_trajectory")


@pytest.mark.parametrize("entry", ENTRIES)
def test_refusals_before_the_handle(entry):
    cases = [
        (dict(n=()), "trajectories"), (dict(n=(8,) * 1025), "trajectories"),
        (dict(n=(3,)), "control points"), (dict(n=(1025,)), "control points"),
        (dict(samples=0), "samples"), (dict(samples=17), "samples"), (dict(check_samples=0), "check_samples"),
        (dict(check_samples=65), "check_samples"), (dict(memory=0), "memory"), (dict(memory=17), "memory"),
        (dict(dt=0.0), "dt"), (dict(dt=math.inf), "dt"), (dict(v_max=-1.0), "dt"), (dict(a_max=math.nan), "dt"),
        (dict(w_smooth=-1.0), "weights"), (dict(w_collision=math.inf), "weights"), (dict(w_feasibility=math.nan), "weights"),
        (dict(w_unknown=-0.5), "weights"), (dict(clearance=-0.1), "weights"), (dict(g_tol=math.nan), "weights"),
        (dict(max_iters=-1), "max_iters"),
    ]
    for kw, word in cases:
        rc, msg = _call(entry, **kw)
        assert rc == capi.E_INVALID, kw
        if word is not None:
            assert word in msg, (kw, msg)
    # sum N above 2^20: 1024 trajectories of 1024 points is exactly 2^20 and passes to the handle check
    rc, msg = _call(entry, n=(1024,) * 1024)
    assert rc == capi.E_INVALID and "NULL handle" in msg
    q = np.zeros((8, 3))
    q[5, 1] = math.nan
    rc, msg = _call(entry, ctrl=q)
    assert rc == capi.E_INVALID and "not finite" in msg
    for null in ("n", "q", "p", "out", "cost", "info"):
        rc, msg = _call(entry, null=null)
        assert rc == capi.E_INVALID and "NULL" in msg, null
    rc, msg = _call(entry)
    assert rc == capi.E_INVALID and "NULL handle" in msg


def test_abi_version_is_unchanged():
    assert capi.ABI_VERSION == 6 and capi.load().tslam_abi_version() == 6
