"""Trajectories against an ESDF (tslam_esdf_trajectory / tslam_octo_esdf_trajectory, include/tslam.h; DESIGN.md
section 7, "Trajectories"): uniform cubic B-splines whose free control points are optimised on the GPU, and the numpy
helpers that make control points from a path and sample a curve."""
import ctypes as C

import numpy as np

from . import _capi as capi

# solver settings and their defaults (tslam_traj_params_t); clearance has no default
DEFAULTS = dict(dt=0.5, v_max=2.0, a_max=2.0, w_smooth=1.0, w_collision=100.0, w_feasibility=1.0, w_unknown=1000.0,
                g_tol=1e-6, max_iters=200, memory=8, samples=4, check_samples=16)


def control_points(path, spacing):
    """Control points of a uniform B-spline along a polyline f[n,3] (e.g. a travel_path result): the polyline resampled
    by arc length at `spacing` (the last point always kept), each end point repeated so that the first and the last
    three control points are equal (zero velocity and acceleration at both ends) -> f64[m,3], m >= 6."""
    p = np.asarray(path, np.float64).reshape(-1, 3)
    if p.shape[0] == 0:
        raise ValueError("control_points needs at least one path point")
    if not (np.isfinite(spacing) and spacing > 0):
        raise ValueError("spacing must be finite and > 0")
    seg = np.linalg.norm(np.diff(p, axis=0), axis=1)
    s = np.concatenate([[0.0], np.cumsum(seg)])
    L = float(s[-1])
    n = max(int(np.ceil(L / spacing)), 1)
    t = np.linspace(0.0, L, n + 1)
    if L > 0:
        keep = np.concatenate([[True], seg > 0])
        q = np.stack([np.interp(t, s[keep], p[keep, a]) for a in range(3)], 1)
    else:
        q = p[:1].repeat(n + 1, 0)
    return np.concatenate([q[:1], q[:1], q, q[-1:], q[-1:]], 0)


def sample(ctrl, dt, per_span):
    """Positions, velocities and accelerations f64[(N-3) per_span + 1, 3] of the B-spline with control points ctrl
    f[N,3] and knot span dt, at u = k / per_span on every span plus u = 1 on the last."""
    Q = np.asarray(ctrl, np.float64).reshape(-1, 3)
    nsp = Q.shape[0] - 3
    if nsp < 1:
        raise ValueError("a cubic B-spline needs at least 4 control points")
    u = np.arange(per_span) / per_span
    j = np.repeat(np.arange(nsp), per_span)
    u = np.tile(u, nsp)
    j, u = np.append(j, nsp - 1), np.append(u, 1.0)
    w = 1.0 - u
    B = np.stack([w ** 3, 3 * u ** 3 - 6 * u ** 2 + 4, -3 * u ** 3 + 3 * u ** 2 + 3 * u + 1, u ** 3], 1) / 6.0
    dB = np.stack([-w ** 2, 3 * u ** 2 - 4 * u, -3 * u ** 2 + 2 * u + 1, u ** 2], 1) / 2.0 / dt
    ddB = np.stack([w, 3 * u - 2, -3 * u + 1, u], 1) / dt ** 2
    Qs = np.stack([Q[j + o] for o in range(4)], 1)
    return tuple(np.einsum("no,noa->na", b, Qs) for b in (B, dB, ddB))


def solve(fn, handle, submap, ctrls, clearance, **kw):
    """Pack the trajectories for tslam_*esdf_trajectory `fn`, call it, unpack: a list of dicts, one per trajectory,
    ctrl f64[N,3], J_s, J_c, J_f, J_u (at the result), J_in, iterations, evaluations, status, and the dense check at the
    result: min_dist (inf when no sample is valid), min_at (span, k) or None, invalid, close, ok (all valid, min_dist >=
    clearance)."""
    unknown = set(kw) - set(DEFAULTS)
    if unknown:
        raise TypeError(f"unknown trajectory settings: {sorted(unknown)}")
    prm = dict(DEFAULTS, **kw)
    qs = [np.ascontiguousarray(np.asarray(q, np.float64).reshape(-1, 3)) for q in ctrls]
    T = len(qs)
    n = np.array([q.shape[0] for q in qs], np.int32)
    q_in = np.ascontiguousarray(np.concatenate(qs, 0) if T else np.zeros((0, 3)))
    q_out = np.zeros_like(q_in)
    cost = np.zeros((max(T, 1), 6))
    info = np.zeros((max(T, 1), 7), np.int32)
    p = capi.TrajParams(float(prm["dt"]), float(prm["v_max"]), float(prm["a_max"]), float(prm["w_smooth"]),
                        float(prm["w_collision"]), float(prm["w_feasibility"]), float(prm["w_unknown"]), float(clearance),
                        float(prm["g_tol"]), int(prm["max_iters"]), int(prm["memory"]), int(prm["samples"]),
                        int(prm["check_samples"]))
    capi.check(fn(handle, int(submap), T, capi.np_ptr(n), capi.np_ptr(q_in), C.byref(p), capi.np_ptr(q_out), capi.np_ptr(cost),
                  capi.np_ptr(info), capi.stream_ptr()))
    out, o = [], 0
    for t in range(T):
        c, f = cost[t], info[t]
        md = float(c[5])
        out.append(dict(ctrl=q_out[o:o + n[t]].copy(), J_s=float(c[0]), J_c=float(c[1]), J_f=float(c[2]), J_u=float(c[3]),
                        J_in=float(c[4]), iterations=int(f[0]), evaluations=int(f[1]), status=int(f[2]), min_dist=md,
                        min_at=(int(f[5]), int(f[6])) if f[5] >= 0 else None, invalid=int(f[3]), close=int(f[4]),
                        ok=bool(f[3] == 0 and md >= float(clearance))))
        o += int(n[t])
    return out
