"""numpy f64 statement of the trajectory solver: tslam_esdf_trajectory / tslam_octo_esdf_trajectory (csrc/tslam_traj.cuh).

This is the definition the kernel is held to, bit for bit.  The library builds with -fmad=false, so every f64 step below
is one correctly rounded operation in the kernel's order; numpy's elementwise f64 arithmetic rounds the same way.

The field is a callable `field(x)`: f32[n,3] points -> (d f32[n], g f32[n,3], valid bool[n]), what the ESDF query
returns at those points.  On the GPU tests it is the library's own esdf_query (the kernel reads the field through the
same per-point function), on the CPU tests an analytic field or tests/esdf_query_reference.py.  Each evaluation makes
one call with all its samples, so `solve` is also the host-driven form of the solver.

Trajectory: control points Q f64[N,3], knot span dt; spans j = 0 .. N-4 use Q_j .. Q_{j+3}; Q_0..2 and Q_{N-3..N-1}
are fixed, the free variables are the coordinates of Q_3 .. Q_{N-4} in index order e = 3 i + axis (flat index of Q).

Basis rows for n samples per span, u = k/n, k = 0 .. n (row n: u = 1):
    w = 1 - u, u2 = u u, u3 = u2 u
    b0 = ((w w) w)/6   b1 = ((3 u3 - 6 u2) + 4)/6   b2 = (((-3 u3 + 3 u2) + 3 u) + 1)/6   b3 = u3/6
Samples: rows 0 .. n-1 on every span, row n on the last; position f32(((b0 Q_j + b1 Q_{j+1}) + b2 Q_{j+2}) + b3 Q_{j+3}).

Sums ("tsum"): with P = 256 threads, thread t adds its items t, t + P, ... in item order to a partial starting at 0;
the partials are added by the halving tree p[i] += p[i + s], s = P/2 .. 1.  Item lists:
    J_s   jerk terms i = 0 .. N-4: |jerk_i|^2, jerk_i = ((Q_{i+3} - 3 Q_{i+2}) + 3 Q_{i+1}) - Q_i, |v|^2 = (x x + y y) + z z
    J_c   spans j; within a span its samples in order, each (c - d)^2 when valid and d < c (else nothing)
    J_u   spans j; +1 per invalid sample (an exact count)
    J_f   velocity terms i = 0 .. N-2, then acceleration terms i = 0 .. N-3, into the same partial: max(0, h)^2 with
          h = |V_i|^2 - v^2, V_i = (Q_{i+1} - Q_i)/dt;  h = |A_i|^2 - a^2, A_i = ((Q_{i+2} - 2 Q_{i+1}) + Q_i)/dt2, dt2 = dt dt
    dots  free coordinates e, items a_e b_e
J = ((w_s J_s + w_c J_c) + w_f J_f) + w_u J_u.  The gradient is given in csrc/tslam_traj.cuh and restated in `evaluate`.
"""
import numpy as np

P = 256            # threads per CTA (TJ_THREADS)
TRIALS = 30
C1 = 1e-4
CURV = 1e-10
MAX_N, MAX_T, MAX_SUM_N, MAX_K, MAX_C, MAX_M = 1024, 1024, 1 << 20, 16, 64, 16

DEFAULTS = dict(dt=0.5, v_max=2.0, a_max=2.0, w_smooth=1.0, w_collision=100.0, w_feasibility=1.0, w_unknown=1000.0,
                clearance=0.2, g_tol=1e-6, max_iters=200, memory=8, samples=4, check_samples=16)


def basis(n):
    """f64[n+1, 4] basis rows."""
    b = np.zeros((n + 1, 4))
    for k in range(n + 1):
        u = float(k) / float(n)
        w = 1.0 - u
        u2 = u * u
        u3 = u2 * u
        b[k] = (((w * w) * w) / 6.0, ((3.0 * u3 - 6.0 * u2) + 4.0) / 6.0, (((-3.0 * u3 + 3.0 * u2) + 3.0 * u) + 1.0) / 6.0,
                u3 / 6.0)
    return b


def thread_partials(items):
    """Per-thread partials of tsum: items f64[n] (or [n, w]: a row per item, w values of that item added in order)."""
    a = np.asarray(items, np.float64)
    if a.ndim == 1:
        a = a[:, None]
    n, w = a.shape
    rows = -(-n // P)
    pad = np.zeros((rows * P, w))
    pad[:n] = a
    pad = pad.reshape(rows, P, w)
    p = np.zeros(P)
    for r in range(rows):
        for c in range(w):
            p = p + pad[r, :, c]  # + 0.0 on padding: exact
    return p


def tree(p):
    p = np.array(p, np.float64)
    s = P // 2
    while s >= 1:
        p[:s] = p[:s] + p[s:2 * s]
        s //= 2
    return float(p[0])


def tsum(items):
    return tree(thread_partials(items))


def tsum_lists(*lists):
    """One partial fed by several item lists in turn (J_f: velocity items, then acceleration items)."""
    p = np.zeros(P)
    for items in lists:
        a = np.asarray(items, np.float64)
        n = a.shape[0]
        rows = -(-n // P)
        pad = np.zeros(rows * P)
        pad[:n] = a
        for r in range(rows):
            p = p + pad[r * P:(r + 1) * P]
    return tree(p)


def positions(Q, b):
    """f64 positions f[nsp, n+1, 3] of every basis row on every span (row n used on the last span only)."""
    nsp = Q.shape[0] - 3
    q0, q1, q2, q3 = (Q[o:o + nsp][:, None, :] for o in range(4))
    b = b[None, :, :, None]
    return ((b[..., 0, :] * q0 + b[..., 1, :] * q1) + b[..., 2, :] * q2) + b[..., 3, :] * q3


def sample_mask(nsp, n):
    m = np.zeros((nsp, n + 1), bool)
    m[:, :n] = True
    m[-1, n] = True
    return m


def _jerk(Q):
    return ((Q[3:] - 3.0 * Q[2:-1]) + 3.0 * Q[1:-2]) - Q[:-3]


def _sq3(v):
    return (v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1]) + v[..., 2] * v[..., 2]


def evaluate(Q, field, prm, bk):
    """-> (J, (J_s, J_c, J_f, J_u), G f64[N,3] (zero outside the free control points), field calls)."""
    N = Q.shape[0]
    nsp, K = N - 3, prm["samples"]
    c = float(prm["clearance"])
    dt = float(prm["dt"])
    dt2 = dt * dt
    v2, a2 = float(prm["v_max"]) * float(prm["v_max"]), float(prm["a_max"]) * float(prm["a_max"])
    x = positions(Q, bk).astype(np.float32)                   # [nsp, K+1, 3]
    mask = sample_mask(nsp, K)
    d, g, ok = field(x[mask])
    D = np.zeros((nsp, K + 1), np.float32)
    Gf = np.zeros((nsp, K + 1, 3), np.float32)
    V = np.zeros((nsp, K + 1), bool)
    D[mask], Gf[mask], V[mask] = d, g, ok
    D64 = D.astype(np.float64)
    close = V & (D64 < c)
    r = np.where(close, c - D64, 0.0)
    Jc = tsum(np.where(close, r * r, 0.0))                    # items = spans, each its samples in order
    Ju = tsum((mask & ~V).astype(np.float64))
    jerk = _jerk(Q)
    Js = tsum(_sq3(jerk))
    vel = (Q[1:] - Q[:-1]) / dt
    acc = ((Q[2:] - 2.0 * Q[1:-1]) + Q[:-2]) / dt2
    hv = _sq3(vel) - v2
    ha = _sq3(acc) - a2
    Jf = tsum_lists(np.where(hv > 0.0, hv * hv, 0.0), np.where(ha > 0.0, ha * ha, 0.0))
    J = ((prm["w_smooth"] * Js + prm["w_collision"] * Jc) + prm["w_feasibility"] * Jf) + prm["w_unknown"] * Ju
    # span terms cs[j, o, axis]: sum over the span's close samples in order of (-2 r b_o) g_axis
    cs = np.zeros((nsp, 4, 3))
    for k in range(K + 1):
        m = -2.0 * r[:, k]
        for o in range(4):
            t = (m * bk[k, o])[:, None] * Gf[:, k, :].astype(np.float64)
            cs[:, o, :] = cs[:, o, :] + np.where(close[:, k, None], t, 0.0)
    G = np.zeros((N, 3))
    if N >= 7:
        i = np.arange(3, N - 3)
        gs = np.zeros((i.size, 3))
        for m_off, cj in zip((3, 2, 1, 0), (1.0, -3.0, 3.0, -1.0)):   # m = i-3 .. i; Q_i's coefficient in jerk_m
            gs = gs + (2.0 * jerk[i - m_off]) * cj
        gc = np.zeros((i.size, 3))
        for j_off in (3, 2, 1, 0):
            gc = gc + cs[i - j_off, j_off, :]
        gf = np.zeros((i.size, 3))
        for m_off in (1, 0):                                          # m = i-1, i
            m = i - m_off
            h = hv[m][:, None]
            t = (4.0 * h) * vel[m]
            t = -t if m_off == 0 else t
            gf = gf + np.where(h > 0.0, t / dt, 0.0)
        for m_off in (2, 1, 0):                                       # m = i-2 .. i
            m = i - m_off
            h = ha[m][:, None]
            t = (4.0 * h) * acc[m]
            t = -2.0 * t if m_off == 1 else t
            gf = gf + np.where(h > 0.0, t / dt2, 0.0)
        G[3:N - 3] = (prm["w_smooth"] * gs + prm["w_collision"] * gc) + prm["w_feasibility"] * gf
    return J, (Js, Jc, Jf, Ju), G


def check(Q, field, prm):
    """Dense check -> (min d (inf when no valid sample), n_invalid, n_close, span, k)."""
    C = prm["check_samples"]
    nsp = Q.shape[0] - 3
    x = positions(Q, basis(C)).astype(np.float32)
    mask = sample_mask(nsp, C)
    d, _, ok = field(x[mask])
    js, ks = np.nonzero(mask)
    n_inv = int((~ok).sum())
    n_close = int((ok & (d.astype(np.float64) < float(prm["clearance"]))).sum())
    if not ok.any():
        return np.inf, n_inv, n_close, -1, -1
    dv = np.where(ok, d, np.float32(np.inf))
    q = int(np.argmin(dv))                                            # first minimum: lowest (span, k)
    return float(dv[q]), n_inv, n_close, int(js[q]), int(ks[q])


def free(a):
    return a[3:-3].ravel()


def dot(a, b):
    return tsum(free(a) * free(b))


def solve(Q, field, vs, **kw):
    """One trajectory -> dict(ctrl, cost (J_s, J_c, J_f, J_u, J_in, min_d), info (iters, evals, status, n_invalid,
    n_close, span, k)).  vs: the field's voxel size (f32 value)."""
    prm = dict(DEFAULTS)
    prm.update(kw)
    Q = np.array(Q, np.float64).reshape(-1, 3)
    N, M = Q.shape[0], int(prm["memory"])
    bk = basis(int(prm["samples"]))
    vs = float(np.float32(vs))
    J, J4, G = evaluate(Q, field, prm, bk)
    J_in, iters, evals, status = J, 0, 1, 3
    hist = []          # (s, y, rho), oldest first
    gamma = 1.0
    while N >= 7:
        gi = float(np.max(np.abs(free(G))))
        if gi <= prm["g_tol"]:
            status = 1
            break
        if iters >= prm["max_iters"]:
            status = 0
            break
        steep = not hist
        gd = 0.0
        if not steep:
            D = G.copy()
            al = []
            for s, y, rho in reversed(hist):
                a = rho * dot(s, D)
                al.append(a)
                D[3:N - 3] = D[3:N - 3] - a * y[3:N - 3]
            D[3:N - 3] = gamma * D[3:N - 3]
            for (s, y, rho), a in zip(hist, reversed(al)):
                b = rho * dot(y, D)
                D[3:N - 3] = D[3:N - 3] + (a - b) * s[3:N - 3]
            D = -D
            gd = dot(G, D)
            if not gd < 0.0:
                steep = True
                hist = []
        if steep:
            sc = vs / gi
            D = -(G * sc)
            gd = dot(G, D)
        alpha, ok = 1.0, False
        for _ in range(TRIALS):
            X = Q.copy()
            X[3:N - 3] = Q[3:N - 3] + alpha * D[3:N - 3]
            Jt, J4t, Gt = evaluate(X, field, prm, bk)
            evals += 1
            if Jt <= J + (C1 * alpha) * gd:
                ok = True
                break
            alpha *= 0.5
        if not ok:
            status = 2
            break
        s, y = X - Q, Gt - G
        sy, yy = tsum(free(s) * free(y)), tsum(free(y) * free(y))
        if sy > CURV * yy:
            hist.append((s, y, 1.0 / sy))
            if len(hist) > M:
                hist.pop(0)
            gamma = sy / yy
        Q, G, J, J4 = X, Gt, Jt, J4t
        iters += 1
    md, n_inv, n_close, js, ks = check(Q, field, prm)
    return dict(ctrl=Q, cost=np.array([J4[0], J4[1], J4[2], J4[3], J_in, md]),
                info=np.array([iters, evals, status, n_inv, n_close, js, ks], np.int64))


def solve_many(ctrls, field, vs, **kw):
    """Each trajectory alone (the kernel's results depend on nothing else in the call)."""
    return [solve(q, field, vs, **kw) for q in ctrls]
