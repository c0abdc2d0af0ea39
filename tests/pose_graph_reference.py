"""A numpy statement of tslam_pose_graph_solve (include/tslam.h; DESIGN.md section 7, "Pose-graph optimisation").

Nodes X_i = (R_i, t_i) map submap-local to world coordinates.  Edge k = (i, j, Z_k, Omega_k, c_k), Z_k maps i-local to
j-local.  Residual e_k = Log(X_j^-1 X_i Z_k^-1) in xi = (rho, phi); s_k = e_k^T Omega_k e_k; rho_k(s) = s (c_k = 0) or
c_k^2 log1p(s / c_k^2); F = 1/2 sum rho_k(s_k); w_k = rho_k'(s_k).  Left perturbation X_i <- exp(delta_i) X_i in the world
frame: J_i = Jl^-1(e_k) Ad(X_j^-1), J_j = -J_i.  Levenberg-Marquardt with the registration's schedule; here the damped
system is solved exactly (scipy.sparse), where the library runs preconditioned conjugate gradients.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

SMALL = 1e-2     # below this rotation angle every coefficient is its series (terms through theta^4)
CHUNK = 256      # F sums the edge terms in order within chunks of 256 edges, then the chunk sums in chunk order
MAX_N, MAX_E = 4096, 65536
CONVERGED, MAX_ITERS, NO_PROGRESS, NOT_PD = 0, 1, 2, 3


def hat(v):
    """[v]x for v [..., 3]."""
    v = np.asarray(v, np.float64)
    z = np.zeros(v.shape[:-1])
    return np.stack([np.stack([z, -v[..., 2], v[..., 1]], -1), np.stack([v[..., 2], z, -v[..., 0]], -1),
                     np.stack([-v[..., 1], v[..., 0], z], -1)], -2)


def _coeffs(th):
    """A = sin/th, B = (1 - cos)/th^2, C = (th - sin)/th^3, D = (1 - (th/2) cot(th/2))/th^2, c2 = (th^2 + 2 cos - 2)/(2 th^4),
    c3 = (2 th - 3 sin + th cos)/(2 th^5); series below SMALL."""
    th = np.asarray(th, np.float64)
    t2 = th * th
    t4 = t2 * t2
    s = th < SMALL
    tt = np.where(s, 1.0, th)
    sn, cs, h = np.sin(tt), np.cos(tt), np.sin(0.5 * tt)
    A = np.where(s, 1.0 - t2 / 6.0 + t4 / 120.0, sn / tt)
    B = np.where(s, 0.5 - t2 / 24.0 + t4 / 720.0, 2.0 * h * h / (tt * tt))
    C = np.where(s, 1.0 / 6.0 - t2 / 120.0 + t4 / 5040.0, (tt - sn) / (tt * tt * tt))
    D = np.where(s, 1.0 / 12.0 + t2 / 720.0 + t4 / 30240.0, (1.0 - 0.5 * tt * np.cos(0.5 * tt) / h) / (tt * tt))
    c2 = np.where(s, 1.0 / 24.0 - t2 / 720.0 + t4 / 40320.0, (tt * tt - 4.0 * h * h) / (2.0 * tt ** 4))
    c3 = np.where(s, 1.0 / 120.0 - t2 / 2520.0 + t4 / 120960.0, (2.0 * tt - 3.0 * sn + tt * cs) / (2.0 * tt ** 5))
    return A, B, C, D, c2, c3


def exp(xi):
    """Exp(xi) for xi [..., 6] = (rho, phi) -> (R, t): R = I + A K + B K^2, t = V rho, V = I + B K + C K^2."""
    xi = np.asarray(xi, np.float64)
    rho, phi = xi[..., :3], xi[..., 3:]
    A, B, C, _, _, _ = _coeffs(np.sqrt(np.sum(phi * phi, -1)))
    K = hat(phi)
    K2 = K @ K
    I = np.eye(3)
    R = I + A[..., None, None] * K + B[..., None, None] * K2
    V = I + B[..., None, None] * K + C[..., None, None] * K2
    return R, np.einsum("...ij,...j->...i", V, rho)


def update(R, t, xi):
    """exp(xi) (R, t): R' = Exp(phi) R, t' = Exp(phi) t + V(phi) rho (submap_register_reference.se3_update)."""
    E, v = exp(xi)
    return E @ R, np.einsum("...ij,...j->...i", E, t) + v


def log(R, t):
    """Log(R, t) -> xi [..., 6], the exact inverse of exp: theta = atan2(|w| / 2, (tr R - 1) / 2), w = vee(R - R^T);
    phi = theta w / (2 sin theta) (series below SMALL) for cos theta >= 0, else theta times the axis read from the
    symmetric part (R + R^T) / 2 - cos theta I = (1 - cos theta) u u^T, signed so that u . w >= 0; rho = V^-1 t."""
    R = np.asarray(R, np.float64)
    t = np.asarray(t, np.float64)
    w = np.stack([R[..., 2, 1] - R[..., 1, 2], R[..., 0, 2] - R[..., 2, 0], R[..., 1, 0] - R[..., 0, 1]], -1)
    c = 0.5 * (R[..., 0, 0] + R[..., 1, 1] + R[..., 2, 2] - 1.0)
    sn = 0.5 * np.sqrt(np.sum(w * w, -1))
    th = np.arctan2(sn, c)
    t2 = th * th
    small = th < SMALL
    f = np.where(small, 0.5 * (1.0 + t2 / 6.0 + 7.0 * t2 * t2 / 360.0), 0.5 * th / np.where(small | (sn == 0), 1.0, sn))
    phi = f[..., None] * w
    big = c < 0.0
    if np.any(big):
        Rb, cb, thb, wb = R[big], c[big], th[big], w[big]
        S = 0.5 * (Rb + np.swapaxes(Rb, -1, -2)) - cb[:, None, None] * np.eye(3)
        k = np.argmax(np.diagonal(S, 0, -2, -1), -1)
        n = np.arange(len(k))
        uk = np.sqrt(S[n, k, k] / (1.0 - cb))
        u = S[n, k, :] / ((1.0 - cb) * uk)[:, None]
        u[n, k] = uk
        sg = np.where(np.sum(u * wb, -1) < 0.0, -1.0, 1.0)
        phi[big] = (sg * thb)[:, None] * u
    _, _, _, D, _, _ = _coeffs(th)
    K = hat(phi)
    Vi = np.eye(3) - 0.5 * K + D[..., None, None] * (K @ K)
    return np.concatenate([np.einsum("...ij,...j->...i", Vi, t), phi], -1)


def jl_inv(xi):
    """The inverse left Jacobian of SE(3) at xi [..., 6]: [[Ji, -Ji Q Ji], [0, Ji]], Ji = I - K/2 + D K^2 the inverse
    left Jacobian of SO(3), Q Barfoot's Q(rho, phi)."""
    xi = np.asarray(xi, np.float64)
    rho, phi = xi[..., :3], xi[..., 3:]
    th = np.sqrt(np.sum(phi * phi, -1))
    _, _, C, D, c2, c3 = _coeffs(th)
    P, Rh = hat(phi), hat(rho)
    PR, RP, PP = P @ Rh, Rh @ P, P @ P
    PRP = PR @ P
    Q = (0.5 * Rh + C[..., None, None] * (PR + RP + PRP) + c2[..., None, None] * (P @ PR + RP @ P - 3.0 * PRP)
         + c3[..., None, None] * (PRP @ P + P @ PRP))
    Ji = np.eye(3) - 0.5 * P + D[..., None, None] * PP
    out = np.zeros(xi.shape[:-1] + (6, 6))
    out[..., :3, :3] = Ji
    out[..., 3:, 3:] = Ji
    out[..., :3, 3:] = -(Ji @ Q @ Ji)
    return out


def adjoint(R, t):
    """Ad(R, t) = [[R, [t]x R], [0, R]] for xi = (rho, phi)."""
    out = np.zeros(np.shape(R)[:-2] + (6, 6))
    out[..., :3, :3] = R
    out[..., 3:, 3:] = R
    out[..., :3, 3:] = hat(t) @ R
    return out


def sym_omega(om):
    """The symmetric 6x6 read from the upper triangle of om [..., 6, 6]."""
    U = np.triu(om)
    return U + np.swapaxes(np.triu(om, 1), -1, -2)


def residuals(R, T, ij, ZR, ZT):
    """e [E, 6] and J_i [E, 6, 6] (J_j = -J_i)."""
    i, j = ij[:, 0], ij[:, 1]
    Rj_t = np.swapaxes(R[j], -1, -2)
    RM = Rj_t @ R[i]
    tM = np.einsum("eab,eb->ea", Rj_t, T[i] - T[j])
    RE = RM @ np.swapaxes(ZR, -1, -2)
    tE = tM - np.einsum("eab,eb->ea", RE, ZT)
    e = log(RE, tE)
    J = jl_inv(e) @ adjoint(Rj_t, -np.einsum("eab,eb->ea", Rj_t, T[j]))
    return e, J


def seq_sum(x):
    """The sum of x in order, one rounding per addition."""
    x = np.asarray(x, np.float64)
    return float(np.cumsum(x)[-1]) if x.size else 0.0


def cost_terms(e, om, c):
    """s_k, w_k, rho_k(s_k)."""
    O = sym_omega(om)
    s = np.einsum("ea,eab,eb->e", e, O, e)
    c2 = np.where(c > 0, c * c, 1.0)
    rob = c > 0
    w = np.where(rob, 1.0 / (1.0 + s / c2), 1.0)
    rho = np.where(rob, c2 * np.log1p(s / c2), s)
    return s, w, rho


def total_cost(rho):
    """F = 1/2 (sum over chunks of CHUNK edges, in chunk order, of each chunk's sum in edge order)."""
    return 0.5 * seq_sum([seq_sum(rho[a:a + CHUNK]) for a in range(0, len(rho), CHUNK)])


def evaluate(R, T, ij, ZR, ZT, om, c):
    e, J = residuals(R, T, ij, ZR, ZT)
    s, w, rho = cost_terms(e, om, c)
    return dict(e=e, J=J, chi2=s, weight=w, F=total_cost(rho))


def normal_equations(R, T, ij, ZR, ZT, om, c, fixed):
    """(Dblk [nF,6,6], Off (scipy.sparse, the off-diagonal blocks), g [6 nF], free nodes, evaluation) of the IRLS
    linearisation over the free nodes (6 rows each, in node order).  A = blockdiag(Dblk) + Off."""
    ev = evaluate(R, T, ij, ZR, ZT, om, c)
    N = R.shape[0]
    free = np.flatnonzero(~fixed)
    fi = -np.ones(N, np.int64)
    fi[free] = np.arange(len(free))
    O = sym_omega(om)
    J = ev["J"]
    B = ev["weight"][:, None, None] * np.einsum("eba,ebc,ecd->ead", J, O, J)
    gv = ev["weight"][:, None] * np.einsum("eba,ebc,ec->ea", J, O, ev["e"])
    nF = len(free)
    a, b = fi[ij[:, 0]], fi[ij[:, 1]]
    D = np.zeros((nF, 6, 6))
    g = np.zeros((nF, 6))
    np.add.at(D, a[a >= 0], B[a >= 0])
    np.add.at(D, b[b >= 0], B[b >= 0])
    np.add.at(g, a[a >= 0], gv[a >= 0])
    np.add.at(g, b[b >= 0], -gv[b >= 0])
    both = (a >= 0) & (b >= 0)
    r6 = np.arange(6)
    rows, cols, vals = [], [], []
    for u, v in ((a[both], b[both]), (b[both], a[both])):
        rows.append((6 * u[:, None, None] + r6[None, :, None] + 0 * r6[None, None, :]).ravel())
        cols.append((6 * v[:, None, None] + 0 * r6[None, :, None] + r6[None, None, :]).ravel())
        vals.append((-B[both]).ravel())
    Off = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * nF, 6 * nF))
    return D, Off, g.ravel(), free, ev


def dense_A(D, Off):
    """The assembled A as a dense array (small graphs only)."""
    return sp.block_diag(list(D)).toarray() + Off.toarray() if len(D) else np.zeros((0, 0))


def damped_step(D, Off, g, lam):
    """Solve (A + lam diag(max(A_ii, 1e-9 max_j A_jj))) d = -g exactly; None when a damped 6x6 diagonal block is not
    positive definite (the library's preconditioner test)."""
    dg = np.diagonal(D, 0, 1, 2)
    Dd = D.copy()
    Dd[:, r6, r6] += lam * np.maximum(dg, 1e-9 * dg.max())
    try:
        np.linalg.cholesky(Dd)
    except np.linalg.LinAlgError:
        return None
    M = sp.block_diag([sp.csr_matrix(b) for b in Dd], format="csr") + Off
    return spla.spsolve(M.tocsc(), -g)


r6 = np.arange(6)


def apply_step(R, T, free, d):
    R2, T2 = R.copy(), T.copy()
    xi = d.reshape(-1, 6)
    R2[free], T2[free] = update(R[free], T[free], xi)
    return R2, T2


def solve(R, T, fixed, ij, ZR, ZT, om, c, max_iters=100, eps_t=1e-6, eps_r=1e-8, **_):
    """The contract's LM with exact linear steps -> dict(R, T, chi2, weight, F0, F, evaluations, accepted, converged,
    status)."""
    R, T = np.array(R, np.float64), np.array(T, np.float64)
    fixed = np.asarray(fixed, bool)
    ij = np.asarray(ij, np.int64)
    c = np.asarray(c, np.float64)
    D, Off, g, free, ev = normal_equations(R, T, ij, ZR, ZT, om, c, fixed)
    F0 = F = ev["F"]
    lam, evals, acc, status = 1e-4, 0, 0, MAX_ITERS
    while evals < max_iters:
        d = damped_step(D, Off, g, lam)
        evals += 1
        if d is None:
            status = NOT_PD
            break
        R2, T2 = apply_step(R, T, free, d)
        F2 = evaluate(R2, T2, ij, ZR, ZT, om, c)["F"]
        if F2 < F:
            R, T, F, lam, acc = R2, T2, F2, lam / 10.0, acc + 1
            x = d.reshape(-1, 6)
            if np.abs(x[:, :3]).max() < eps_t and np.abs(x[:, 3:]).max() < eps_r:
                status = CONVERGED
                break
            D, Off, g, free, ev = normal_equations(R, T, ij, ZR, ZT, om, c, fixed)
        else:
            lam *= 10.0
            if lam > 1e16:
                status = NO_PROGRESS
                break
    ev = evaluate(R, T, ij, ZR, ZT, om, c)
    return dict(R=R, T=T, chi2=ev["chi2"], weight=ev["weight"], F0=F0, F=ev["F"], evaluations=evals, accepted=acc,
                converged=status == CONVERGED, status=status)


def gradient(R, T, fixed, ij, ZR, ZT, om, c):
    """g of the IRLS linearisation at (R, T) over the free nodes: zero at a stationary point of F."""
    return normal_equations(R, T, ij, ZR, ZT, om, c, np.asarray(fixed, bool))[2]


def check(N, R, T, fixed, ij, ZR, ZT, om, c, max_iters=100, max_cg=500, cg_tol=1e-10, eps_t=1e-6, eps_r=1e-8, pcg_grid=0):
    """The refusals in the library's order: returns None or a short reason."""
    E = len(ij)
    if not (2 <= N <= MAX_N) or not (1 <= E <= MAX_E):
        return "size"
    if not (np.isfinite(eps_t) and eps_t >= 0 and np.isfinite(eps_r) and eps_r >= 0 and np.isfinite(cg_tol)
            and 0 <= cg_tol < 1 and 0 <= max_iters <= 100000 and 1 <= max_cg <= 100000 and pcg_grid >= 0):
        return "params"
    I3 = np.eye(3)
    for n in range(N):
        if not (np.all(np.isfinite(R[n])) and np.all(np.isfinite(T[n]))):
            return "pose not finite"
        if np.abs(R[n].T @ R[n] - I3).max() > 1e-6:
            return "pose rotation"
    for k in range(E):
        i, j = int(ij[k][0]), int(ij[k][1])
        if not (0 <= i < N and 0 <= j < N) or i == j:
            return "endpoint"
        U = np.triu(om[k])
        if not (np.all(np.isfinite(ZR[k])) and np.all(np.isfinite(ZT[k])) and np.all(np.isfinite(U)) and np.isfinite(c[k])):
            return "edge not finite"
        if c[k] < 0:
            return "cauchy"
        if np.abs(ZR[k].T @ ZR[k] - I3).max() > 1e-6:
            return "edge rotation"
        if np.any(np.diag(om[k]) < 0):
            return "omega diagonal"
    parent = list(range(N))

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a
    for i, j in ij:
        parent[find(int(i))] = find(int(j))
    anchored = {find(n) for n in range(N) if fixed[n]}
    if any(find(n) not in anchored for n in range(N)):
        return "component without a fixed node"
    return None


def rot(axis, deg):
    a = np.asarray(axis, np.float64)
    return exp(np.r_[0.0, 0.0, 0.0, np.deg2rad(deg) * a / np.linalg.norm(a)])[0]


def information(sigma_t, sigma_r):
    return np.diag([sigma_t ** -2] * 3 + [sigma_r ** -2] * 3)


def relative(Ri, ti, Rj, tj):
    """Z = X_j^-1 X_i: i-local -> j-local."""
    return Rj.T @ Ri, Rj.T @ (ti - tj)


def random_walk_graph(n, seed=0, loop_every=4, false_frac=0.1, rank3_frac=0.2, sigma_t=0.01, sigma_r=0.005,
                      loop_cauchy=3.0):
    """A seeded test graph: a random walk of n poses (true), odometry edges i -> i+1 measured with noise, a loop edge
    from every loop_every-th node back to a random node 2 to 24 steps earlier (true relative pose plus noise), of which false_frac are
    false (moved by about 1 m and 20 degrees) and rank3_frac carry plane-only (rank-3) information; loops are
    Cauchy-robust with scale loop_cauchy.  Node 0 is fixed; the initial poses compose the noisy odometry.  Returns
    (R0, T0, fixed, edges, Rtrue, Ttrue, false_mask)."""
    rng = np.random.default_rng(seed)
    Rt, Tt = np.zeros((n, 3, 3)), np.zeros((n, 3))
    Rt[0] = np.eye(3)
    for k in range(1, n):
        d = np.r_[rng.normal(0, 0.3, 3), rng.normal(0, 0.05, 3)]
        Rt[k], Tt[k] = update(Rt[k - 1], Tt[k - 1], d)
    ij, ZR, ZT, om, c, bad = [], [], [], [], [], []
    Oodo = information(sigma_t, sigma_r)

    def noisy(Z, sc):
        return update(Z[0], Z[1], np.r_[rng.normal(0, sigma_t * sc, 3), rng.normal(0, sigma_r * sc, 3)])
    for k in range(n - 1):
        Z = noisy(relative(Rt[k], Tt[k], Rt[k + 1], Tt[k + 1]), 1.0)
        ij.append((k, k + 1)); ZR.append(Z[0]); ZT.append(Z[1]); om.append(Oodo); c.append(0.0); bad.append(False)
    for k in range(loop_every, n, loop_every):
        j = k - int(rng.integers(2, min(k, 24) + 1))
        Z = noisy(relative(Rt[k], Tt[k], Rt[j], Tt[j]), 0.5)
        f = rng.random() < false_frac
        if f:
            ax = rng.normal(size=3)
            dt = rng.normal(size=3)
            Z = update(Z[0], Z[1], np.r_[dt / np.linalg.norm(dt), np.deg2rad(20.0) * ax / np.linalg.norm(ax)])
        O = information(0.5 * sigma_t, 0.5 * sigma_r)
        if rng.random() < rank3_frac:
            O = np.diag([0.0, 0.0, (0.5 * sigma_t) ** -2, (0.5 * sigma_r) ** -2, (0.5 * sigma_r) ** -2, 0.0])
        ij.append((k, j)); ZR.append(Z[0]); ZT.append(Z[1]); om.append(O); c.append(loop_cauchy); bad.append(f)
    ij = np.array(ij, np.int64)
    ZR, ZT = np.array(ZR), np.array(ZT)
    R0, T0 = np.zeros_like(Rt), np.zeros_like(Tt)
    R0[0], T0[0] = Rt[0], Tt[0]
    for k in range(n - 1):  # X_{k+1} = X_k Z^-1
        R0[k + 1] = R0[k] @ ZR[k].T
        T0[k + 1] = T0[k] - R0[k + 1] @ ZT[k]
    fixed = np.zeros(n, bool)
    fixed[0] = True
    edges = dict(ij=ij, R=ZR, T=ZT, omega=np.array(om), cauchy=np.array(c))
    return R0, T0, fixed, edges, Rt, Tt, np.array(bad)


def solve_edges(R, T, fixed, edges, **opts):
    """solve() on an edges dict (pose_graph.optimize's layout)."""
    return solve(R, T, fixed, edges["ij"], edges["R"], edges["T"], edges["omega"],
                 edges.get("cauchy", np.zeros(len(edges["ij"]))), **opts)
