"""numpy statement of tslam_tsdf_register (csrc/tslam_register.cu; DESIGN.md section 7, "Submap registration").

The per-point f32 values are the kernel's bit for bit (the library builds with -fmad=false; every f32 step below is one
correctly rounded operation in the kernel's order, and the interpolation is tests/esdf_query_reference.py's).  The f64
sums are the same terms added in another order, so they agree to rounding; the LM loop is the host solver's, step for
step.

Inputs are voxel rows as gather() returns them: idx int32[m,3] (centred indices), tsdf f32[m], w f32[m] of the observed
voxels of one submap.
  reference points   rows with w > 0, w >= min_weight, |tsdf| <= band;  p_v = f32(idx) * vs, d_v = tsdf
  reading corners    rows with w > 0 (an observed voxel of a present block); everything else is not a valid corner
Residual of a point at pose (R, t) (rounded to f32 once): x = ((R0 px + R1 py) + R2 pz) + t0 per row in f32, D_B(x) and its
gradient g by the ESDF query rules, r = D_B(x) - d_v in f32, then in f64: J = [g, x cross g], w = 1 if |r| <= delta else
delta / |r|, rho = r^2 / 2 or delta (|r| - delta / 2); H = sum w J J^T, b = sum w J r, cost = sum rho, n_valid.
"""
import numpy as np

import esdf_query_reference as eqr

F = np.float32
NS = 29


class Reading:
    """The reading submap's corners (valid: observed with W > 0) and the volume."""

    def __init__(self, idx, tsdf, w, N, Nz, vs):
        idx, tsdf, w = np.asarray(idx, np.int32).reshape(-1, 3), np.asarray(tsdf, F), np.asarray(w, F)
        keep = w > 0
        self.st = eqr.EsdfState(idx[keep], np.zeros(int(keep.sum()), F), tsdf[keep], N, Nz, vs)


def select_points(idx, tsdf, w, vs, band, min_weight=0.0):
    """-> p f32[n,3], d f32[n] of the registration points."""
    idx, tsdf, w = np.asarray(idx, np.int32).reshape(-1, 3), np.asarray(tsdf, F), np.asarray(w, F)
    with np.errstate(invalid="ignore"):
        keep = (w > 0) & (w >= F(min_weight)) & (np.abs(tsdf) <= F(band))
    return idx[keep].astype(F) * F(vs), tsdf[keep]


def point_terms(reading, p, d, R, t, delta):
    """Per-point values at pose (R, t) (f64 in, rounded to f32): dict(x f32[n,3], r f32[n], g f32[n,3], valid bool[n],
    J f64[n,6], w f64[n], rho f64[n]) - J, w, rho only for the valid points."""
    R32, t32 = np.asarray(R, np.float64).reshape(3, 3).astype(F), np.asarray(t, np.float64).reshape(3).astype(F)
    x = np.stack([((R32[i, 0] * p[:, 0] + R32[i, 1] * p[:, 1]) + R32[i, 2] * p[:, 2]) + t32[i] for i in range(3)], 1).astype(F)
    D, g, valid = eqr.query(reading.st, x)
    r = (D - d).astype(F)
    xv, gv, rv = x[valid].astype(np.float64), g[valid].astype(np.float64), r[valid].astype(np.float64)
    J = np.concatenate([gv, np.stack([xv[:, 1] * gv[:, 2] - xv[:, 2] * gv[:, 1], xv[:, 2] * gv[:, 0] - xv[:, 0] * gv[:, 2],
                                      xv[:, 0] * gv[:, 1] - xv[:, 1] * gv[:, 0]], 1)], 1)
    ar = np.abs(rv)
    delta = float(F(delta))
    with np.errstate(divide="ignore"):
        wt = np.where(ar <= delta, 1.0, delta / np.maximum(ar, 1e-300))
    rho = np.where(ar <= delta, 0.5 * rv * rv, delta * (ar - 0.5 * delta))
    return dict(x=x, r=r, g=g, valid=valid, J=J, w=wt, rho=rho, rv=rv)


def normal_equations(reading, p, d, R, t, delta):
    """-> S f64[29]: H (upper triangle row by row), b, cost, n_valid."""
    q = point_terms(reading, p, d, R, t, delta)
    J, wt, rv = q["J"], q["w"], q["rv"]
    wJ = wt[:, None] * J
    S = np.zeros(NS)
    k = 0
    for i in range(6):
        for j in range(i, 6):
            S[k] = np.sum(wJ[:, i] * J[:, j])
            k += 1
    S[21:27] = np.sum(wJ * rv[:, None], 0)
    S[27] = np.sum(q["rho"])
    S[28] = float(q["valid"].sum())
    return S


def sym(S):
    H = np.zeros((6, 6))
    k = 0
    for i in range(6):
        for j in range(i, 6):
            H[i, j] = H[j, i] = S[k]
            k += 1
    return H


def se3_update(R, t, xi):
    """exp(xi) * (R, t), xi = (rho, phi): R' = Exp(phi) R, t' = Exp(phi) t + V(phi) rho."""
    rho, phi = np.asarray(xi[:3], np.float64), np.asarray(xi[3:], np.float64)
    th2 = float(phi @ phi)
    th = np.sqrt(th2)
    if th < 1e-4:
        A, B, C = 1.0 - th2 / 6.0, 0.5 - th2 / 24.0, 1.0 / 6.0 - th2 / 120.0
    else:
        A, B, C = np.sin(th) / th, (1.0 - np.cos(th)) / th2, (th - np.sin(th)) / (th2 * th)
    K = np.array([[0.0, -phi[2], phi[1]], [phi[2], 0.0, -phi[0]], [-phi[1], phi[0], 0.0]])
    K2 = K @ K
    E = np.eye(3) + A * K + B * K2
    V = np.eye(3) + B * K + C * K2
    return E @ R, E @ t + V @ rho


def solve_step(S, lam):
    """(H + lam diag(max(H_ii, 1e-9 max H_jj))) xi = -b by Cholesky; None when not positive definite."""
    H = sym(S)
    dg = np.diag(H).copy()
    H[np.diag_indices(6)] += lam * np.maximum(dg, 1e-9 * dg.max())
    try:
        L = np.linalg.cholesky(H)
    except np.linalg.LinAlgError:
        return None
    y = np.linalg.solve(L, -S[21:27])
    return np.linalg.solve(L.T, y)


def mean_cost(S):
    return S[27] / S[28] if S[28] > 0 else np.inf


def register(reading, p, d, R0, T0, vs, huber=None, max_iters=20, min_points=100):
    """The host solver of one pair -> dict(R, T, S (at the final pose), cost_init, iterations, converged, status)."""
    delta = float(F(vs if huber is None else huber))
    R, t = np.asarray(R0, np.float64).reshape(3, 3).copy(), np.asarray(T0, np.float64).reshape(3).copy()
    S = normal_equations(reading, p, d, R, t, delta)
    out = dict(cost_init=S[27], iterations=0, converged=0, status=0)
    if S[28] < min_points:
        out["status"] = 1
    lam, it = 1e-4, 0
    rho_tol, phi_tol = 1e-4 * float(F(vs)), 1e-6
    active = out["status"] == 0 and max_iters > 0
    while active:
        xi = solve_step(S, lam)
        if xi is None:
            break
        if np.linalg.norm(xi[:3]) < rho_tol and np.linalg.norm(xi[3:]) < phi_tol:
            out["converged"] = 1
            break
        Rn, tn = se3_update(R, t, xi)
        Sn = normal_equations(reading, p, d, Rn, tn, delta)
        it += 1
        if Sn[28] >= min_points and mean_cost(Sn) < mean_cost(S):
            R, t, S, lam = Rn, tn, Sn, lam / 10.0
        else:
            lam *= 10.0
        if it >= max_iters:
            break
    out.update(R=R, T=t, S=S, iterations=it)
    return out


def rot(axis, deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    x, y, z = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.array([[c + x * x * (1 - c), x * y * (1 - c) - z * s, x * z * (1 - c) + y * s],
                     [y * x * (1 - c) + z * s, c + y * y * (1 - c), y * z * (1 - c) - x * s],
                     [z * x * (1 - c) - y * s, z * y * (1 - c) + x * s, c + z * z * (1 - c)]])


def pose_error(R, t, Rt, tt):
    """(translation error m, rotation error deg) of (R, t) against the truth (Rt, tt)."""
    dR = R @ Rt.T
    ang = np.degrees(np.arccos(np.clip((np.trace(dR) - 1.0) / 2.0, -1.0, 1.0)))
    return float(np.linalg.norm(t - tt)), float(ang)


# The integrated scene of the recovery tests: one scene_room view (camera at the world origin), integrated into two
# submaps whose base poses differ by 30 degrees about the vertical (camera y) axis and 0.7 m, from different but
# overlapping frame subsets (scene_room seeds: the frames differ in their random dropouts).
ROOM_BASE_A = (np.eye(3), np.zeros(3))
ROOM_BASE_B = (rot([0.0, 1.0, 0.0], 30.0), np.array([0.6, 0.0, 0.36]))
ROOM_SEEDS_A, ROOM_SEEDS_B = (3, 4), (4, 5)
ROOM_PERTURB = [((0.1, 0.0, 0.0), ([0.0, 1.0, 0.0], 3.0)), ((0.0, -0.07, 0.07), ([1.0, 0.0, 0.0], -3.0)),
                ((0.05, 0.05, -0.05), ([1.0, 1.0, 1.0], 2.5))]


def local_pose(base, R_wc=np.eye(3), t_wc=np.zeros(3)):
    """Camera pose in a submap's local frame: base^-1 * T_wc."""
    Rb, tb = base
    return Rb.T @ R_wc, Rb.T @ (t_wc - tb)


def true_relative(base_a, base_b):
    """T = base_b^-1 * base_a: reference-local -> reading-local."""
    (Ra, ta), (Rb, tb) = base_a, base_b
    return Rb.T @ Ra, Rb.T @ (ta - tb)


def perturbed(R, t, k):
    """The k-th start of the recovery tests: the truth moved by ROOM_PERTURB[k] (a left perturbation)."""
    dt, (ax, deg) = ROOM_PERTURB[k]
    dR = rot(ax, deg)
    return dR @ R, dR @ t + np.asarray(dt)


def abs_sums(reading, p, d, R, t, delta):
    """Sum of |term| per entry of S: the scale against which two summation orders of the same terms are compared."""
    q = point_terms(reading, p, d, R, t, delta)
    J, wt, rv = q["J"], q["w"], q["rv"]
    wJ = np.abs(wt[:, None] * J)
    A = np.zeros(NS)
    k = 0
    for i in range(6):
        for j in range(i, 6):
            A[k] = np.sum(wJ[:, i] * np.abs(J[:, j]))
            k += 1
    A[21:27] = np.sum(wJ * np.abs(rv)[:, None], 0)
    A[27] = np.sum(np.abs(q["rho"]))
    A[28] = float(q["valid"].sum())
    return A, q
