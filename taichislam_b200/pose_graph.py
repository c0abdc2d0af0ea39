"""Submap pose-graph optimisation (tslam_pose_graph_solve, include/tslam.h; DESIGN.md section 7, "Pose-graph
optimisation"): Levenberg-Marquardt over SE(3) node poses from odometry and loop constraints, Cauchy-robust per edge, with
the damped normal equations solved by preconditioned conjugate gradients on the GPU."""
import numpy as np

from . import _capi as capi

# max_cg: block-Jacobi CG needs on the order of the chain length in iterations on long odometry chains (about 2500 per
# LM evaluation on the 1024-node random walk of the tests); CG stops at cg_tol first on easier graphs.
DEFAULTS = dict(max_iters=100, max_cg=20000, cg_tol=1e-10, eps_t=1e-6, eps_r=1e-8, pcg_grid=0)
STATUS = ("converged", "max_iters", "no progress", "not positive definite")


def optimize(R, T, fixed, edges, **solver):
    """Optimise the node poses X_i = (R[i], T[i]) (world <- submap-local; R [N,3,3], T [N,3]) with the nodes where
    fixed[i] is true held still.  edges is a dict of arrays: ij int [E,2] (i, j), R [E,3,3] and T [E,3] (Z_k: i-local ->
    j-local), omega [E,6,6] (information in (rho, phi) order; the upper triangle is read), cauchy [E] (Cauchy scale, 0 =
    least squares; optional, default 0).  solver: DEFAULTS.  Returns a dict: R [N,3,3], T [N,3] (fixed nodes bit-identical
    to the input), chi2 [E] and weight [E] at the final poses, F0, F, evaluations, accepted, cg_iterations, cg_residual
    (the largest final relative CG residual), converged, status (index into STATUS), status_name.  Raises TslamError
    (E_INVALID) on input the contract refuses."""
    o = dict(DEFAULTS)
    unknown = set(solver) - set(o)
    if unknown:
        raise TypeError(f"unknown solver options {sorted(unknown)}")
    o.update(solver)
    R = np.ascontiguousarray(np.asarray(R, np.float64).reshape(-1, 9))
    N = R.shape[0]
    T = np.ascontiguousarray(np.asarray(T, np.float64).reshape(N, 3))
    fx = np.ascontiguousarray(np.asarray(fixed, bool).reshape(N).astype(np.uint8))
    ij = np.ascontiguousarray(np.asarray(edges["ij"], np.int32).reshape(-1, 2))
    E = ij.shape[0]
    ZR = np.ascontiguousarray(np.asarray(edges["R"], np.float64).reshape(E, 9))
    ZT = np.ascontiguousarray(np.asarray(edges["T"], np.float64).reshape(E, 3))
    om = np.ascontiguousarray(np.asarray(edges["omega"], np.float64).reshape(E, 36))
    c = edges.get("cauchy")
    c = np.zeros(E) if c is None else np.ascontiguousarray(np.broadcast_to(np.asarray(c, np.float64), (E,)))
    prm = capi.PgParams(float(o["eps_t"]), float(o["eps_r"]), float(o["cg_tol"]), int(o["max_iters"]), int(o["max_cg"]),
                        int(o["pcg_grid"]))
    Ro, To = np.zeros((N, 9)), np.zeros((N, 3))
    chi2, w, f3, info = np.zeros(max(E, 1)), np.zeros(max(E, 1)), np.zeros(3), np.zeros(5, np.int64)
    capi.check(capi.load().tslam_pose_graph_solve(N, capi.np_ptr(R), capi.np_ptr(T), capi.np_ptr(fx), E, capi.np_ptr(ij),
                                                  capi.np_ptr(ZR), capi.np_ptr(ZT), capi.np_ptr(om), capi.np_ptr(c), prm,
                                                  capi.np_ptr(Ro), capi.np_ptr(To), capi.np_ptr(chi2), capi.np_ptr(w),
                                                  capi.np_ptr(f3), capi.np_ptr(info), capi.stream_ptr()))
    st = int(info[4])
    return dict(R=Ro.reshape(N, 3, 3), T=To, chi2=chi2[:E], weight=w[:E], F0=float(f3[0]), F=float(f3[1]),
                cg_residual=float(f3[2]), evaluations=int(info[0]), accepted=int(info[1]), cg_iterations=int(info[2]),
                converged=bool(info[3]), status=st, status_name=STATUS[st])
