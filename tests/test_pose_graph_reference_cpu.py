"""tests/pose_graph_reference.py pinned on hand-worked cases: Exp/Log, the Jacobians, small graphs whose optimum is known,
scipy's least squares, the Cauchy kernel against a false loop, rank-3 information, and every refusal."""
import numpy as np
import pytest
from scipy.optimize import least_squares

import pose_graph_reference as P
import submap_register_reference as S


def graph(poses, edges_, fixed=(0,)):
    R = np.stack([p[0] for p in poses])
    T = np.stack([p[1] for p in poses])
    fx = np.zeros(len(poses), bool)
    fx[list(fixed)] = True
    ij = np.array([e[0] for e in edges_])
    return R, T, fx, dict(ij=ij, R=np.stack([e[1][0] for e in edges_]), T=np.stack([e[1][1] for e in edges_]),
                          omega=np.stack([e[2] for e in edges_]), cauchy=np.array([e[3] if len(e) > 3 else 0.0 for e in edges_]))


@pytest.mark.parametrize("th", [0.0, 1e-9, 1e-6, 5e-3, 1e-2, 0.02, np.pi / 2, np.pi - 1e-9, np.pi - 1e-4, np.pi - 1e-2])
def test_exp_log_round_trip_and_registration_exponential(th):
    rng = np.random.default_rng(3)
    for _ in range(8):
        ax = rng.normal(size=3)
        xi = np.r_[rng.normal(size=3), th * ax / np.linalg.norm(ax)]
        R, t = P.exp(xi)
        assert np.abs(R.T @ R - np.eye(3)).max() < 4e-15
        assert np.abs(P.log(R, t) - xi).max() < 1e-12
        Rb, tb = P.exp(rng.normal(size=6))
        Ru, tu = P.update(Rb, tb, xi)
        Rs, ts = S.se3_update(Rb, tb, xi)
        assert np.abs(Ru - Rs).max() < 1e-14 and np.abs(tu - ts).max() < 1e-14


def test_jacobians_against_central_differences():
    rng = np.random.default_rng(5)
    N = 4
    R = np.stack([P.exp(rng.normal(size=6))[0] for _ in range(N)])
    T = rng.normal(size=(N, 3))
    ij = np.array([[0, 1], [2, 1], [1, 3], [3, 0]])
    Z = [P.exp(rng.normal(size=6) * s) for s in (1.0, 1e-3, 1e-7, 2.5)]
    ZR, ZT = np.stack([z[0] for z in Z]), np.stack([z[1] for z in Z])
    _, J = P.residuals(R, T, ij, ZR, ZT)
    h = 1e-6
    for k in range(len(ij)):
        for side, sign in ((0, 1.0), (1, -1.0)):
            n = ij[k, side]
            Jn = np.zeros((6, 6))
            for a in range(6):
                d = np.zeros(6)
                d[a] = h
                Rp, Tp, Rm, Tm = R.copy(), T.copy(), R.copy(), T.copy()
                Rp[n], Tp[n] = P.update(R[n], T[n], d)
                Rm[n], Tm[n] = P.update(R[n], T[n], -d)
                Jn[:, a] = (P.residuals(Rp, Tp, ij, ZR, ZT)[0][k] - P.residuals(Rm, Tm, ij, ZR, ZT)[0][k]) / (2 * h)
            assert np.abs(Jn - sign * J[k]).max() <= 1e-6 * np.abs(J[k]).max(), (k, side)


def test_two_node_graph_moves_the_free_node_onto_the_measurement():
    Z = P.exp([0.3, -0.2, 0.1, 0.05, 0.2, -0.1])
    X1 = P.exp([1.0, 0.0, 0.0, 0.0, 0.0, 0.3])
    R, T, fx, ed = graph([(np.eye(3), np.zeros(3)), X1], [((0, 1), Z, P.information(0.1, 0.01))])
    r = P.solve_edges(R, T, fx, ed, eps_t=1e-12, eps_r=1e-12)
    # X_1^-1 X_0 = Z  ->  X_1 = Z^-1
    assert np.abs(r["R"][1] - Z[0].T).max() < 1e-12 and np.abs(r["T"][1] + Z[0].T @ Z[1]).max() < 1e-12
    assert r["F"] < 1e-20 and r["converged"]


def test_consistent_chain_has_zero_cost_and_composes_exactly():
    rng = np.random.default_rng(1)
    true = [(np.eye(3), np.zeros(3))]
    for _ in range(5):
        true.append(P.update(*true[-1], rng.normal(size=6) * 0.3))
    edges_ = [((k, k + 1), P.relative(*true[k], *true[k + 1]), P.information(0.1, 0.01)) for k in range(5)]
    R, T, fx, ed = graph(true, edges_)
    ev = P.evaluate(R, T, ed["ij"], ed["R"], ed["T"], ed["omega"], ed["cauchy"])
    assert ev["F"] < 1e-24
    r = P.solve_edges(R, T, fx, ed, max_iters=5)
    assert np.abs(r["R"] - R).max() < 1e-14 and np.abs(r["T"] - T).max() < 1e-14


def test_translation_square_shares_the_bias_equally():
    I = np.eye(3)
    corners = [np.array(p, float) for p in ((0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0))]
    O = P.information(0.1, 1e-7)  # rotations held at the identity: what is left is linear in the translations
    edges_ = []
    for k in range(4):
        a, b = k, (k + 1) % 4
        t = corners[a] - corners[b]          # Z = X_b^-1 X_a with identity rotations
        if k == 2:
            t = t + np.array([0.04, 0.0, 0.0])  # one biased edge
        edges_.append(((a, b), (I, t), O))
    R, T, fx, ed = graph([(I, np.zeros(3))] * 4, edges_)
    r = P.solve_edges(R, T, fx, ed, eps_t=1e-12, eps_r=1e-12)
    e = P.residuals(r["R"], r["T"], ed["ij"], ed["R"], ed["T"])[0]
    assert np.abs(r["R"] - I).max() < 1e-9
    assert np.allclose(np.abs(e[:, 0]), 0.01, atol=1e-8) and np.abs(e[:, 1:]).max() < 1e-8


def test_optimum_matches_scipy_least_squares():
    R0, T0, fx, ed, _, _, _ = P.random_walk_graph(24, seed=4, false_frac=0.0, rank3_frac=0.0, loop_cauchy=0.0)
    ed["cauchy"][:] = 0.0
    r = P.solve_edges(R0, T0, fx, ed, eps_t=1e-12, eps_r=1e-14)
    free = np.flatnonzero(~fx)
    L = np.linalg.cholesky(P.sym_omega(ed["omega"]))

    def fun(x):
        R, T = P.apply_step(R0, T0, free, x)
        e = P.residuals(R, T, ed["ij"], ed["R"], ed["T"])[0]
        return np.einsum("eba,eb->ea", L, e).ravel()
    ls = least_squares(fun, np.zeros(6 * len(free)), xtol=1e-15, ftol=1e-15, gtol=1e-15)
    R, T = P.apply_step(R0, T0, free, ls.x)
    assert abs(0.5 * np.sum(ls.fun ** 2) - r["F"]) <= 1e-9 * r["F"]
    assert np.abs(T - r["T"]).max() < 1e-7 and np.abs(R - r["R"]).max() < 1e-8


def test_cauchy_outvotes_a_false_loop():
    rng = np.random.default_rng(2)
    true = [(np.eye(3), np.zeros(3))]
    for _ in range(7):
        true.append(P.update(*true[-1], np.r_[rng.normal(size=3), 0.2 * rng.normal(size=3)]))
    O = P.information(0.05, 0.01)
    c = 0.01  # the pull of a far outlier on the Cauchy tail scales with c^2
    edges_ = [((k, (k + 1) % 8), P.relative(*true[k], *true[(k + 1) % 8]), O, c) for k in range(8)]
    edges_ += [((k, (k + 3) % 8), P.relative(*true[k], *true[(k + 3) % 8]), O, c) for k in range(0, 8, 2)]
    bad = P.update(*P.relative(*true[1], *true[5]), [1.0, 0.0, 0.0, 0.0, 0.0, np.deg2rad(20.0)])
    edges_.append(((1, 5), bad, O, c))
    start = [P.update(*p, 0.002 * rng.normal(size=6)) if k else p for k, p in enumerate(true)]
    R, T, fx, ed = graph(start, edges_)
    r = P.solve_edges(R, T, fx, ed, eps_t=1e-12, eps_r=1e-12)
    assert r["weight"][-1] < 1e-2
    assert np.abs(r["T"] - np.stack([p[1] for p in true])).max() < 1e-6
    assert np.abs(r["R"] - np.stack([p[0] for p in true])).max() < 1e-6


def test_rank3_plane_information_is_held_by_odometry():
    true = [(np.eye(3), np.zeros(3)), P.exp([1.0, 0.0, 0.0, 0.0, 0.0, 0.1]), P.exp([2.0, 0.5, 0.0, 0.0, 0.0, 0.2])]
    plane = np.diag([0.0, 0.0, 1e4, 1e4, 1e4, 0.0])  # z, roll, pitch only: registration against one floor
    edges_ = [((0, 1), P.relative(*true[0], *true[1]), P.information(0.1, 0.01)),
              ((1, 2), P.relative(*true[1], *true[2]), P.information(0.1, 0.01)),
              ((2, 0), P.relative(*true[2], *true[0]), plane)]
    start = [true[0]] + [P.update(*p, [0.05, -0.03, 0.02, 0.01, -0.01, 0.02]) for p in true[1:]]
    R, T, fx, ed = graph(start, edges_)
    r = P.solve_edges(R, T, fx, ed, eps_t=1e-12, eps_r=1e-12)
    assert r["status"] in (P.CONVERGED, P.NO_PROGRESS) and r["F"] < 1e-16
    assert np.abs(r["T"] - np.stack([p[1] for p in true])).max() < 1e-8


def test_every_refusal():
    I = np.eye(3)
    R, T, fx, ed = graph([(I, np.zeros(3)), (I, np.ones(3)), (I, np.zeros(3))],
                         [((0, 1), (I, np.ones(3)), P.information(1, 1)), ((1, 2), (I, np.zeros(3)), P.information(1, 1))])

    def chk(N=3, R=R, T=T, fx=fx, ed=ed, **kw):
        return P.check(N, R, T, fx, ed["ij"], ed["R"], ed["T"], ed["omega"], ed["cauchy"], **kw)
    assert chk() is None
    assert chk(N=1) == "size" and chk(N=4097) == "size"
    assert chk(ed=dict(ed, ij=ed["ij"][:0])) == "size"
    for kw in (dict(eps_t=-1.0), dict(eps_r=np.nan), dict(cg_tol=1.0), dict(max_iters=-1), dict(max_cg=0), dict(pcg_grid=-1)):
        assert chk(**kw) == "params", kw
    Tb = T.copy(); Tb[1, 0] = np.inf
    assert chk(T=Tb) == "pose not finite"
    Rb = R.copy(); Rb[2] = 1.01 * I
    assert chk(R=Rb) == "pose rotation"
    for ij in ([0, 3], [-1, 1], [1, 1]):
        assert chk(ed=dict(ed, ij=np.array([ij, [1, 2]]))) == "endpoint", ij
    om = ed["omega"].copy(); om[0, 0, 5] = np.nan
    assert chk(ed=dict(ed, omega=om)) == "edge not finite"
    om = ed["omega"].copy(); om[0, 5, 0] = np.nan  # below the diagonal: not read
    assert chk(ed=dict(ed, omega=om)) is None
    assert chk(ed=dict(ed, cauchy=np.array([-1.0, 0.0]))) == "cauchy"
    zr = ed["R"].copy(); zr[1] = P.rot([0, 0, 1], 10) * 1.001
    assert chk(ed=dict(ed, R=zr)) == "edge rotation"
    om = ed["omega"].copy(); om[1, 3, 3] = -1.0
    assert chk(ed=dict(ed, omega=om)) == "omega diagonal"
    assert chk(ed=dict(ed, ij=np.array([[0, 1], [0, 1]]))) == "component without a fixed node"
    assert chk(fx=np.array([False, False, False])) == "component without a fixed node"
