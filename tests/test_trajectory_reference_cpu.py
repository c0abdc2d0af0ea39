"""The numpy statement of the trajectory solver (trajectory_reference.py) pinned on hand-worked answers, and the host
helpers of taichislam_b200.trajectory."""
import numpy as np

import trajectory_reference as tref
from taichislam_b200.trajectory import control_points, sample

F32 = np.float32
VS = 0.05


def const_field(d0=1.0):
    def f(x):
        n = x.shape[0]
        return np.full(n, d0, F32), np.zeros((n, 3), F32), np.ones(n, bool)
    return f


def plane_field(valid_above=None, sign=1.0, y0=0.0):
    """d = sign (y - y0), g = (0, sign, 0); valid where y > valid_above (everywhere when None)"""
    def f(x):
        y = x[:, 1].astype(np.float64)
        d = (sign * (y - y0)).astype(F32)
        g = np.tile(np.array([0.0, sign, 0.0], F32), (x.shape[0], 1))
        v = np.ones(x.shape[0], bool) if valid_above is None else y > valid_above
        return np.where(v, d, np.nan).astype(F32), np.where(v[:, None], g, np.nan).astype(F32), v
    return f


def test_tsum_is_the_thread_partials_and_halving_tree():
    rng = np.random.default_rng(0)
    for n in (1, 5, 256, 257, 1000, 3000):
        x = rng.integers(-1000, 1000, n).astype(np.float64)
        assert tref.tsum(x) == float(x.sum())
        y = rng.normal(size=n)
        p = [0.0] * tref.P
        for i in range(n):
            p[i % tref.P] += y[i]
        s = tref.P // 2
        while s >= 1:
            for i in range(s):
                p[i] = p[i] + p[i + s]
            s //= 2
        assert tref.tsum(y) == p[0]


def test_basis_rows_sum_to_one_and_interpolate_the_spline():
    b = tref.basis(4)
    assert np.allclose(b.sum(1), 1.0, atol=1e-15)
    assert b[0].tolist() == [1 / 6, 4 / 6, 1 / 6, 0.0] and b[4, 3] == 1 / 6


def test_collinear_line_at_binary_spacing_is_already_optimal():
    Q = np.stack([np.arange(10) * 0.25, np.zeros(10), np.zeros(10)], 1)
    r = tref.solve(Q, const_field(1.0), VS, clearance=0.2)
    assert r["info"][:3].tolist() == [0, 1, 1]
    assert r["ctrl"].tobytes() == Q.tobytes()
    assert r["cost"][:4].tolist() == [0.0, 0.0, 0.0, 0.0]
    assert r["info"][3:5].tolist() == [0, 0] and r["cost"][5] == 1.0 and tuple(r["info"][5:]) == (0, 0)


def test_smoothness_alone_reaches_the_linear_solve():
    rng = np.random.default_rng(1)
    N = 12
    Q = np.stack([np.arange(N) * 0.2, np.zeros(N), np.zeros(N)], 1)
    Q[3:N - 3] += rng.normal(0, 0.05, (N - 6, 3))
    r = tref.solve(Q, const_field(), VS, clearance=0.0, w_collision=0.0, w_feasibility=0.0, w_unknown=0.0, g_tol=1e-13,
                   max_iters=2000, memory=16)
    # J_s = |A x + b|^2 per axis, x the free control points
    A = np.zeros((N - 3, N))
    for i in range(N - 3):
        A[i, i:i + 4] = [-1, 3, -3, 1]
    Af, Ax = A[:, 3:N - 3], np.concatenate([A[:, :3], A[:, N - 3:]], 1)
    fixed = np.concatenate([Q[:3], Q[N - 3:]], 0)
    x = np.linalg.solve(Af.T @ Af, -Af.T @ (Ax @ fixed))
    assert r["info"][2] in (1, 2)
    assert np.abs(r["ctrl"][3:N - 3] - x).max() <= 1e-9


def test_planar_field_pushes_the_line_out_of_the_clearance():
    N = 16
    Q = np.stack([np.arange(N) * 0.1, np.full(N, 0.1), np.zeros(N)], 1)
    Q[:3, 1] = Q[-3:, 1] = 0.5
    r = tref.solve(Q, plane_field(), VS, clearance=0.3, w_collision=1e4, max_iters=500, check_samples=32)
    assert r["cost"][5] >= 0.3 - 1e-3, r
    assert r["ctrl"][:3].tobytes() == Q[:3].tobytes() and r["ctrl"][-3:].tobytes() == Q[-3:].tobytes()


def _feas_only(Q, **kw):
    prm = dict(tref.DEFAULTS, clearance=0.0, w_smooth=0.0, w_collision=0.0, w_unknown=0.0, **kw)
    return tref.evaluate(Q, const_field(), prm, tref.basis(prm["samples"]))


def _central(Q, prm_kw, fld, eps):
    prm = dict(tref.DEFAULTS, **prm_kw)
    bk = tref.basis(prm["samples"])
    g = np.zeros_like(Q)
    for i in range(3, Q.shape[0] - 3):
        for a in range(3):
            Qp, Qm = Q.copy(), Q.copy()
            Qp[i, a] += eps
            Qm[i, a] -= eps
            g[i, a] = (tref.evaluate(Qp, fld, prm, bk)[0] - tref.evaluate(Qm, fld, prm, bk)[0]) / (2 * eps)
    return g


def test_feasibility_hinges():
    N = 10
    Q = np.stack([np.arange(N) * 0.1, np.zeros(N), np.zeros(N)], 1)
    J, J4, G = _feas_only(Q, dt=0.5)                       # v = 0.2 < 2, a = 0: below both limits
    assert J4[2] == 0.0 and not G.any()
    rng = np.random.default_rng(2)
    Q = np.cumsum(rng.normal(0, 0.6, (N, 3)), 0)           # fast and jerky: both hinges active
    kw = dict(clearance=0.0, w_smooth=0.0, w_collision=0.0, w_unknown=0.0, dt=0.3, v_max=1.0, a_max=1.0)
    J, J4, G = tref.evaluate(Q, const_field(), dict(tref.DEFAULTS, **kw), tref.basis(4))
    assert J4[2] > 0
    num = _central(Q, kw, const_field(), 1e-6)
    assert np.allclose(G, num, rtol=1e-5, atol=1e-6 * np.abs(num).max())


def test_full_cost_gradient_against_central_differences():
    def sphere(x):
        p = x.astype(np.float64) - np.array([0.5, 0.3, 0.0])
        r = np.linalg.norm(p, axis=1)
        return (r - 0.4).astype(F32), (p / r[:, None]).astype(F32), np.ones(x.shape[0], bool)
    N = 12
    Q = np.stack([np.linspace(-0.2, 1.2, N), np.full(N, 0.05), np.linspace(0, 0.1, N)], 1)
    kw = dict(clearance=0.5, w_collision=100.0, dt=0.1, v_max=1.0, a_max=3.0)
    J, J4, G = tref.evaluate(Q, sphere, dict(tref.DEFAULTS, **kw), tref.basis(4))
    assert J4[1] > 0 and J4[2] > 0
    num = _central(Q, kw, sphere, 1e-4)
    assert np.allclose(G, num, rtol=2e-3, atol=2e-3 * np.abs(num).max())


def test_invalid_samples_are_counted_and_never_entered():
    N = 14
    Q = np.stack([np.arange(N) * 0.1, np.full(N, 0.3), np.zeros(N)], 1)
    fld = plane_field(valid_above=0.05, sign=-1.0, y0=0.5)  # obstacle above y = 0.5, unknown below y = 0.05
    r0 = tref.solve(Q, fld, VS, clearance=0.4, max_iters=0, samples=4)
    assert r0["cost"][3] == 0.0 and r0["info"][2] == 0
    r = tref.solve(Q, fld, VS, clearance=0.4, w_collision=1e3, max_iters=300, samples=4, check_samples=4)
    assert r["cost"][3] == 0.0 and r["info"][3] == 0                      # never stepped into unknown space
    assert r["ctrl"][3:-3, 1].min() < 0.3                                 # the collision term pulled towards it
    # counted: a line that dips below y = 0.05
    Q2 = Q.copy()
    Q2[5:9, 1] = -0.2
    r2 = tref.solve(Q2, fld, VS, clearance=0.4, max_iters=0, samples=4)
    x = tref.positions(Q2, tref.basis(4)).astype(F32)[tref.sample_mask(N - 3, 4)]
    assert r2["cost"][3] == float((x[:, 1].astype(np.float64) <= 0.05).sum()) > 0


def test_dense_check_outputs():
    N = 8
    Q = np.stack([1.0 + np.arange(N) * 0.25, np.zeros(N), np.zeros(N)], 1)

    def fx(x):
        d = x[:, 0].copy()
        return d, np.tile(np.array([1, 0, 0], F32), (x.shape[0], 1)), x[:, 0] < 2.5
    md, n_inv, n_close, js, ks = tref.check(Q, fx, dict(tref.DEFAULTS, clearance=1.5, check_samples=4))
    x = tref.positions(Q, tref.basis(4)).astype(F32)[tref.sample_mask(N - 3, 4)]
    assert md == float(x[0, 0]) and (js, ks) == (0, 0)
    assert n_inv == int((x[:, 0] >= 2.5).sum()) and n_close == int(((x[:, 0] < 2.5) & (x[:, 0] < 1.5)).sum())
    md, n_inv, _, js, ks = tref.check(Q, lambda x: (np.full(len(x), np.nan, F32), np.full((len(x), 3), np.nan, F32),
                                                    np.zeros(len(x), bool)), dict(tref.DEFAULTS, check_samples=4))
    assert md == np.inf and (js, ks) == (-1, -1) and n_inv == (N - 3) * 4 + 1


def test_control_points_and_sample():
    path = np.array([[0.0, 0, 0], [1.0, 0, 0], [1.0, 1.0, 0]])
    q = control_points(path, 0.25)
    assert q.shape == (9 + 4, 3)
    assert (q[:3] == path[0]).all() and (q[-3:] == path[-1]).all()
    assert np.allclose(np.linalg.norm(np.diff(q[2:-2], axis=0), axis=1), 0.25)
    p, v, a = sample(q, 0.5, 4)
    assert p.shape == ((len(q) - 3) * 4 + 1, 3)
    assert np.allclose(p[0], path[0]) and np.allclose(p[-1], path[-1])
    assert np.allclose(v[0], 0) and np.allclose(v[-1], 0) and np.allclose(a[0], 0) and np.allclose(a[-1], 0)
