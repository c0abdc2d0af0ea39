"""tslam_pose_graph_solve on the GPU against tests/pose_graph_reference.py: the evaluation at the input, one exact LM step,
full solves on hand-worked and seeded random-walk graphs (optimality checked with the reference's gradient), bit-identical
fixed nodes and repeated calls whatever the CG grid, and the SubmapMapping flow on the loop world."""
import numpy as np
import pytest

import pose_graph_reference as P
from taichislam_b200 import _capi as capi
from taichislam_b200 import pose_graph

pytestmark = pytest.mark.gpu


def rot_err(Ra, Rb):
    return np.abs(P.log(np.swapaxes(Rb, -1, -2) @ Ra, np.zeros(Ra.shape[:-1]))[..., 3:]).max()


def test_max_iters_zero_evaluates_the_input():
    R0, T0, fx, ed, *_ = P.random_walk_graph(64, seed=3)
    g = pose_graph.optimize(R0, T0, fx, ed, max_iters=0)
    ev = P.evaluate(R0, T0, ed["ij"], ed["R"], ed["T"], ed["omega"], ed["cauchy"])
    assert g["evaluations"] == 0 and g["status"] == P.MAX_ITERS
    assert np.array_equal(g["R"], R0) and np.array_equal(g["T"], T0)
    assert abs(g["F0"] - ev["F"]) <= 1e-12 * ev["F"] and g["F"] == g["F0"]
    assert np.all(np.abs(g["chi2"] - ev["chi2"]) <= 1e-12 * np.maximum(ev["chi2"], 1e-300) + 1e-18)
    assert np.all(np.abs(g["weight"] - ev["weight"]) <= 1e-12 * ev["weight"])


@pytest.mark.parametrize("n", [64, 1024])
def test_one_step_is_the_exact_step(n):
    R0, T0, fx, ed, *_ = P.random_walk_graph(n, seed=5)
    g = pose_graph.optimize(R0, T0, fx, ed, max_iters=1, cg_tol=1e-14, max_cg=20000)
    r = P.solve_edges(R0, T0, fx, ed, max_iters=1)
    assert g["accepted"] == r["accepted"] == 1
    assert np.abs(g["T"] - r["T"]).max() <= 1e-9 and rot_err(g["R"], r["R"]) <= 1e-9
    assert g["cg_residual"] <= 1e-14 or g["cg_iterations"] == 20000


def hand_graphs():
    I = np.eye(3)
    corners = [np.array(p, float) for p in ((0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0))]
    ij, ZR, ZT = [], [], []
    for k in range(4):
        a, b = k, (k + 1) % 4
        ij.append((a, b)); ZR.append(I); ZT.append(corners[a] - corners[b] + (np.array([0.04, 0, 0]) if k == 2 else 0.0))
    square = (np.stack([I] * 4), np.zeros((4, 3)), np.array([1, 0, 0, 0], bool),
              dict(ij=np.array(ij), R=np.stack(ZR), T=np.stack(ZT), omega=np.stack([P.information(0.1, 0.01)] * 4),
                   cauchy=np.zeros(4)))
    true = [(I, np.zeros(3)), P.exp([1.0, 0.0, 0.0, 0.0, 0.0, 0.1]), P.exp([2.0, 0.5, 0.0, 0.0, 0.0, 0.2])]
    plane = np.diag([0.0, 0.0, 1e4, 1e4, 1e4, 0.0])
    st = [true[0]] + [P.update(*p, [0.05, -0.03, 0.02, 0.01, -0.01, 0.02]) for p in true[1:]]
    rel = [P.relative(*true[a], *true[b]) for a, b in ((0, 1), (1, 2), (2, 0))]
    rank3 = (np.stack([p[0] for p in st]), np.stack([p[1] for p in st]), np.array([1, 0, 0], bool),
             dict(ij=np.array([(0, 1), (1, 2), (2, 0)]), R=np.stack([z[0] for z in rel]), T=np.stack([z[1] for z in rel]),
                  omega=np.stack([P.information(0.1, 0.01)] * 2 + [plane]), cauchy=np.zeros(3)))
    return [square, rank3]


def check_against_reference(R0, T0, fx, ed, t_tol=1e-7, r_tol=1e-8):
    opts = dict(eps_t=1e-8, eps_r=1e-10)
    g = pose_graph.optimize(R0, T0, fx, ed, **opts)
    r = P.solve_edges(R0, T0, fx, ed, **opts)
    assert g["status"] in (P.CONVERGED, P.NO_PROGRESS, P.MAX_ITERS) and g["F"] <= g["F0"]
    et, er = np.abs(g["T"] - r["T"]).max(), rot_err(g["R"], r["R"])
    g0 = np.abs(P.gradient(R0, T0, fx, ed["ij"], ed["R"], ed["T"], ed["omega"], ed["cauchy"])).max()
    gg = np.abs(P.gradient(g["R"], g["T"], fx, ed["ij"], ed["R"], ed["T"], ed["omega"], ed["cauchy"])).max()
    gr = np.abs(P.gradient(r["R"], r["T"], fx, ed["ij"], ed["R"], ed["T"], ed["omega"], ed["cauchy"])).max()
    print(f"N={len(R0)} E={len(ed['ij'])} gpu: {g['status_name']} evals {g['evaluations']} cg {g['cg_iterations']} "
          f"F {g['F']:.9g} | ref: status {r['status']} evals {r['evaluations']} F {r['F']:.9g} | dT {et:.2e} dR {er:.2e} "
          f"|g| init {g0:.2e} gpu {gg:.2e} ref {gr:.2e}")
    assert et <= t_tol and er <= r_tol
    assert gg <= max(1e-6 * g0, 10 * gr)
    assert np.array_equal(g["R"][fx], R0[fx]) and np.array_equal(g["T"][fx], T0[fx])
    return g, r


@pytest.mark.parametrize("k", [0, 1])
def test_hand_worked_graphs(k):
    check_against_reference(*hand_graphs()[k])


@pytest.mark.parametrize("n", [64, 256, 1024, 4096])
def test_random_walk_graphs(n):
    R0, T0, fx, ed, _, _, bad = P.random_walk_graph(n, seed=n)
    g, r = check_against_reference(R0, T0, fx, ed)
    assert np.abs(g["weight"] - r["weight"]).max() <= 1e-6
    assert g["weight"][bad].max() < 0.1 < g["weight"][~bad].min()


def test_bits_do_not_depend_on_the_grid_or_the_call():
    R0, T0, fx, ed, *_ = P.random_walk_graph(1024, seed=9)
    fx[[100, 500]] = True
    a = pose_graph.optimize(R0, T0, fx, ed, max_iters=20)
    for kw in (dict(), dict(pcg_grid=1), dict(pcg_grid=3), dict(pcg_grid=7), dict(pcg_grid=64)):
        b = pose_graph.optimize(R0, T0, fx, ed, max_iters=20, **kw)
        for key in ("R", "T", "chi2", "weight"):
            assert np.array_equal(a[key].view(np.int64), b[key].view(np.int64)), (kw, key)
        assert (a["F"], a["cg_iterations"], a["evaluations"]) == (b["F"], b["cg_iterations"], b["evaluations"])
    assert np.array_equal(a["R"][fx].view(np.int64), R0[fx].view(np.int64))
    assert np.array_equal(a["T"][fx].view(np.int64), T0[fx].view(np.int64))


def test_refusals_and_lower_triangle_ignored():
    R0, T0, fx, ed, *_ = P.random_walk_graph(64, seed=2)
    with pytest.raises(capi.TslamError):
        pose_graph.optimize(R0, T0, np.zeros_like(fx), ed)
    with pytest.raises(capi.TslamError):
        pose_graph.optimize(R0, T0, fx, dict(ed, cauchy=-ed["cauchy"] - 1.0))
    om = ed["omega"].copy()
    om[:, 5, 0] = np.nan
    a = pose_graph.optimize(R0, T0, fx, ed, max_iters=3)
    b = pose_graph.optimize(R0, T0, fx, dict(ed, omega=om), max_iters=3)
    assert np.array_equal(a["T"], b["T"])
