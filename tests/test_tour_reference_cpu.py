"""The numpy statement of the exploration-tour contract (tour_reference.py) on hand-worked answers, literal values of its
generator, every refusal, and properties on fixed seeds: converged tours have no improving move (checked by a plain
loop that rebuilds every neighbour tour), restart 0 never loses to nearest-neighbour, and for m <= 7 the best restart
is the brute-force optimum."""
import itertools
from fractions import Fraction

import numpy as np
import pytest

import tour_reference as tr

F32 = np.float32
INF = np.inf
U0 = 1 << 23  # q of 1.0 when the least positive entry is in [1, 2)


def line(xs):
    """|x_a - x_b| for the start at 0 and goals at xs"""
    x = np.array([0.0] + list(xs))
    return np.abs(x[:, None] - x[None, :]).astype(F32)


def test_m0_and_m1():
    r = tr.solve(np.zeros((1, 1), F32), restarts=3)
    assert r["tours"].tolist() == [[0]] * 3 and r["cost2"].tolist() == [[0, 0]] * 3
    assert r["passes"].tolist() == [0] * 3 and r["converged"].tolist() == [1] * 3 and r["best"] == 0
    assert r["info2"].tolist() == [0, -23]
    C = np.array([[0, INF, INF], [1, 0, 2], [4, 2, 0]], F32)         # nothing reachable from the start
    r = tr.solve(C, restarts=2)
    assert r["tours"].tolist() == [[0, -1, -1]] * 2 and r["cost2"].tolist() == [[0, 0]] * 2 and r["info2"][0] == 0
    C = np.array([[0, 3, INF], [1, 0, 2], [4, 2, 0]], F32)
    r = tr.solve(C, restarts=2)
    assert r["tours"].tolist() == [[0, 1, -1]] * 2 and r["cost2"].tolist() == [[0, 3 * U0]] * 2
    assert r["info2"].tolist() == [1, -23] and r["converged"].all() and not r["passes"].any()


def test_line_nearest_neighbour_fixed_by_one_2opt():
    # goals at x = -6, -5, -1, 2.  NN: 0 -> 3 (1) -> 4 (3) -> 2 (7) -> 1 (1) = 12; reversing t[1..2] gives
    # 0 -> 4 (2) -> 3 (3) -> 2 (4) -> 1 (1) = 10, the optimum
    C = line([-6, -5, -1, 2])
    Wi, Wq, e_lo = tr.weights(C)
    assert e_lo == 0
    nn = tr.nearest_neighbour([1, 2, 3, 4], Wi, Wq)
    assert nn == [0, 3, 4, 2, 1] and tr.tour_cost(nn, Wi, Wq) == (0, 12 * U0)
    assert tr.best_move(nn, Wi, Wq) == (0, 1, 2, 0, -2 * U0)
    r = tr.solve(C, restarts=1)
    assert r["tours"][0].tolist() == [0, 4, 3, 2, 1] and r["cost2"][0].tolist() == [0, 10 * U0]
    assert r["passes"][0] == 1 and r["converged"][0] == 1


def test_only_an_or_opt_move_improves():
    # goals at x = -6, -5, -3, 4.  NN: 0 -> 3 -> 2 -> 1 -> 4 = 3 + 2 + 1 + 10 = 16; no 2-opt improves, moving node 4
    # to follow the start (L = 1, i = 4, p = 0) gives 4 + 7 + 2 + 1 = 14
    C = line([-6, -5, -3, 4])
    Wi, Wq, _ = tr.weights(C)
    nn = tr.nearest_neighbour([1, 2, 3, 4], Wi, Wq)
    assert nn == [0, 3, 2, 1, 4]
    kind, I, J, di, dq = tr.deltas(nn, Wi, Wq)
    assert (dq[kind == 0] >= 0).all() and (dq[kind > 0] < 0).any()
    assert tr.best_move(nn, Wi, Wq) == (1, 4, 0, 0, -2 * U0)
    r = tr.solve(C, restarts=1)
    assert r["tours"][0].tolist() == [0, 4, 3, 2, 1] and r["cost2"][0].tolist() == [0, 14 * U0] and r["passes"][0] == 1


def test_reversed_legs_are_charged_in_their_new_direction():
    # [0, 1, 2] costs 1 + 8 = 9.  Reversed, the leg 1 -> 2 becomes 2 -> 1, which costs 1: [0, 2, 1] = 2 + 1 = 3.
    # Charged at the old direction it would cost 2 + 8 = 10 and no move would improve.
    C = np.array([[0, 1, 2], [9, 0, 8], [9, 1, 0]], F32)
    Wi, Wq, _ = tr.weights(C)
    assert tr.nearest_neighbour([1, 2], Wi, Wq) == [0, 1, 2]
    kind, I, J, di, dq = tr.deltas([0, 1, 2], Wi, Wq)
    assert dq[(kind == 0) & (I == 1) & (J == 2)].tolist() == [-6 * U0]
    r = tr.solve(C, restarts=1)
    assert r["tours"][0].tolist() == [0, 2, 1] and r["cost2"][0].tolist() == [0, 3 * U0]


def test_tie_order_between_equal_cost_moves():
    # on [0, 1, 2] the 2-opt (1, 2) and the Or-opt moves (1, 1, 2) and (1, 2, 0) all give [0, 2, 1]: the 2-opt is first
    C = np.array([[0, 5, 1], [5, 0, 1], [1, 1, 0]], F32)
    Wi, Wq, _ = tr.weights(C)
    kind, I, J, di, dq = tr.deltas([0, 1, 2], Wi, Wq)
    assert sorted(zip(kind.tolist(), I.tolist(), J.tolist(), dq.tolist())) == [(0, 1, 2, -4 * U0), (1, 1, 2, -4 * U0),
                                                                                (1, 2, 0, -4 * U0)]
    assert tr.best_move([0, 1, 2], Wi, Wq) == (0, 1, 2, 0, -4 * U0)
    # between two Or-opt moves of one segment, the smaller p wins: node 3 may follow node 0 or node 1 at equal cost
    C = np.array([[0, 1, 9, 1], [1, 0, 1, 1], [9, 1, 0, 9], [1, 1, 9, 0]], F32)
    Wi, Wq, _ = tr.weights(C)
    kind, I, J, di, dq = tr.deltas([0, 1, 2, 3], Wi, Wq)
    best = dq.min()
    firsts = [(k, i, j) for k, i, j, d in zip(kind.tolist(), I.tolist(), J.tolist(), dq.tolist()) if d == best]
    assert len(firsts) >= 2 and tr.best_move([0, 1, 2, 3], Wi, Wq)[:3] == firsts[0]


def test_unreachable_goals_are_left_out():
    C = line([1, 2, 3, 4])
    C[0, 2] = C[0, 4] = INF
    r = tr.solve(C, restarts=4)
    assert r["info2"][0] == 2
    for t in r["tours"]:
        assert sorted(t[1:3].tolist()) == [1, 3] and t[3:].tolist() == [-1, -1]
    assert r["tours"][r["best"]].tolist() == [0, 1, 3, -1, -1] and r["cost2"][r["best"]].tolist() == [0, 3 * U0]


def test_an_infinite_leg_between_kept_goals_counts_first():
    # [0, 1, 2] = (1 inf, 1) and [0, 2, 1] = (0 inf, 101): fewer infinite legs beat a smaller q.  NN breaks the tie
    # between goals 1 and 2 (both 1 away) to the smaller node and takes the infinite leg; one 2-opt removes it.
    C = np.array([[0, 1, 1], [1, 0, INF], [1, 100, 0]], F32)
    Wi, Wq, _ = tr.weights(C)
    assert tr.nearest_neighbour([1, 2], Wi, Wq) == [0, 1, 2] and tr.tour_cost([0, 1, 2], Wi, Wq) == (1, U0)
    r = tr.solve(C, restarts=1)
    assert r["tours"][0].tolist() == [0, 2, 1] and r["cost2"][0].tolist() == [0, 101 * U0] and r["passes"][0] == 1
    # with no way round it, the infinite leg stays and is counted
    C = np.array([[0, 1, INF], [1, 0, INF], [1, INF, 0]], F32)
    r = tr.solve(C, restarts=2)
    assert r["tours"][r["best"]].tolist() == [0, 1, -1] and r["info2"][0] == 1
    C = np.array([[0, 1, 1], [1, 0, INF], [1, INF, 0]], F32)
    r = tr.solve(C, restarts=2)
    assert r["cost2"][r["best"]].tolist() == [1, 1 * U0]


def test_exact_sums_across_a_2_22_range():
    rng = np.random.default_rng(11)
    n = 40
    e = rng.integers(-30, -8, size=(n, n))                           # 22 binades
    mant = rng.integers(1 << 23, 1 << 24, size=(n, n))
    C = np.ldexp(mant.astype(np.float64), e - 23).astype(F32)
    np.fill_diagonal(C, 0)
    r = tr.solve(C, restarts=6, seed=3)
    m, ue = r["info2"].tolist()
    assert m == n - 1 and ue == int(e[~np.eye(n, dtype=bool)].min()) - 23
    unit = Fraction(2) ** ue
    for t, (ni, q) in zip(r["tours"], r["cost2"].tolist()):
        exact = sum(Fraction(float(C[a, b])) for a, b in zip(t[:-1], t[1:]))
        assert ni == 0 and Fraction(q) * unit == exact
    # a tour through legs from the whole range, smallest unit to 2^22 times it
    Wi, Wq, _ = tr.weights(C)
    t = [0] + np.argsort(-C[0])[:-1].tolist()
    exact = sum(Fraction(float(C[a, b])) for a, b in zip(t[:-1], t[1:]))
    q = tr.tour_cost(t, Wi, Wq)[1]
    assert Fraction(q) * unit == exact and q >= 1 << 45


def test_mix64_and_shuffle_literals():
    assert tr.mix64(0) == 0
    assert tr.mix64(1) == 0x5692161d100b05e5
    assert tr.mix64(0x0123456789abcdef) == 0xb2c058e4ebb5112c
    assert tr.mix64((1 << 64) - 1) == 0xb4d055fcf2cbbd7b
    K = list(range(1, 11))
    assert tr.shuffle(K, 0, 1) == [1, 4, 9, 5, 6, 3, 8, 7, 2, 10]
    assert tr.shuffle(K, 0, 2) == [2, 10, 6, 8, 9, 4, 3, 7, 1, 5]
    assert tr.shuffle(K, 12345, 1) == [8, 5, 7, 2, 1, 10, 6, 9, 4, 3]
    # restart r >= 1 starts from exactly this shuffle
    C = line(range(1, 11))
    r = tr.solve(C, restarts=2, seed=12345, max_passes=0)
    assert r["tours"][1].tolist() == [0, 8, 5, 7, 2, 1, 10, 6, 9, 4, 3] and r["converged"][1] == 0


def test_refusals():
    ok = line([1, 2, 3])
    for bad in (np.nan, -1.0, -np.inf, 1e-40):
        C = ok.copy()
        C[1, 2] = bad
        with pytest.raises(tr.Refused):
            tr.solve(C)
    C = ok.copy()
    C[1, 1] = np.nan                                                 # the diagonal is ignored
    C[2, 2] = -5
    tr.solve(C, restarts=1)
    C = ok.copy()
    C[0, 1] = -0.0                                                   # a zero
    tr.solve(C, restarts=1)
    C = ok.copy()
    C[1, 2] = 2.0 ** 28                                              # e_lo = 0, e_hi = 28: accepted
    assert tr.solve(C, restarts=1)["info2"][1] == -23
    C[1, 2] = 2.0 ** 29
    with pytest.raises(tr.Refused):
        tr.solve(C)
    for shape in ((0, 0), (1025, 1025), (3, 4)):
        with pytest.raises(tr.Refused):
            tr.solve(np.zeros(shape, F32))
    for R in (0, 4097):
        with pytest.raises(tr.Refused):
            tr.solve(ok, restarts=R)
    with pytest.raises(tr.Refused):
        tr.solve(ok, max_passes=-1)
    tr.solve(ok, restarts=4096, max_passes=0)


def neighbours(t):
    """every tour one move away, rebuilt move by move with plain loops"""
    m = len(t) - 1
    for i in range(1, m + 1):
        for j in range(i + 1, m + 1):
            yield t[:i] + t[i:j + 1][::-1] + t[j + 1:]
    for L in (1, 2, 3):
        for i in range(1, m - L + 2):
            seg = t[i:i + L]
            for p in range(0, m + 1):
                if i - 1 <= p <= i + L - 1:
                    continue
                rest = [x for x in t if x not in seg]
                at = rest.index(t[p]) + 1
                yield rest[:at] + seg + rest[at:]


def random_matrix(rng, n, inf_frac=0.0, zero_frac=0.0, sym=False):
    xy = rng.uniform(0, 10, (n, 3))
    C = np.linalg.norm(xy[:, None] - xy[None], axis=2) * rng.uniform(1.0, 1.3, (n, n))
    if sym:
        C = np.minimum(C, C.T)
    C[rng.random((n, n)) < inf_frac] = np.inf
    C[rng.random((n, n)) < zero_frac] = 0.0
    np.fill_diagonal(C, 0)
    return C.astype(F32)


@pytest.mark.parametrize("seed", range(6))
def test_converged_tours_are_local_optima_and_restart_0_beats_nearest_neighbour(seed):
    rng = np.random.default_rng(seed)
    C = random_matrix(rng, 13, inf_frac=0.1 * (seed % 2), zero_frac=0.05 * (seed % 3 == 0), sym=seed % 3 == 1)
    r = tr.solve(C, restarts=5, seed=seed)
    Wi, Wq, _ = tr.weights(C)
    m = int(r["info2"][0])
    K = [g for g in range(1, 13) if np.isfinite(C[0, g])]
    assert m == len(K) and r["converged"].all()
    for t in r["tours"]:
        t = t[:m + 1].tolist()
        assert sorted(t[1:]) == K
        c = tr.tour_cost(t, Wi, Wq)
        assert all(tr.tour_cost(u, Wi, Wq) >= c for u in neighbours(t))
    nn = tr.nearest_neighbour(K, Wi, Wq)
    assert tuple(r["cost2"][0]) <= tr.tour_cost(nn, Wi, Wq)
    assert tuple(r["cost2"][r["best"]]) == min(tuple(c) for c in r["cost2"].tolist())


@pytest.mark.parametrize("seed", range(8))
def test_small_m_reaches_the_brute_force_optimum(seed):
    rng = np.random.default_rng(100 + seed)
    n = 3 + seed % 6                                                 # m = 2 .. 7
    C = random_matrix(rng, n, inf_frac=0.15 * (seed % 2))
    C[0, 1:] = np.where(np.isinf(C[0, 1:]), 1.0, C[0, 1:])           # every goal kept
    Wi, Wq, _ = tr.weights(C)
    opt = min(tr.tour_cost([0] + list(p), Wi, Wq) for p in itertools.permutations(range(1, n)))
    r = tr.solve(C, restarts=16, seed=seed)
    assert tuple(r["cost2"][r["best"]]) == opt
