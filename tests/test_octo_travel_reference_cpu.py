"""The travel-cost reference (octo_travel_reference.py) on hand-worked answers, and against scipy's Dijkstra in f64."""
import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import dijkstra

import octo_esdf_reference as oe
import octo_travel_reference as tr

VS = 0.05
F = np.float32
C1, C2, C3 = oe.costs(VS)
L_OCC = 0
FREE, OCC = -400, 800


def rows(free, occ=()):
    idx = np.asarray(list(free) + list(occ), np.int64).reshape(-1, 3)
    L = np.array([FREE] * len(free) + [OCC] * len(occ), np.int64)
    return idx, L


def field(free, occ=(), start=(0, 0, 0), **kw):
    idx, L = rows(free, occ)
    return tr.Field(idx, L, L_OCC, VS, np.asarray(start, F) * F(VS), **kw)


def g_at(f, c):
    return f.query(np.asarray(c, F).reshape(-1, 3) * F(VS), 64, 64)


def seq(c, k):
    """c added k times in f32, one step at a time"""
    s = F(0)
    for _ in range(k):
        s = F(s + c)
    return s


def test_straight_corridor_sums_c1_step_by_step():
    f = field([(i, 0, 0) for i in range(60)])
    G = g_at(f, [(i, 0, 0) for i in range(60)])
    want = np.array([seq(C1, i) for i in range(60)], F)
    assert np.array_equal(G.view(np.int32), want.view(np.int32))
    assert (want != (np.arange(60) * C1).astype(F)).any()   # the sequential sums are not k * c1
    assert f.start_ok and f.reachable()[0].shape[0] == 60


def test_single_c2_and_c3_steps():
    sq = field([(i, j, 0) for i in (0, 1) for j in (0, 1)])
    assert g_at(sq, [(1, 1, 0)])[0] == C2 and g_at(sq, [(1, 0, 0)])[0] == C1
    cube = field([(i, j, k) for i in (0, 1) for j in (0, 1) for k in (0, 1)])
    assert g_at(cube, [(1, 1, 1)])[0] == C3 and g_at(cube, [(0, 1, 1)])[0] == C2


def test_diagonal_crack_forces_the_way_round():
    free = [(i, j, 0) for i in range(-1, 3) for j in range(-1, 3) if (i, j) not in ((1, 0), (0, 1))]
    f = field(free, occ=[(1, 0, 0), (0, 1, 0)])
    assert g_at(f, [(1, 1, 0)])[0] == seq(C1, 6)          # not c2 through the crack
    p = f.path(np.array([1, 1, 0], F) * F(VS))
    assert p.shape[0] == 7 and (p[-1] == 0).all()
    steps = np.abs(np.diff(p, axis=0)).sum(1)
    assert (steps == 1).all()


def test_unknown_slab_blocks():
    free = [(i, j, k) for i in range(5) for j in range(-2, 3) for k in range(-2, 3) if i != 2]
    f = field(free)
    G = g_at(f, [(1, 0, 0), (3, 0, 0), (4, 2, 2)])
    assert np.isfinite(G[0]) and np.isinf(G[1:]).all()
    assert f.reachable()[0].shape[0] == 2 * 25


def test_clearance_excludes_cells_next_to_an_obstacle():
    free = [(i, j, 0) for i in range(-3, 4) for j in range(-3, 4) if (i, j) != (0, 0)]
    idx, L = rows(free, [(0, 0, 0)])
    E = oe.esdf(idx, L, L_OCC, VS, 1.0)
    f = tr.Field(idx, L, L_OCC, VS, np.array([3, 3, 0], F) * F(VS), clearance=0.06, esdf=(idx, E))
    assert f.tidx.shape[0] == 48 - 4                       # the four face neighbours hold c1 < 0.06; diagonals c2 >= 0.06
    G = g_at(f, [(1, 0, 0), (0, -1, 0), (1, 1, 0), (-3, -3, 0)])
    assert np.isinf(G[:2]).all() and np.isfinite(G[2:]).all()
    # clearance 0: every FREE cell
    assert tr.Field(idx, L, L_OCC, VS, np.zeros(3, F)).tidx.shape[0] == 48


def test_max_cost_kept_at_the_value_dropped_one_ulp_below():
    free = [(i, 0, 0) for i in range(10)]
    g3 = seq(C1, 3)
    at = field(free, max_cost=g3)
    G = g_at(at, [(3, 0, 0), (4, 0, 0)])
    assert G[0] == g3 and np.isinf(G[1])
    below = field(free, max_cost=np.nextafter(g3, F(0)))
    G = g_at(below, [(2, 0, 0), (3, 0, 0)])
    assert G[0] == seq(C1, 2) and np.isinf(G[1])
    assert below.reachable()[0].shape[0] == 3


def test_invalid_starts():
    free = [(i, j, 0) for i in range(-3, 4) for j in range(-3, 4) if (i, j) != (0, 0)]
    idx, L = rows(free, [(0, 0, 0)])
    E = oe.esdf(idx, L, L_OCC, VS, 1.0)
    starts = dict(unknown=(0, 0, 5), occ=(0, 0, 0), outside=(100000, 0, 0), nan=(np.nan, 0, 0), inf=(0, np.inf, 0))
    for name, s in starts.items():
        f = tr.Field(idx, L, L_OCC, VS, np.asarray(s, F) * F(VS))
        assert not f.start_ok and f.reachable()[0].shape[0] == 0 and np.isinf(f.G).all(), name
    near = tr.Field(idx, L, L_OCC, VS, np.array([1, 0, 0], F) * F(VS), clearance=0.06, esdf=(idx, E))
    assert not near.start_ok and near.reachable()[0].shape[0] == 0
    assert near.tidx.shape[0] == 44                         # traversable cells are still counted


def test_path_tie_rule_and_paths_end_at_the_start():
    free = [(i, j, 0) for i in range(3) for j in (-1, 0, 1) if (i, j) != (1, 0)]
    f = field(free, occ=[(1, 0, 0)])
    assert g_at(f, [(2, 0, 0)])[0] == seq(C1, 4)
    p = f.path(np.array([2, 0, 0], F) * F(VS))
    # (2,1,0) and (2,-1,0) are both predecessors at 3 c1: the first in OFFSETS order, dy = -1, wins
    assert p.tolist() == [[2, 0, 0], [2, -1, 0], [1, -1, 0], [0, -1, 0], [0, 0, 0]]
    assert f.path(np.zeros(3, F)).tolist() == [[0, 0, 0]]
    assert f.path(np.array([1, 0, 0], F) * F(VS)).shape[0] == 0      # OCC target
    assert f.path(np.array([np.nan, 0, 0], F)).shape[0] == 0
    # the smallest G(h) wins over the OFFSETS order: into (1,1,0) of a 2x2 square both (0,0,0) + c2 and nothing else
    sq = field([(i, j, 0) for i in (0, 1) for j in (0, 1)])
    assert sq.path(np.array([1, 1, 0], F) * F(VS)).tolist() == [[1, 1, 0], [0, 0, 0]]


def blob(seed, n=12):
    rng = np.random.default_rng(seed)
    c = np.argwhere(np.ones((n, n, n), bool)) - n // 2
    r = rng.uniform(size=len(c))
    free, occ = c[r < 0.75], c[(r >= 0.75) & (r < 0.85)]
    free = np.concatenate([free, np.zeros((1, 3), np.int64)]) if not (free == 0).all(1).any() else free
    occ = occ[~(occ == 0).all(1)]
    return free, occ


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_blobs_match_dijkstra_in_f64(seed):
    free, occ = blob(seed)
    f = field(free, occ)
    m = f.tidx.shape[0]
    w = np.where(tr.NZ == 1, VS, np.where(tr.NZ == 2, np.sqrt(2.0) * VS, np.sqrt(3.0) * VS))
    src, dst, wt = [], [], []
    for k in range(26):
        ok = f.allowed[:, k] & (f.nbr[:, k] < m)
        src.append(f.nbr[ok, k]); dst.append(np.nonzero(ok)[0]); wt.append(np.full(ok.sum(), w[k]))
    A = csr_matrix((np.concatenate(wt), (np.concatenate(src), np.concatenate(dst))), shape=(m, m))
    D = dijkstra(A, indices=f.start)
    assert np.array_equal(np.isfinite(D), np.isfinite(f.G))
    r = np.isfinite(D)
    assert r.sum() > 100
    Gd = f.G[r].astype(np.float64)
    tol = D[r] * (D[r] / VS + 4) * 2.0 ** -22
    assert (np.abs(Gd - D[r]) <= tol).all()
    # every reachable cell's path ends at the start with strictly decreasing costs
    for v in np.nonzero(r)[0][:: max(1, r.sum() // 40)]:
        p = f.path(f.tidx[v].astype(F) * F(VS))
        assert (p[-1] == f.tidx[f.start]).all()
        Gp = g_at(f, p)
        assert (np.diff(Gp) < 0).all()
