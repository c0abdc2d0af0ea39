"""What the many-source travel costs promise, pinned on the single-source reference (octo_travel_reference.py; the
many-source reference is one tr.Field per start): the cost matrix is not symmetric in the last bits, both directions lie
within an f32 rounding bound of the f64 Dijkstra value, and reachability is symmetric under the default max_cost."""
import numpy as np
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import dijkstra

import octo_travel_reference as tr
from test_octo_travel_reference_cpu import VS, blob, field, g_at

F = np.float32


def rounding_bound(d):
    """|G - D| for an f32 path sum G of f64 length D (the bound test_octo_travel_reference_cpu checks on random blobs)"""
    return d * (d / VS + 4) * 2.0 ** -22


def dijkstra_f64(f):
    """f64 Dijkstra distances over f's traversable cells and allowed steps, from f's start"""
    m = f.tidx.shape[0]
    w = np.where(tr.NZ == 1, VS, np.where(tr.NZ == 2, np.sqrt(2.0) * VS, np.sqrt(3.0) * VS))
    src, dst, wt = [], [], []
    for k in range(26):
        ok = f.allowed[:, k] & (f.nbr[:, k] < m)
        src.append(f.nbr[ok, k]); dst.append(np.nonzero(ok)[0]); wt.append(np.full(ok.sum(), w[k]))
    A = csr_matrix((np.concatenate(wt), (np.concatenate(src), np.concatenate(dst))), shape=(m, m))
    return dijkstra(A, indices=f.start)


def test_a_pair_whose_two_directions_differ_in_f32():
    free, occ = blob(1, 16)
    s, t = (-4, -7, -8), (5, -7, -3)                       # found by search on this blob
    fs, ft = field(free, occ, start=s), field(free, occ, start=t)
    assert fs.start_ok and ft.start_ok
    g_st, g_ts = g_at(fs, [t])[0], g_at(ft, [s])[0]
    assert g_st == F(0.5828427) and g_ts == F(0.58284277) and g_st != g_ts
    # both are f32 sums of one minimal path, added in opposite orders: each within the rounding bound of Dijkstra in f64
    D = dijkstra_f64(fs)[ft.start]
    assert D == dijkstra_f64(ft)[fs.start]
    for g in (g_st, g_ts):
        assert abs(float(g) - D) <= rounding_bound(D)
    assert abs(float(g_st) - float(g_ts)) <= 2 * rounding_bound(D)
    # a max_cost between the two makes reachability one-sided: the default limit is what keeps it symmetric
    lo = min(g_st, g_ts)
    one = field(free, occ, start=s, max_cost=lo)
    other = field(free, occ, start=t, max_cost=lo)
    assert np.isfinite(g_at(one, [t])[0]) != np.isfinite(g_at(other, [s])[0])


def test_reachability_is_symmetric_under_the_default_limit():
    for seed in (0, 2):
        free, occ = blob(seed, 14)
        rng = np.random.default_rng(seed)
        starts = np.concatenate([free[rng.choice(len(free), 20, replace=False)], occ[:2], [[50, 0, 0]]])
        fields = [field(free, occ, start=p) for p in starts]
        M = np.stack([g_at(f, starts) for f in fields])
        fin = np.isfinite(M)
        assert np.array_equal(fin, fin.T)
        assert (~fin).any() and fin.sum() > 200             # some pairs are cut off (OCC and outside starts, pockets)
        ok = np.array([f.start_ok for f in fields])
        assert (np.diag(M)[ok] == 0).all() and np.isinf(np.diag(M)[~ok]).all()
        asym = fin & (M != M.T)
        assert asym.any()                                   # not symmetric in the last bits ...
        hi = np.where(fin, np.maximum(M, M.T), 0).astype(np.float64) * (1 + 2.0 ** -18)
        assert (np.abs(M[fin] - M.T[fin]) <= 2 * rounding_bound(hi[fin])).all()   # ... but within the rounding bound
