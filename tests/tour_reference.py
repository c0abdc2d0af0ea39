"""numpy statement of tslam_tour_open (include/tslam.h, DESIGN.md section 7 "Exploration tours"), in int64 / uint64.

A leg weighs (inf, q): (1, 0) for +inf, (0, x / U) for a finite entry x, U = 2^(e_lo - 23).  Tour costs are sums of
those pairs, compared lexicographically.  Every move of a step is evaluated at once (vectorised) in the contract's move
order, and the first least delta is taken.  The tour is padded with a sentinel node n whose legs weigh (0, 0), which
makes "after the last node" an ordinary position, as in the kernel."""
import numpy as np

MAX_N = 1024
MAX_RESTARTS = 4096
MAX_RANGE = 28
M64 = (1 << 64) - 1


class Refused(ValueError):
    """what the library refuses with TSLAM_E_INVALID"""


def mix64(z):
    """the SplitMix64 finaliser on a Python int, wrapping at 2^64"""
    z &= M64
    z ^= z >> 30
    z = (z * 0xbf58476d1ce4e5b9) & M64
    z ^= z >> 27
    z = (z * 0x94d049bb133111eb) & M64
    z ^= z >> 31
    return z


def shuffle(K, seed, r):
    """Fisher-Yates of the ascending kept goals K for restart r >= 1"""
    a = list(K)
    for i in range(len(a) - 1, 0, -1):
        j = mix64((seed & M64) ^ ((r << 32) & M64) ^ i) % (i + 1)
        a[i], a[j] = a[j], a[i]
    return a


def weights(C):
    """-> (Wi int64[n+1,n+1], Wq int64[n+1,n+1], e_lo) of a valid matrix, row / column n the sentinel; raises Refused"""
    C = np.asarray(C, np.float32)
    if C.ndim != 2 or C.shape[0] != C.shape[1] or not 1 <= C.shape[0] <= MAX_N:
        raise Refused(f"the matrix must be [n, n] with 1 <= n <= {MAX_N}, not {C.shape}")
    n = C.shape[0]
    off = ~np.eye(n, dtype=bool)
    x = C[off]
    if np.isnan(x).any():
        raise Refused("NaN")
    if (x < 0).any():
        raise Refused("negative value")
    pos = x[(x > 0) & np.isfinite(x)]
    if (pos < np.finfo(np.float32).tiny).any():
        raise Refused("subnormal value")
    e_lo = e_hi = 0
    if pos.size:
        e = np.frexp(pos)[1].astype(np.int64) - 1  # floor(log2 x) of a normal f32
        e_lo, e_hi = int(e.min()), int(e.max())
    if e_hi - e_lo > MAX_RANGE:
        raise Refused(f"range {e_hi - e_lo} > {MAX_RANGE}")
    Wi = np.zeros((n + 1, n + 1), np.int64)
    Wq = np.zeros((n + 1, n + 1), np.int64)
    Wi[:n, :n] = np.isinf(C) & off
    fin = np.isfinite(C) & off
    Wq[:n, :n][fin] = np.ldexp(C[fin].astype(np.float64), 23 - e_lo).astype(np.int64)  # exact: < 2^52
    return Wi, Wq, e_lo


def tour_cost(t, Wi, Wq):
    """(inf, q) of the open tour t as Python ints"""
    t = np.asarray(t)
    return int(Wi[t[:-1], t[1:]].sum()), int(Wq[t[:-1], t[1:]].sum())


def nearest_neighbour(K, Wi, Wq):
    t, left, cur = [0], list(K), 0
    while left:
        g = min(left, key=lambda g: (Wi[cur, g], Wq[cur, g], g))
        t.append(g)
        left.remove(g)
        cur = g
    return t


def _moves(m):
    """the move list in contract order: kind (0 2-opt, L Or-opt), i, j or p"""
    cached = _moves.cache.get(m)
    if cached is None:
        I, J = np.triu_indices(m + 1, 1)
        keep = I >= 1
        kinds, Is, Js = [np.zeros(keep.sum(), np.int64)], [I[keep]], [J[keep]]
        for L in (1, 2, 3):
            II, PP = np.meshgrid(np.arange(1, m - L + 2), np.arange(m + 1), indexing="ij")
            E = II + L - 1
            v = ((PP < II - 1) | (PP > E)).ravel()
            kinds.append(np.full(v.sum(), L, np.int64))
            Is.append(II.ravel()[v])
            Js.append(PP.ravel()[v])
        cached = _moves.cache[m] = (np.concatenate(kinds), np.concatenate(Is).astype(np.int64), np.concatenate(Js).astype(np.int64))
    return cached


_moves.cache = {}


def deltas(t, Wi, Wq):
    """(kind, i, j/p, d_inf, d_q) of every move on tour t (list, t[0] = 0), in contract order"""
    m = len(t) - 1
    n = Wi.shape[0] - 1
    te = np.array(list(t) + [n], np.int64)
    kind, I, J = _moves(m)
    out = []
    for W in (Wi, Wq):
        F = np.concatenate([[0], np.cumsum(W[te[:-1], te[1:]])])       # F[k] = sum_{p<k} w(t[p], t[p+1]), k <= m + 1
        Rv = np.concatenate([[0], np.cumsum(W[te[1:-1], te[:-2]])])    # Rv[k] = sum_{p<k} w(t[p+1], t[p]), k <= m
        d = np.empty(kind.shape[0], np.int64)
        two = kind == 0
        i, j = I[two], J[two]
        d[two] = W[te[i - 1], te[j]] + W[te[i], te[j + 1]] + Rv[j] - Rv[i] - F[j + 1] + F[i - 1]
        o = ~two
        i, p, L = I[o], J[o], kind[o]
        e = i + L - 1
        d[o] = (W[te[i - 1], te[e + 1]] - (F[i] - F[i - 1]) - (F[e + 1] - F[e])
                + W[te[p], te[i]] + W[te[e], te[p + 1]] - (F[p + 1] - F[p]))
        out.append(d)
    return kind, I, J, out[0], out[1]


def apply_move(t, kind, i, j):
    t = list(t)
    if kind == 0:
        t[i:j + 1] = t[i:j + 1][::-1]
        return t
    e = i + kind - 1
    seg = t[i:e + 1]
    rest = t[:i] + t[e + 1:]
    at = j + 1 if j < i else j - kind + 1  # the position after t[p] in `rest`
    return rest[:at] + seg + rest[at:]


def best_move(t, Wi, Wq):
    """the move the contract applies, (kind, i, j/p, d_inf, d_q), or None when no move improves"""
    if len(t) <= 2:
        return None
    kind, I, J, di, dq = deltas(t, Wi, Wq)
    mi = di.min()
    qm = dq[di == mi].min()
    if not (mi < 0 or (mi == 0 and qm < 0)):
        return None
    k = int(np.argmax((di == mi) & (dq == qm)))
    return int(kind[k]), int(I[k]), int(J[k]), int(mi), int(qm)


def search(t, Wi, Wq, max_passes):
    """-> (tour, passes, converged)"""
    passes = 0
    while True:
        mv = best_move(t, Wi, Wq)
        if mv is None:
            return t, passes, True
        if passes == max_passes:
            return t, passes, False
        t = apply_move(t, *mv[:3])
        passes += 1


def solve(C, restarts=64, seed=0, max_passes=None):
    """tslam_tour_open -> dict(tours int32[R,n], cost2 int64[R,2], passes int32[R], converged uint8[R], best, info2)"""
    Wi, Wq, e_lo = weights(C)
    n = Wi.shape[0] - 1
    R = int(restarts)
    if not 1 <= R <= MAX_RESTARTS:
        raise Refused(f"restarts {R}")
    mp = 64 * n if max_passes is None else int(max_passes)
    if mp < 0:
        raise Refused(f"max_passes {mp}")
    K = [g for g in range(1, n) if Wi[0, g] == 0]
    m = len(K)
    tours = np.full((R, n), -1, np.int32)
    cost2 = np.zeros((R, 2), np.int64)
    passes = np.zeros(R, np.int32)
    conv = np.zeros(R, np.uint8)
    for r in range(R):
        t0 = nearest_neighbour(K, Wi, Wq) if r == 0 else [0] + shuffle(K, seed, r)
        t, passes[r], c = search(t0, Wi, Wq, mp)
        conv[r] = c
        tours[r, :m + 1] = t
        cost2[r] = tour_cost(t, Wi, Wq)
    best = min(range(R), key=lambda r: (cost2[r, 0], cost2[r, 1], r))
    return dict(tours=tours, cost2=cost2, passes=passes, converged=conv, best=best, info2=np.array([m, e_lo - 23], np.int32))
