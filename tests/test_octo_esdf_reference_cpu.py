"""The occupancy-ESDF reference (octo_esdf_reference.py) on hand-worked answers."""
import heapq
import itertools

import numpy as np

import octo_esdf_reference as oe

F = np.float32
VS = 0.05
L_OCC = 0
OCC, FREE = 868, -415


def box(shape, occ_cells=(), unknown=None):
    """Fully known box of FREE voxels with OCC cells; unknown: bool mask of cells without a row."""
    g = np.argwhere(np.ones(shape, bool))
    L = np.full(len(g), FREE, np.int64)
    key = {tuple(c): r for r, c in enumerate(g.tolist())}
    for c in occ_cells:
        L[key[tuple(c)]] = OCC
    keep = np.ones(len(g), bool) if unknown is None else ~unknown[tuple(g.T)]
    return g[keep].astype(np.int32), L[keep]


def table(idx, E):
    return {tuple(c): v for c, v in zip(idx.tolist(), E.tolist())}


def seq_sum(k):
    s = F(0)
    for _ in range(k):
        s = F(s + F(VS))
    return s


def test_single_occupied_voxel():
    c = (7, 7, 7)
    idx, L = box((15, 15, 15), [c])
    E = table(idx, oe.esdf(idx, L, L_OCC, VS, 10.0))
    c1, c2, c3 = oe.costs(VS)
    assert E[c] == -F(VS)
    for d in itertools.product((-1, 0, 1), repeat=3):
        nz = sum(x != 0 for x in d)
        if nz:
            assert E[tuple(np.add(c, d))] == (c1, c2, c3)[nz - 1], d
    for k in range(1, 8):
        for ax in range(3):
            for sgn in (-1, 1):
                p = list(c)
                p[ax] += sgn * k
                assert E[tuple(p)] == seq_sum(k), (k, ax, sgn)


def chamfer(d):
    a, b, c = sorted(np.abs(d).tolist(), reverse=True)
    return c * np.sqrt(3.0) + (b - c) * np.sqrt(2.0) + (a - b)


def test_random_sparse_sites_match_closed_form():
    rng = np.random.default_rng(5)
    shape = (24, 20, 16)
    sites = {tuple(int(v) for v in rng.integers(0, shape)) for _ in range(12)}
    idx, L = box(shape, sites)
    E = oe.esdf(idx, L, L_OCC, VS, 100.0)
    S = np.array(sorted(sites))
    occ = L > L_OCC
    for r in np.nonzero(~occ)[0]:
        dd = [chamfer(idx[r] - s) for s in S]
        steps = max(np.abs(idx[r] - S[int(np.argmin(dd))]).max(), 1)
        want = min(dd) * VS
        assert abs(float(E[r]) - want) <= (steps + 2) * 2.0 ** -23 * want, (idx[r], E[r], want)
    isolated = [r for r in np.nonzero(occ)[0]]
    assert all(E[r] == -F(VS) for r in isolated)   # every site has a FREE 6-neighbour


def test_occupied_cube():
    cube = [tuple(np.add((5, 5, 5), d)) for d in itertools.product((-1, 0, 1), repeat=3)]
    idx, L = box((11, 11, 11), cube)
    E = table(idx, oe.esdf(idx, L, L_OCC, VS, 10.0))
    assert E[(5, 5, 5)] == -F(F(VS) + F(VS))
    for d in itertools.product((-1, 0, 1), repeat=3):
        if sum(x != 0 for x in d):
            assert E[tuple(np.add((5, 5, 5), d))] == -F(VS), d   # faces, edges, corners touch free space


def test_truncation():
    D = 2.5 * VS
    idx, L = box((15, 3, 3), [(0, 1, 1)])
    E = table(idx, oe.esdf(idx, L, L_OCC, VS, D))
    assert E[(1, 1, 1)] == F(VS) and E[(2, 1, 1)] == seq_sum(2)
    assert all(E[(k, 1, 1)] == F(D) for k in range(3, 15))
    assert max(E.values()) == F(D)


def dijkstra(idx, occ, src_rows, vs):
    """f64 26-neighbour chamfer distance from the given OCC rows over the known FREE voxels."""
    key = {tuple(c): r for r, c in enumerate(idx.tolist())}
    dist = np.full(len(idx), np.inf)
    pq = []
    for r in src_rows:
        for d in oe.OFFSETS.tolist():
            h = key.get(tuple(np.add(idx[r], d)))
            if h is not None and not occ[h]:
                c = np.sqrt(sum(x != 0 for x in d)) * vs
                if c < dist[h]:
                    dist[h] = c
                    heapq.heappush(pq, (c, h))
    while pq:
        dv, v = heapq.heappop(pq)
        if dv > dist[v]:
            continue
        for d in oe.OFFSETS.tolist():
            h = key.get(tuple(np.add(idx[v], d)))
            if h is None or occ[h]:
                continue
            nd = dv + np.sqrt(sum(x != 0 for x in d)) * vs
            if nd < dist[h]:
                dist[h] = nd
                heapq.heappush(pq, (nd, h))
    return dist


def test_paths_go_around_unknown_space():
    shape = (20, 20, 3)
    unknown = np.zeros(shape, bool)
    unknown[8:10, :, :] = True        # an unknown slab across x = 8..9 ...
    unknown[8:10, 17:19, :] = False   # ... with a known hole at y = 17..18
    src = (3, 5, 1)
    idx, L = box(shape, [src], unknown)
    E = oe.esdf(idx, L, L_OCC, VS, 100.0)
    occ = L > L_OCC
    want = dijkstra(idx, occ, np.nonzero(occ)[0], VS)
    free = ~occ
    assert np.all(np.abs(E[free] - want[free]) <= 64 * 2.0 ** -23 * want[free])
    T = table(idx, E)
    behind = (12, 5, 1)
    assert T[behind] > chamfer(np.subtract(behind, src)) * VS * 2   # the straight path is cut by the slab
    assert T[behind] < 100.0


def test_isolated_known_voxels_keep_D():
    idx = np.array([[0, 0, 0], [5, 5, 5], [9, 0, 0], [10, 0, 0]], np.int32)
    L = np.array([FREE, OCC, FREE, FREE])
    E = oe.esdf(idx, L, L_OCC, VS, 1.0)
    assert E.tolist() == [F(1.0), F(-1.0), F(1.0), F(1.0)]
    # two OCC voxels next to each other and nothing free: both stay -D
    E = oe.esdf(np.array([[0, 0, 0], [1, 0, 0]], np.int32), np.array([OCC, OCC]), L_OCC, VS, 1.0)
    assert E.tolist() == [F(-1.0), F(-1.0)]
