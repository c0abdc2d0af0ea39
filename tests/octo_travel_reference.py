"""numpy f32 statement of the travel-cost field of a log-odds Octomap (DESIGN.md section 7, "Travel cost on the log-odds
Octomap"; csrc/tslam_octo_travel.cu).

Input: the known voxels of one submap as rows, `idx` int32[n,3] and `L` int32[n] (OctoHandle.gather()), l_occ, the
volume N, Nz, the f32 voxel scale vs; for clearance > 0 also the ESDF rows (eidx, E) of the last esdf_update
(OctoHandle.esdf_gather()).  Nothing here knows about blocks or tiles.

    traversable   FREE (known, L <= l_occ; known cells are in the volume), and with clearance > 0 an ESDF row with
                  E >= clearance (which makes it FREE at that update too: FREE voxels hold E > 0, OCC voxels E < 0)
    steps         26-neighbours at c1 = vs, c2 = f32(sqrt 2) vs, c3 = f32(sqrt 3) vs; allowed iff every cell of the box
                  the two cells span is traversable
    field         G(c0) = 0 when c0 = rha(p / vs) is traversable; G(v) = min over allowed steps of f32(G(h) + c), values
                  above max_cost dropped; unreachable cells are +inf
    path          from the target's cell, the predecessor is the reachable neighbour h with an allowed step and
                  f32(G(h) + c) == G(v), smallest G(h), ties to the first in OFFSETS order, until the start

The field iteration is Jacobi (every new value from the previous iterate), restricted after the first pass to the
neighbours of the cells that changed, as octo_esdf_reference.esdf does it; f32 min/+ is monotone and every kept step
increases the value, so the fixed point is unique and the schedule does not matter.
"""
import numpy as np

import octo_esdf_reference as oe
import octo_logodds_reference as ref

F = np.float32
INF = F(np.inf)
_BIT = {tuple(o): k for k, o in enumerate(oe.OFFSETS.tolist())}


def _box_columns():
    """per offset k: the columns (OFFSETS indices) of the box cells other than the cell itself"""
    cols = []
    for dx, dy, dz in oe.OFFSETS.tolist():
        s = {(a * dx, b * dy, c * dz) for a in (0, 1) for b in (0, 1) for c in (0, 1)} - {(0, 0, 0)}
        cols.append(sorted(_BIT[t] for t in s))
    return cols


BOX = _box_columns()
NZ = np.abs(oe.OFFSETS).sum(1)


def step_costs(vs):
    c1, c2, c3 = oe.costs(vs)
    return np.where(NZ == 1, c1, np.where(NZ == 2, c2, c3)).astype(F)


def start_cell(p, vs):
    """c0 = rha(f32(p) / f32(vs)) and whether p is finite enough to convert"""
    p = np.asarray(p, F).reshape(1, 3)
    with np.errstate(all="ignore"):
        u = p / F(vs)
    ok = bool((np.abs(u) < F(1e9)).all())
    return (ref.round_half_away(u)[0].astype(np.int64) if ok else None), ok


class Field:
    """The field of one update.  Attributes: tidx int64[m,3] traversable cells, allowed bool[m,26], nbr int64[m,26]
    (row of each neighbour among the traversable cells, m where none), G f32[m], start_ok, start row."""

    def __init__(self, idx, L, l_occ, vs, start, clearance=0.0, max_cost=None, esdf=None, chunk=1 << 18):
        idx = np.asarray(idx, np.int64).reshape(-1, 3)
        L = np.asarray(L, np.int64).reshape(-1)
        self.vs = F(vs)
        self.max_cost = F(np.ldexp(F(vs), 22)) if max_cost is None else F(max_cost)
        trav = L <= int(l_occ)
        if F(clearance) > 0:
            eidx, E = esdf
            ok = np.asarray(E, F) >= F(clearance)
            keys = np.sort(oe.pack(np.asarray(eidx, np.int64)[ok]))
            k = oe.pack(idx)
            pos = np.clip(np.searchsorted(keys, k), 0, max(keys.size - 1, 0))
            trav &= (keys[pos] == k) if keys.size else np.zeros(k.size, bool)
        self.tidx = idx[trav]
        m = self.tidx.shape[0]
        self.nbr = oe.neighbours(self.tidx)
        has = self.nbr < m
        self.allowed = np.stack([has[:, c].all(1) for c in BOX], 1) if m else np.zeros((0, 26), bool)
        self.cost = step_costs(vs)
        self.G = np.full(m, INF, F)
        c0, fin = start_cell(start, vs)
        self.start = -1
        if fin and m:
            hit = np.nonzero((self.tidx == c0[None]).all(1))[0]
            if hit.size:
                self.start = int(hit[0])
        self.start_ok = self.start >= 0
        if self.start_ok:
            self.G[self.start] = F(0)
            self._relax(chunk)

    def _relax(self, chunk):
        m = self.tidx.shape[0]
        active = np.unique(self.nbr[self.start][self.nbr[self.start] < m])
        cost = self.cost[None, :]
        while active.size:
            Gx = np.append(self.G, INF)   # row m: "no neighbour"
            new = np.empty(active.size, F)
            for s in range(0, active.size, chunk):
                a = active[s:s + chunk]
                with np.errstate(over="ignore", invalid="ignore"):
                    cand = Gx[self.nbr[a]] + cost
                cand = np.where(self.allowed[a] & (cand <= self.max_cost), cand, INF)
                new[s:s + chunk] = np.minimum(self.G[a], cand.min(1))
            ch = new < self.G[active]
            changed = active[ch]
            self.G[changed] = new[ch]
            nxt = self.nbr[changed].reshape(-1)
            active = np.unique(nxt[nxt < m])

    def reachable(self):
        """(idx int64[r,3], G f32[r]) of the reachable cells"""
        r = np.isfinite(self.G)
        return self.tidx[r], self.G[r]

    def _row(self, c):
        hit = np.nonzero((self.tidx == np.asarray(c, np.int64)[None]).all(1))[0]
        return int(hit[0]) if hit.size else -1

    def query(self, xyz, N, Nz):
        """G of the cell of each point: +inf where unreachable, outside the volume or not finite"""
        xyz = np.asarray(xyz, F).reshape(-1, 3)
        with np.errstate(all="ignore"):
            u = xyz / self.vs
        ok = (np.abs(u) < F(1e9)).all(1)
        c = ref.round_half_away(np.where(ok[:, None], u, F(0))).astype(np.int64)
        keys = oe.pack(self.tidx)
        o = np.argsort(keys)
        sk = keys[o]
        out = np.full(xyz.shape[0], INF, F)
        if sk.size == 0:
            return out
        k = oe.pack(c)
        p = np.clip(np.searchsorted(sk, k), 0, sk.size - 1)
        hit = ok & (sk[p] == k)
        out[hit] = self.G[o[p[hit]]]
        return out

    def path(self, target):
        """cells int64[len,3] from the target's cell to the start (empty when unreachable); target in metres"""
        xyz = np.asarray(target, F).reshape(1, 3)
        with np.errstate(all="ignore"):
            u = xyz / self.vs
        if not (np.abs(u) < F(1e9)).all():
            return np.zeros((0, 3), np.int64)
        v = self._row(ref.round_half_away(u)[0].astype(np.int64))
        if v < 0 or not np.isfinite(self.G[v]):
            return np.zeros((0, 3), np.int64)
        m = self.tidx.shape[0]
        out = [self.tidx[v]]
        while self.G[v] != F(0):
            best, bg = -1, INF
            for k in range(26):
                h = self.nbr[v, k]
                if h >= m or not self.allowed[v, k]:
                    continue
                gh = self.G[h]
                if gh < bg and F(gh + self.cost[k]) == self.G[v]:
                    best, bg = h, gh
            assert best >= 0, "no predecessor: the field is not a fixed point"
            v = best
            out.append(self.tidx[v])
        return np.asarray(out, np.int64)
