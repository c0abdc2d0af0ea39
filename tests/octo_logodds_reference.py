"""numpy f32 restatement of the log-odds Octomap (DESIGN.md section 7, "Log-odds Octomap"): what one integrate call
does to the map, and how fusion, the planner queries and the LoD export read it.  Every f32 expression is written in
the kernels' operation order (the library builds with -fmad=false, so each operation rounds once), so the GPU state
must equal this one bit for bit.  The reference project has no such model to execute; this module is the oracle.

State: per submap, sorted packed cell keys and their int32 L (Q10 log-odds).  A cell that is absent is unknown.
"""
import math

import numpy as np

from march_reference import round_half_away

f32 = np.float32
_OFF = 1 << 20


def q10(p):
    """l = round_half_away(logit(p) * 1024), in f64."""
    return int(round_half_away(np.array([math.log(p / (1.0 - p)) * 1024.0]))[0])


def params(prob_hit=0.7, prob_miss=0.4, prob_min=0.1192, prob_max=0.971, prob_occupied=0.5):
    return dict(l_hit=q10(prob_hit), l_miss=q10(prob_miss), l_min=q10(prob_min), l_max=q10(prob_max), l_occ=q10(prob_occupied))


def pack(c):
    c = np.asarray(c, np.int64).reshape(-1, 3) + _OFF
    return (c[:, 0] << 42) | (c[:, 1] << 21) | c[:, 2]


def unpack(k):
    k = np.asarray(k, np.int64)
    return np.stack([(k >> 42) & ((1 << 21) - 1), (k >> 21) & ((1 << 21) - 1), k & ((1 << 21) - 1)], 1) - _OFF


def cells(p, vs):
    """xyz_to_sijk: round_half_away(x / vs) per axis, x and vs f32."""
    return round_half_away(np.asarray(p, f32) / f32(vs))


def _mat(R, T):
    return np.asarray(R, np.float64).astype(f32).reshape(3, 3), np.asarray(T, np.float64).astype(f32).reshape(3)


def _rot(R, x, y, z):
    """((R0 x + R1 y) + R2 z) per row, f32."""
    return [(R[r, 0] * x + R[r, 1] * y) + R[r, 2] * z for r in range(3)]


def depth_endpoints(depth, R, T, K, min_ray, max_ray, step):
    """k_octo_lo_depth: (endpoints f32 [n,3], clipped bool [n]) of the sampled pixels that cast a ray, in pixel order."""
    R, T = _mat(R, T)
    fx, fy, cx, cy = (f32(K[0]), f32(K[4]), f32(K[2]), f32(K[5]))
    dmin, dmax = f32(min_ray * 1000.0), f32(max_ray * 1000.0)
    h, w = depth.shape
    hh, ww = int(h / step), int(w / step)
    jj, ii = np.meshgrid(np.arange(hh), np.arange(ww), indexing="ij")
    j, i = (jj * step).reshape(-1), (ii * step).reshape(-1)
    d = np.asarray(depth)[j, i]
    df = d.astype(f32)
    valid = (d != 0) & ~(df < dmin)
    j, i, df = j[valid], i[valid], df[valid]
    clipped = df > dmax
    dep = np.where(clipped, f32(max_ray), df / f32(1000.0)).astype(f32)
    x = ((i.astype(f32) - cx) * dep) / fx
    y = ((j.astype(f32) - cy) * dep) / fy
    p = _rot(R, x, y, dep)
    return np.stack([p[0] + T[0], p[1] + T[1], p[2] + T[2]], 1).astype(f32), clipped


def point_endpoints(xyz, R, T, min_ray, max_ray):
    """k_octo_lo_points: range r = |R p|; r < min_ray or not finite -> no ray; r > max_ray -> cut at max_ray."""
    R, T = _mat(R, T)
    xyz = np.asarray(xyz, f32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        r3 = _rot(R, xyz[:, 0], xyz[:, 1], xyz[:, 2])
        r = np.sqrt((r3[0] * r3[0] + r3[1] * r3[1]) + r3[2] * r3[2])
        valid = (r >= f32(min_ray)) & (r < np.inf)
        clipped = r > f32(max_ray)
        sc = f32(max_ray) / r
        p = [np.where(clipped, a * sc, a).astype(f32) for a in r3]
    e = np.stack([p[0] + T[0], p[1] + T[1], p[2] + T[2]], 1).astype(f32)
    return e[valid], clipped[valid]


def walk(origin, ends, clipped, vs):
    """k_octo_lo_walk.  Amanatides-Woo in voxel units from c0 = cell(origin) to c1 = cell(end): t of the next boundary of
    axis a = ((c_a + 0.5 s_a) - p0_a) * (1 / (p1_a - p0_a)), recomputed from the current cell; each step takes the axis
    with the smallest t among those with steps left, ties to the lower axis.  Returns (ray, cell) of every miss visit in
    path order per ray: all cells before c1, and c1 itself when the ray was clipped."""
    vs = f32(vs)
    p0 = np.asarray(origin, f32).reshape(3) / vs
    p1 = np.asarray(ends, f32).reshape(-1, 3) / vs
    n = p1.shape[0]
    c0 = round_half_away(p0)
    c1 = round_half_away(p1)
    left = np.abs(c1 - c0)
    s = np.where(c1 > c0, 1, -1)
    h = (f32(0.5) * s.astype(f32)).astype(f32)
    with np.errstate(divide="ignore"):
        inv = np.where(left > 0, f32(1.0) / (p1 - p0), f32(0.0)).astype(f32)
    c = np.broadcast_to(c0, (n, 3)).copy()
    tm = (((c.astype(f32) + h) - p0) * inv).astype(f32)
    rem = left.sum(1)
    clipped = np.asarray(clipped, bool)
    rays, out = [], []
    act = np.arange(n)
    while act.size:
        emit = act[(rem[act] > 0) | clipped[act]]
        rays.append(emit)
        out.append(c[emit].copy())
        act = act[rem[act] > 0]
        if not act.size:
            break
        lx, ly, lz = left[act, 0] > 0, left[act, 1] > 0, left[act, 2] > 0
        a = np.full(act.size, 3)
        tb = np.zeros(act.size, f32)
        a[lx], tb[lx] = 0, tm[act[lx], 0]
        m = ly & ((a == 3) | (tm[act, 1] < tb))
        a[m], tb[m] = 1, tm[act[m], 1]
        m = lz & ((a == 3) | (tm[act, 2] < tb))
        a[m] = 2
        c[act, a] += s[act, a]
        left[act, a] -= 1
        rem[act] -= 1
        tm[act, a] = ((c[act, a].astype(f32) + h[act, a]) - p0[a]) * inv[act, a]
    if not rays:
        return np.zeros(0, np.int64), np.zeros((0, 3), np.int64)
    return np.concatenate(rays), np.concatenate(out)


class LogoddsMap:
    """Reference state of a log-odds Octomap: N x N x Nz cells, i in [-N/2, N - N/2), per submap."""

    def __init__(self, N, Nz, voxel_scale, min_ray_length=0.3, max_ray_length=3.0, recast_step=2, K=None, **prob):
        self.N, self.Nz, self.vs = N, Nz, voxel_scale
        self.hN, self.hNz = N // 2, Nz // 2
        self.min_ray, self.max_ray, self.step = min_ray_length, max_ray_length, recast_step
        self.K = K
        self.p = params(**prob)
        self.maps = {}
        self.stats = np.zeros(4, np.int64)

    def in_bounds(self, c):
        c = np.asarray(c).reshape(-1, 3)
        return ((c[:, 0] >= -self.hN) & (c[:, 0] < self.N - self.hN) & (c[:, 1] >= -self.hN) & (c[:, 1] < self.N - self.hN)
                & (c[:, 2] >= -self.hNz) & (c[:, 2] < self.Nz - self.hNz))

    def state(self, submap=0):
        return self.maps.get(submap, (np.zeros(0, np.int64), np.zeros(0, np.int32)))

    def frame(self, origin, ends, clipped, submap=0):
        """One integrate call: rays from origin (f32 sensor position, map frame) to ends."""
        ends = np.asarray(ends, f32).reshape(-1, 3)
        clipped = np.asarray(clipped, bool)
        hc = cells(ends[~clipped], self.vs)
        H = np.unique(pack(hc[self.in_bounds(hc)]))
        _, mc = walk(origin, ends, clipped, self.vs)
        mc = mc[self.in_bounds(mc)]
        M = np.setdiff1d(np.unique(pack(mc)), H)
        U = np.concatenate([H, M])
        inc = np.concatenate([np.full(H.size, self.p["l_hit"]), np.full(M.size, self.p["l_miss"])]).astype(np.int64)
        keys, L = self.state(submap)
        uk = np.union1d(keys, U)
        Lf = np.zeros(uk.size, np.int64)
        Lf[np.searchsorted(uk, keys)] = L
        iu = np.searchsorted(uk, U)
        Lf[iu] = np.clip(Lf[iu] + inc, self.p["l_min"], self.p["l_max"])
        self.maps[submap] = (uk, Lf.astype(np.int32))
        self.stats += [ends.shape[0], mc.shape[0], H.size, U.size]

    def integrate_depth(self, depth, R, T, submap=0):
        e, cl = depth_endpoints(depth, R, T, self.K, self.min_ray, self.max_ray, self.step)
        self.frame(np.asarray(T, np.float64).astype(f32), e, cl, submap)

    def integrate_points(self, xyz, R, T, submap=0):
        e, cl = point_endpoints(xyz, R, T, self.min_ray, self.max_ray)
        self.frame(np.asarray(T, np.float64).astype(f32), e, cl, submap)

    def gather(self, submap=0):
        """(idx int32 [n,3], L int32 [n]) of the known cells, in key order."""
        keys, L = self.state(submap)
        return unpack(keys).astype(np.int32), L.copy()

    # -- readers ----------------------------------------------------------------------------------------------------
    def _lookup(self, c, submap):
        keys, L = self.state(submap)
        k = pack(c)
        pos = np.clip(np.searchsorted(keys, k), 0, max(keys.size - 1, 0))
        known = (keys.size > 0) & (keys[pos] == k) if keys.size else np.zeros(k.size, bool)
        known = known & self.in_bounds(c)
        val = np.where(known, L[pos] if keys.size else 0, 0)
        return known, val

    def occupied_cells(self, c, submap=0):
        known, val = self._lookup(c, submap)
        return known & (val > self.p["l_occ"]), known

    def query_points(self, xyz, submap=0):
        """(occupied, unknown) of the points' cells (k_query_points<OcProbe<OcLogodds>>)."""
        occ, known = self.occupied_cells(cells(xyz, self.vs), submap)
        return occ, ~known

    def query_near(self, xyz, voxel, submap=0):
        c0 = cells(xyz, self.vs)
        out = np.zeros(c0.shape[0], bool)
        r = range(-voxel, voxel)
        for a in r:
            for b in r:
                for d in r:
                    out |= self.occupied_cells(c0 + np.array([a, b, d]), submap)[0]
        return out

    def raycast(self, pos, dirs, max_dist, submap=0):
        """BaseMap.raycast: samples at len = j * vs, x = d * len + p, until the first occupied cell."""
        vs = f32(self.vs)
        pos, dirs = np.asarray(pos, f32).reshape(-1, 3), np.asarray(dirs, f32).reshape(-1, 3)
        n = pos.shape[0]
        steps = int(f32(max_dist) / vs)
        hit = np.zeros(n, bool)
        x = np.zeros((n, 3), f32)
        ln = np.zeros(n, f32)
        act = np.arange(n)
        for j in range(steps):
            if not act.size:
                break
            le = f32(j) * vs
            xa = (dirs[act] * le + pos[act]).astype(f32)
            x[act], ln[act] = xa, le
            occ = self.occupied_cells(cells(xa, vs), submap)[0]
            hit[act[occ]] = True
            act = act[~occ]
        return hit, x, ln

    def export(self, level, K=2, R=None, T=None, submap=0):
        """cvt_occupy_to_voxels(level): corner voxels of K^(level-1) groups that are known and L > l_occ, at f32
        position R (i vs) + T (the submap's pose-table row)."""
        group = K ** (max(int(level), 1) - 1)
        idx, L = self.gather(submap)
        idx = idx.astype(np.int64)
        keep = (L > self.p["l_occ"]) & ((idx[:, 0] + self.hN) % group == 0) & ((idx[:, 1] + self.hN) % group == 0) \
            & ((idx[:, 2] + self.hNz) % group == 0)
        li = idx[keep].astype(f32) * f32(self.vs)
        Rm, Tm = _mat(np.eye(3) if R is None else R, np.zeros(3) if T is None else T)
        p = _rot(Rm, li[:, 0], li[:, 1], li[:, 2])
        return np.stack([p[0] + Tm[0], p[1] + Tm[1], p[2] + Tm[2]], 1).astype(f32)


def fuse(dst, src, poses):
    """fuse_submaps on log-odds maps: every known voxel of every source submap s adds its L to the target cell
    round((R_s (i vs) + T_s) / vs) of submap 0; one clamp once all sums are in.  poses: {s: (R, T)} of dst's table."""
    dst.maps = {}
    vs = f32(dst.vs)
    allk, allL = [], []
    for s, (keys, L) in src.maps.items():
        R, T = _mat(*poses[s])
        li = unpack(keys).astype(f32) * vs
        p = _rot(R, li[:, 0], li[:, 1], li[:, 2])
        c = cells(np.stack([p[0] + T[0], p[1] + T[1], p[2] + T[2]], 1), vs)
        ok = dst.in_bounds(c)
        allk.append(pack(c[ok]))
        allL.append(L[ok].astype(np.int64))
    if not allk:
        return
    k, L = np.concatenate(allk), np.concatenate(allL)
    uk, inv = np.unique(k, return_inverse=True)
    S = np.zeros(uk.size, np.int64)
    np.add.at(S, inv, L)
    dst.maps[0] = (uk, np.clip(S, dst.p["l_min"], dst.p["l_max"]).astype(np.int32))
