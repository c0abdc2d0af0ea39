"""numpy f32 statement of the viewpoint gain of a log-odds Octomap (DESIGN.md section 7, "Viewpoint gain of the log-odds
Octomap"; csrc/tslam_octo_view.cu).

Input: the known voxels of one submap as rows, `idx` int32[n,3] and `L` int32[n] (OctoHandle.gather()), l_occ, the
volume N, Nz, the f32 voxel scale vs, the views (pos [m,3], R [m,3,3]) and the camera (a dict fx, fy, cx, cy, width,
height, step, max_range).  Classes: OCC = known and L > l_occ, FREE = known and L <= l_occ, UNKNOWN = not known.

    valid          the view's 12 numbers are finite and its cell rha(p / vs) is in the volume and FREE
    unknown gain   the rays of an all-far depth frame (octo_logodds_reference.depth_endpoints at dep = max_range) walk
                   octo_logodds_reference.walk's path, end cell included; a ray sees its in-volume cells before its
                   first in-volume OCC cell; the gain is the number of distinct UNKNOWN cells seen by the view's rays
    frontier gain  frontier voxel c counts when q = R^T (f32(c) vs - p) has 0 < q_z <= max_range, its projection lies in
                   [0, width-1] x [0, height-1], and every cell of walk(p -> f32(c) vs, clipped) before c is FREE
"""
import numpy as np

import octo_frontier_reference as fr
import octo_logodds_reference as ref

f32 = np.float32


class Classes:
    """Class lookup of cells from the gathered (idx, L) rows."""

    def __init__(self, idx, L, l_occ, N, Nz):
        idx = np.asarray(idx, np.int64).reshape(-1, 3)
        self.keys = ref.pack(idx)
        o = np.argsort(self.keys)
        self.keys = self.keys[o]
        self.occ = (np.asarray(L, np.int64).reshape(-1) > int(l_occ))[o]
        self.N, self.Nz = N, Nz

    def in_bounds(self, c):
        hN, hNz = self.N // 2, self.Nz // 2
        return ((c[:, 0] >= -hN) & (c[:, 0] < self.N - hN) & (c[:, 1] >= -hN) & (c[:, 1] < self.N - hN) & (c[:, 2] >= -hNz)
                & (c[:, 2] < self.Nz - hNz))

    def lookup(self, c):
        """(known, occ) per cell"""
        k = ref.pack(c)
        if self.keys.size == 0:
            z = np.zeros(k.size, bool)
            return z, z
        pos = np.clip(np.searchsorted(self.keys, k), 0, self.keys.size - 1)
        known = self.keys[pos] == k
        return known, known & self.occ[pos]


def valid_views(cls, pos, R, vs):
    pos = np.asarray(pos, f32).reshape(-1, 3)
    R = np.asarray(R, f32).reshape(-1, 9)
    ok = np.isfinite(pos).all(1) & np.isfinite(R).all(1)
    with np.errstate(all="ignore"):
        u = pos / f32(vs)
    ok &= (np.abs(u) < f32(1e9)).all(1)
    c = ref.round_half_away(np.where(ok[:, None], u, f32(0)))
    known, occ = cls.lookup(c)
    return ok & cls.in_bounds(c) & known & ~occ


def _path_positions(rays, n):
    """position of every walk() output row along its own ray's path (walk emits the rays step by step)"""
    o = np.argsort(rays, kind="stable")
    counts = np.bincount(rays, minlength=n)
    start = np.concatenate([[0], np.cumsum(counts)[:-1]])
    pos = np.empty(rays.size, np.int64)
    pos[o] = np.arange(rays.size) - np.repeat(start, counts)
    return pos


def unknown_gain(idx, L, l_occ, N, Nz, vs, pos, R, cam):
    """-> (valid bool[m], gain int64[m])"""
    cls = Classes(idx, L, l_occ, N, Nz)
    pos = np.asarray(pos, f32).reshape(-1, 3)
    R = np.asarray(R, f32).reshape(-1, 3, 3)
    valid = valid_views(cls, pos, R, vs)
    gain = np.zeros(pos.shape[0], np.int64)
    K = [cam["fx"], 0.0, cam["cx"], 0.0, cam["fy"], cam["cy"], 0.0, 0.0, 1.0]
    far = np.full((int(cam["height"]), int(cam["width"])), 65535, np.uint16)  # every pixel beyond max_range (< 65.5 m)
    assert f32(cam["max_range"]) * 1000 < 65535
    for v in np.nonzero(valid)[0]:
        ends, clipped = ref.depth_endpoints(far, R[v], pos[v], K, 0.0, float(f32(cam["max_range"])), int(cam["step"]))
        assert clipped.all()
        rays, cells = ref.walk(pos[v], ends, clipped, vs)
        at = _path_positions(rays, ends.shape[0])
        inb = cls.in_bounds(cells)
        known, occ = cls.lookup(cells)
        occ &= inb
        first = np.full(ends.shape[0], np.iinfo(np.int64).max)
        np.minimum.at(first, rays[occ], at[occ])
        seen = inb & (at < first[rays])
        gain[v] = np.unique(ref.pack(cells[seen & ~known])).size
    return valid, gain


def frontier_gain(idx, L, l_occ, N, Nz, vs, pos, R, cam, fidx=None, fcl=None, n_clusters=None):
    """-> (valid bool[m], total int32[m], per_cluster int32[m, n_clusters]).  The frontier set (fidx, fcl, n_clusters)
    defaults to octo_frontier_reference.frontiers of the same rows; pass an older one to read a stale frontier set."""
    if fidx is None:
        fidx, fcl, rec = fr.frontiers(idx, L, l_occ, N, Nz)
        n_clusters = rec.shape[0]
    cls = Classes(idx, L, l_occ, N, Nz)
    pos = np.asarray(pos, f32).reshape(-1, 3)
    R = np.asarray(R, f32).reshape(-1, 3, 3)
    valid = valid_views(cls, pos, R, vs)
    per = np.zeros((pos.shape[0], int(n_clusters)), np.int32)
    fidx = np.asarray(fidx, np.int64).reshape(-1, 3)
    fcl = np.asarray(fcl, np.int64).reshape(-1)
    x = fidx.astype(f32) * f32(vs)
    fx, fy, cx, cy, mr = (f32(cam[k]) for k in ("fx", "fy", "cx", "cy", "max_range"))
    wmax, hmax = f32(int(cam["width"]) - 1), f32(int(cam["height"]) - 1)
    for v in np.nonzero(valid)[0]:
        d = x - pos[v]
        Rv = R[v]
        q = [(Rv[0, a] * d[:, 0] + Rv[1, a] * d[:, 1]) + Rv[2, a] * d[:, 2] for a in range(3)]
        with np.errstate(all="ignore"):
            u = ((q[0] * fx) / q[2]) + cx
            w = ((q[1] * fy) / q[2]) + cy
        inf = (q[2] > 0) & (q[2] <= mr) & (u >= 0) & (u <= wmax) & (w >= 0) & (w <= hmax)
        sel = np.nonzero(inf)[0]
        if sel.size == 0:
            continue
        rays, cells = ref.walk(pos[v], x[sel], np.ones(sel.size, bool), vs)
        at = _path_positions(rays, sel.size)
        last = np.bincount(rays, minlength=sel.size) - 1
        known, occ = cls.lookup(cells)
        bad = (at < last[rays]) & ~(known & ~occ & cls.in_bounds(cells))
        blocked = np.zeros(sel.size, bool)
        blocked[rays[bad]] = True
        np.add.at(per[v], fcl[sel[~blocked]], 1)
    return valid, per.sum(1).astype(np.int32), per
