"""numpy statement of tslam_octo_fuse_update (DESIGN.md section 7, "Incremental Octomap fusion"): what the global map
holds after an update, from the gathered rows of each source submap and dst's pose table.

The update promises tslam_octo_fuse's result for the included submaps, so this is also a statement of k_octo_fuse:
every source voxel the rule carries over (hit counter: c > min_occupy_thres in f32; log-odds: every known voxel) lands
in the cell round_half_away((R (i vs) + T) / vs) of dst (f32, kernel operation order; octo_logodds_reference.fuse places
log-odds voxels the same way), out-of-volume cells are dropped, and per cell
    hit counter: the u32 sum (mod 2^32) of c;          log-odds: clamp(sum L, l_min, l_max), clamped once;
    colour word: the max of the nonzero source colour words (seq << 24 | rgb), 0 when there is none.
"""
import numpy as np

import octo_logodds_reference as lr
from octo_logodds_reference import cells, f32, pack, unpack


def place(idx, R, T, vs):
    """oc_fuse_cell: the dst cells of source cells idx [n,3] of a submap at pose (R, T)."""
    Rm, Tm = lr._mat(R, T)
    li = np.asarray(idx, np.int64).reshape(-1, 3).astype(f32) * f32(vs)
    p = lr._rot(Rm, li[:, 0], li[:, 1], li[:, 2])
    return cells(np.stack([p[0] + Tm[0], p[1] + Tm[1], p[2] + Tm[2]], 1).astype(f32), vs)


def in_bounds(c, N, Nz):
    hN, hNz = N // 2, Nz // 2
    c = np.asarray(c).reshape(-1, 3)
    return ((c[:, 0] >= -hN) & (c[:, 0] < N - hN) & (c[:, 1] >= -hN) & (c[:, 1] < N - hN) & (c[:, 2] >= -hNz)
            & (c[:, 2] < Nz - hNz))


def fuse(rows, poses, vs, N, Nz, model="hits", thres=3, l_min=-2048, l_max=3595, include=None):
    """rows: {s: (idx int [n,3], val [n], cw uint64 [n] or None)} - val is the hit count (hit counter) or L (log-odds)
    of the voxels the source's gather returns; poses: {s: (R, T)}, dst's pose table; include: None (all) or a
    container of included submap ids.  -> (idx int32 [m,3] in key order, val [m] (uint32 counts / int32 L), cw uint64
    [m]) of the cells a gather of dst returns (hit counter: count != 0; log-odds: at least one contribution)."""
    keys, vals, cws = [], [], []
    for s, (idx, val, cw) in rows.items():
        if include is not None and s not in include:
            continue
        idx = np.asarray(idx).reshape(-1, 3)
        val = np.asarray(val)
        if model == "hits":
            keep = val.astype(np.uint32).astype(f32) > f32(thres)
        else:
            keep = np.ones(val.shape[0], bool)
        c = place(idx[keep], *poses[s], vs)
        ok = in_bounds(c, N, Nz)
        keys.append(pack(c[ok]))
        vals.append(val[keep][ok].astype(np.int64))
        cws.append((np.zeros(int(ok.sum()), np.uint64) if cw is None else np.asarray(cw, np.uint64)[keep][ok]))
    if not keys:
        return np.zeros((0, 3), np.int32), np.zeros(0, np.uint32 if model == "hits" else np.int32), np.zeros(0, np.uint64)
    k, v, w = np.concatenate(keys), np.concatenate(vals), np.concatenate(cws)
    uk, inv = np.unique(k, return_inverse=True)
    S = np.zeros(uk.size, np.int64)
    np.add.at(S, inv, v)
    W = np.zeros(uk.size, np.uint64)
    np.maximum.at(W, inv, w)
    if model == "hits":
        out = (S & 0xFFFFFFFF).astype(np.uint32)
        keep = out != 0
        return unpack(uk[keep]).astype(np.int32), out[keep], W[keep]
    return unpack(uk).astype(np.int32), np.clip(S, l_min, l_max).astype(np.int32), W


def sum_word(count, sum_L):
    """The log-odds sum word of a cell: count * 2^32 + sum L (int64)."""
    return np.int64(count) * np.int64(1 << 32) + np.int64(sum_L)


def readout(co, l_min, l_max):
    """k_of_commit: the cnt word of a log-odds cell from its sum word (0: unknown)."""
    co = int(co)
    cnt = (co + (1 << 31)) >> 32
    sl = co - (cnt << 32)
    if cnt <= 0:
        return 0
    return ((int(np.clip(sl, l_min, l_max)) << 1) | 1) & 0xFFFFFFFF


def sorted_rows(idx, *cols):
    """Rows in key order (dst's pool order is free): (idx, *cols) sorted by packed cell key."""
    o = np.argsort(pack(np.asarray(idx).reshape(-1, 3)), kind="stable")
    return (np.asarray(idx)[o],) + tuple(np.asarray(c)[o] for c in cols)
