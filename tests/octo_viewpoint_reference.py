"""numpy f32 statement of the frontier viewpoints of a log-odds Octomap (DESIGN.md section 7, "Frontier viewpoints";
csrc/tslam_octo_view.cu).

Input: the known voxels of one submap as rows, `idx` int32[n,3] and `L` int32[n] (OctoHandle.gather()), l_occ, the
volume N, Nz, the f32 voxel scale vs, the offsets [S,3], the camera (a dict as for octo_view_gain_reference) and, for
clearance > 0, the ESDF rows (eidx, E) of the last esdf_update (esdf_rows() computes them for an unchanged map).

    centroid    m_a = f32(f64(sum_a) / f64(n) * f64(vs)) of each cluster record (octo_frontier_reference.frontiers)
    candidate   p = m + offsets[s] (f32); dx, dy = m - p; h = sqrt(dx*dx + dy*dy); u = (dx, dy) / h (all f32);
                R = [[uy, 0, ux], [-ux, 0, uy], [0, -1, 0]]
    valid       p finite, h > 0, and the cell rha(p / vs) traversable: known and FREE (known cells are in the volume),
                and with clearance > 0 an ESDF row with E >= clearance
    visible     octo_view_gain_reference.frontier_gain of (p, R) against the cluster's own frontier voxels
    kept        valid and visible >= min_visible, ordered by visible descending then s ascending; the first top_k
"""
import numpy as np

import octo_esdf_reference as oe
import octo_frontier_reference as fr
import octo_logodds_reference as ref
import octo_view_gain_reference as vg

f32 = np.float32


def esdf_rows(idx, L, l_occ, vs, D):
    """(idx, E) of an ESDF update of these rows truncated at D"""
    return np.asarray(idx), oe.esdf(idx, L, l_occ, vs, D)


def centroids(rec, vs):
    rec = np.asarray(rec, np.int64).reshape(-1, 16)
    return (rec[:, 2:5].astype(np.float64) / rec[:, 1:2].astype(np.float64) * float(f32(vs))).astype(f32)


def poses(m, offsets):
    """-> (p f32[nc,S,3], R f32[nc,S,3,3], h f32[nc,S]) of every candidate"""
    m = np.asarray(m, f32).reshape(-1, 1, 3)
    off = np.asarray(offsets, f32).reshape(1, -1, 3)
    with np.errstate(all="ignore"):
        p = (m + off).astype(f32)
        dx, dy = m[..., 0] - p[..., 0], m[..., 1] - p[..., 1]
        h = np.sqrt(dx * dx + dy * dy).astype(f32)
        ux, uy = dx / h, dy / h
    z = np.zeros_like(ux)
    R = np.stack([np.stack([uy, z, ux], -1), np.stack([-ux, z, uy], -1), np.stack([z, z - f32(1), z], -1)], -2).astype(f32)
    return p, R, h


def traversable(cls, idx, L, l_occ, p, vs, clearance=0.0, esdf=None):
    """bool per point of p [k,3]: the cell rha(p / vs) under the travel-cost rule"""
    p = np.asarray(p, f32).reshape(-1, 3)
    with np.errstate(all="ignore"):
        u = p / f32(vs)
    ok = (np.abs(u) < f32(1e9)).all(1)
    c = ref.round_half_away(np.where(ok[:, None], u, f32(0)))
    known, occ = cls.lookup(c)
    ok &= known & ~occ & cls.in_bounds(c)
    if f32(clearance) > 0:
        eidx, E = esdf
        keys = np.sort(oe.pack(np.asarray(eidx, np.int64)[np.asarray(E, f32) >= f32(clearance)]))
        k = oe.pack(c)
        pos = np.clip(np.searchsorted(keys, k), 0, max(keys.size - 1, 0))
        ok &= (keys[pos] == k) if keys.size else np.zeros(k.size, bool)
    return ok


def viewpoints(idx, L, l_occ, N, Nz, vs, offsets, cam, clearance=0.0, esdf=None, min_visible=1, top_k=1, frontier=None):
    """-> dict(count int32[nc], sample int32[nc,k], visible int32[nc,k], pos f32[nc,k,3], R f32[nc,k,3,3], valid bool[nc,S],
    score int32[nc,S] (0 where invalid)).  frontier = (fidx, fcl, rec) defaults to octo_frontier_reference.frontiers."""
    fidx, fcl, rec = fr.frontiers(idx, L, l_occ, N, Nz) if frontier is None else frontier
    fidx, fcl = np.asarray(fidx, np.int64).reshape(-1, 3), np.asarray(fcl, np.int64).reshape(-1)
    nc, S, k = rec.shape[0], np.asarray(offsets).reshape(-1, 3).shape[0], int(top_k)
    cls = vg.Classes(idx, L, l_occ, N, Nz)
    p, R, h = poses(centroids(rec, vs), offsets)
    valid = np.isfinite(p).all(-1) & (h > 0)
    valid &= traversable(cls, idx, L, l_occ, p.reshape(-1, 3), vs, clearance, esdf).reshape(nc, S)
    score = np.zeros((nc, S), np.int32)
    for c in range(nc):
        s = np.nonzero(valid[c])[0]
        if s.size:
            own = fidx[fcl == c]
            _, tot, _ = vg.frontier_gain(idx, L, l_occ, N, Nz, vs, p[c, s], R[c, s], cam, own, np.zeros(len(own), np.int64), 1)
            score[c, s] = tot
    out = dict(count=np.zeros(nc, np.int32), sample=np.full((nc, k), -1, np.int32), visible=np.zeros((nc, k), np.int32),
               pos=np.zeros((nc, k, 3), f32), R=np.zeros((nc, k, 3, 3), f32), valid=valid, score=score)
    for c in range(nc):
        s = np.nonzero(valid[c] & (score[c] >= int(min_visible)))[0]
        s = s[np.lexsort((s, -score[c, s].astype(np.int64)))][:k]
        n = s.size
        out["count"][c] = n
        out["sample"][c, :n], out["visible"][c, :n] = s, score[c, s]
        out["pos"][c, :n], out["R"][c, :n] = p[c, s], R[c, s]
    return out
