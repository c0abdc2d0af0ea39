"""numpy statement of tslam_mc_generate2 (csrc/tslam_mc.cu; the reference's marching_cube_mesher.py, whose line numbers
the kernel comments cite and which are cited below).

The input is the map as gather(submap, color=True) returns it, for every submap that holds blocks: rows (idx, tsdf, w,
occ[, colour]).  Every f32 step below is one correctly rounded operation in the kernel's order (the library builds with
-fmad=false; its divisions and sqrtf are IEEE), so the kernel must match this statement bit for bit.

  reads     a voxel reads (T, observed) from its submap's rows; any voxel without a row (absent block, unobserved voxel
            of an allocated block, outside the volume) reads T = 0, observed = 0.  No read crosses submaps.  (The planes
            of unobserved voxels hold 0: reset and fusion zero them.  The normals next to holes check that.)
  cell      (s, i, j, k) is meshed when corner 0 is observed with T < thres (:184; strict, NaN fails) and every corner
            (i, j, k) + step * V_c (:196-206) is observed (:137-140)
  cube      bit c set when T_c < 0.0f (:143-144): -0.0 and NaN are not negative
  table     triangles of the cube index from include/tslam_mc_cases.h (TSLAM_MC_CASE_WORDS, :244-499), edges :208-221
  vertex    |0 - v1| < 1e-6f: p1; else |0 - v2| < 1e-6f: p2; else mu = (0 - v1) / (v2 - v1), p1 + mu (p2 - p1) per
            coordinate (:44-60); then times vs (ijk_to_xyz :40-42)
  normal    non-finite vertex: NaN (:86 is undefined there); else q = roundf(vertex) (half away from zero, :86),
            n = (T(q + x) - T(q - x), ...) read whatever the observed flag says (:88-90), n / sqrt((nx nx + ny ny) + nz nz)
            (:92; NaN when the gradient vanishes)
  colour    vertexInterp_color (:62-82): mu as the vertex but 0 in both snap branches; c1.x == 0: c2; else c2.x != 0:
            c1 + mu (c2 - c1); else c1 (only channel 0 is looked at)
"""
import os
import re

import numpy as np

F = np.float32
EPS = F(1e-6)  # :6
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "tslam_mc_cases.h")
CORNERS = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 1], [0, 1, 1]])  # :196-206
EDGES = np.array([[0, 1], [1, 2], [2, 3], [3, 0], [4, 5], [5, 6], [6, 7], [7, 4], [0, 4], [1, 5], [2, 6], [3, 7]])  # :208-221
QNAN = np.uint32(0x7FC00000)


def case_table(path=HEADER):
    """(tri int8 [256, 15]: edge of corner q of the case's triangles, -1 past the end; ntri int [256]) from the packed
    words of the generated header: nibble q of word c is the edge of corner q, 0xF ends the list."""
    with open(path) as f:
        txt = f.read()
    words = [int(w, 16) for w in re.findall(r"0x([0-9a-fA-F]{16})ull", txt[txt.index("#define TSLAM_MC_CASE_WORDS"):])]
    assert len(words) == 256
    tri = np.full((256, 15), -1, np.int8)
    ntri = np.zeros(256, np.int64)
    for c, w in enumerate(words):
        nib = [(w >> (4 * q)) & 0xF for q in range(16)]
        n = nib.index(0xF)
        assert n % 3 == 0 and all(e == 0xF for e in nib[n:]) and all(e < 12 for e in nib[:n])
        tri[c, :n] = nib[:n]
        ntri[c] = n // 3
    return tri, ntri


TRI, NTRI = case_table()

_OFF = 1 << 15


def _key(s, ijk):
    ijk = np.asarray(ijk, np.int64)
    return (((np.asarray(s, np.int64) << 16 | (ijk[..., 0] + _OFF)) << 16 | (ijk[..., 1] + _OFF)) << 16) | (ijk[..., 2] + _OFF)


class Voxels:
    """The observed voxels of every submap: submaps = {s: gather(s[, color=True]) tuple (idx, tsdf, w, occ[, col])}."""

    def __init__(self, submaps):
        keys, t, col = [], [], []
        self.color = all(len(g) > 4 for g in submaps.values()) and len(submaps) > 0
        for s, g in submaps.items():
            idx = np.asarray(g[0], np.int32).reshape(-1, 3)
            keys.append(_key(np.full(idx.shape[0], s), idx))
            t.append(np.asarray(g[1], F).reshape(-1))
            if self.color:
                col.append(np.asarray(g[4], F).reshape(-1, 3))
        keys = np.concatenate(keys) if keys else np.zeros(0, np.int64)
        o = np.argsort(keys, kind="stable")
        self.keys = keys[o]
        assert np.all(np.diff(self.keys) > 0), "a voxel appears twice"
        self.t = np.concatenate(t)[o] if t else np.zeros(0, F)
        self.col = np.concatenate(col)[o] if self.color else None
        self.s = (self.keys >> 48).astype(np.int64)
        self.ijk = np.stack([((self.keys >> sh) & 0xFFFF) - _OFF for sh in (32, 16, 0)], 1).astype(np.int64)

    def row(self, s, ijk):
        """Row of each voxel (s, ijk), -1 where it has none."""
        k = _key(s, ijk)
        if self.keys.shape[0] == 0:
            return np.full(k.shape, -1, np.int64)
        p = np.minimum(np.searchsorted(self.keys, k), self.keys.shape[0] - 1)
        return np.where(self.keys[p] == k, p, -1)

    def read(self, s, ijk):
        """(T f32, observed bool, row) of voxels (s, ijk): T = 0 and observed = False without a row."""
        r = self.row(s, ijk)
        ok = r >= 0
        return np.where(ok, self.t[np.maximum(r, 0)], F(0)).astype(F), ok, r


def _roundf(x):
    """roundf: half away from zero (np.round rounds half to even).  Exact: x is f32, the sum is formed in f64."""
    x = np.asarray(x, np.float64)
    return (np.sign(x) * np.floor(np.abs(x) + 0.5)).astype(np.int64)


def mesh(submaps, N, Nz, vs, step, thres, color=False, chunk=1 << 20):
    """The full triangle list of tslam_mc_generate2(step, thres) on the map `submaps` ({s: gather tuple}) of an N x N x Nz
    volume.  -> dict, one row per triangle in (s, i, j, k, t) order:
      tag int64 [n, 5] (s, i, j, k, t); verts, normals (, colors) f32 [n, 3, 3]
    and per triangle vertex, for tests that must show they reached a branch:
      edge int8 [n, 3]; snap int8 [n, 3] (0 interpolated, 1 p1, 2 p2); at int64 [n, 3, 3] (the rounded normal point,
      unscaled; 0 for a non-finite vertex); hole bool [n, 3] (a normal read has no row); half bool [n, 3] (a negative
      unscaled coordinate ends in exactly .5, where roundf and rounding half to even differ); cbranch int8 [n, 3]
      (colour: 0 c2, 1 interpolated, 2 c1)
    and counts: cand (cells passing :184), skipped (of those, with an unobserved corner), edge_skipped (of those, with a
    corner outside the volume)."""
    vx = Voxels(submaps)
    step, vs, thres = int(step), F(vs), F(thres)
    hN, hNz = N // 2, Nz // 2
    with np.errstate(invalid="ignore"):
        cand = np.nonzero(vx.t < thres)[0]  # :184 (every row is observed)
    out = {k: [] for k in ("tag", "verts", "normals", "colors", "edge", "snap", "at", "hole", "half", "cbranch")}
    n_skip = n_edge = 0
    for a in range(0, cand.shape[0], chunk):
        c = cand[a:a + chunk]
        s, ijk = vx.s[c], vx.ijk[c]
        cp = ijk[:, None, :] + step * CORNERS[None]                     # [m, 8, 3] corners (:133-136)
        val, obs, crow = vx.read(s[:, None], cp)
        good = obs.all(1)                                                # :137-140
        inside = ((cp[..., :2] >= -hN) & (cp[..., :2] < N - hN)).all(2) & (cp[..., 2] >= -hNz) & (cp[..., 2] < Nz - hNz)
        n_skip += int((~good).sum())
        n_edge += int((~inside.all(1)).sum())
        with np.errstate(invalid="ignore"):
            cube = ((val < F(0)).astype(np.int64) << np.arange(8)[None]).sum(1)  # :141-144
        nt = np.where(good, NTRI[cube], 0)
        cell = np.repeat(np.arange(c.shape[0]), nt)
        if cell.shape[0] == 0:
            continue
        t = np.arange(cell.shape[0]) - np.repeat(np.cumsum(nt) - nt, nt)
        cb = cube[cell]
        e = np.stack([TRI[cb, 3 * t + q] for q in range(3)], 1).astype(np.int64)  # [n, 3] (:110-125)
        ea, eb = EDGES[e, 0], EDGES[e, 1]
        cellv = cell[:, None]
        v1, v2 = val[cellv, ea], val[cellv, eb]
        p1 = cp[cellv, ea].astype(F)                                     # [n, 3, 3]
        p2 = cp[cellv, eb].astype(F)
        snap1 = np.abs(F(0) - v1) < EPS                                  # :49-50
        snap2 = ~snap1 & (np.abs(F(0) - v2) < EPS)                       # :51-54
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            mu = ((F(0) - v1) / (v2 - v1)).astype(F)                     # :56
            pint = (p1 + mu[..., None] * (p2 - p1)).astype(F)            # :57-59
        p = np.where(snap1[..., None], p1, np.where(snap2[..., None], p2, pint)).astype(F)
        with np.errstate(over="ignore", invalid="ignore"):
            verts = (p * vs).astype(F)                                   # :40-42
        # generate_normal :84-93
        fin = np.isfinite(p).all(2)
        q = np.where(fin[..., None], _roundf(np.where(np.isfinite(p), p, F(0))), 0)
        sv = np.broadcast_to(s[cell][:, None], q.shape[:2])
        grads, hole = [], np.zeros(fin.shape, bool)
        for ax in range(3):
            d = np.zeros(3, np.int64)
            d[ax] = 1
            tp, op, _ = vx.read(sv, q + d)
            tm, om, _ = vx.read(sv, q - d)
            hole |= ~op | ~om
            with np.errstate(invalid="ignore", over="ignore"):
                grads.append((tp - tm).astype(F))
        nx, ny, nz = grads
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            nn = np.sqrt(((nx * nx + ny * ny).astype(F) + nz * nz).astype(F)).astype(F)
            nrm = np.stack([nx / nn, ny / nn, nz / nn], 2).astype(F)
        nrm[~fin] = np.nan
        out["tag"].append(np.stack([s[cell], ijk[cell, 0], ijk[cell, 1], ijk[cell, 2], t], 1))
        out["verts"].append(verts)
        out["normals"].append(nrm)
        out["edge"].append(e.astype(np.int8))
        out["snap"].append(np.where(snap1, 1, np.where(snap2, 2, 0)).astype(np.int8))
        out["at"].append(q)
        with np.errstate(invalid="ignore"):
            out["half"].append(np.any((p < 0) & (p - np.floor(p) == F(0.5)), 2))
        out["hole"].append(hole & fin)
        if color:  # vertexInterp_color :62-82
            c1 = vx.col[crow[cellv, ea]]
            c2 = vx.col[crow[cellv, eb]]
            muc = np.where(snap1 | snap2, F(0), mu).astype(F)
            with np.errstate(invalid="ignore", over="ignore"):
                ci = (c1 + muc[..., None] * (c2 - c1)).astype(F)
            z1, z2 = c1[..., 0] == F(0), c2[..., 0] == F(0)
            out["colors"].append(np.where(z1[..., None], c2, np.where(~z2[..., None], ci, c1)).astype(F))
            out["cbranch"].append(np.where(z1, 0, np.where(~z2, 1, 2)).astype(np.int8))
    res = dict(cand=int(cand.shape[0]), skipped=n_skip, edge_skipped=n_edge)
    empty = dict(tag=(0, 5), verts=(0, 3, 3), normals=(0, 3, 3), colors=(0, 3, 3), edge=(0, 3), snap=(0, 3), at=(0, 3, 3),
                 hole=(0, 3), half=(0, 3), cbranch=(0, 3))
    dt = dict(tag=np.int64, verts=F, normals=F, colors=F, edge=np.int8, snap=np.int8, at=np.int64, hole=bool, half=bool, cbranch=np.int8)
    for k, v in out.items():
        if k in ("colors", "cbranch") and not color:
            continue
        res[k] = np.concatenate(v) if v else np.zeros(empty[k], dt[k])
    return res


def block_count(tag, step):
    """Number of distinct 16^3 blocks the 8 corners of each triangle's cell lie in."""
    b = (tag[:, None, 1:4] + step * CORNERS[None]) >> 4
    k = np.sort(((b[..., 0] + 512) << 20) | ((b[..., 1] + 512) << 10) | (b[..., 2] + 512), 1)
    return (np.diff(k, axis=1) != 0).sum(1) + 1


def rows(verts, normals, colors=None):
    """uint32 [n, 18 or 27] rows (vertex, normal[, colour] words of each triangle) with every NaN made the canonical
    quiet NaN, so that NaN positions compare exactly whatever their payload."""
    parts = [np.asarray(a, F).reshape(-1, 9) for a in ((verts, normals) if colors is None else (verts, normals, colors))]
    r = np.ascontiguousarray(np.concatenate(parts, 1))
    u = r.view(np.uint32).copy()
    u[np.isnan(r)] = QNAN
    return u


def sorted_rows(verts, normals, colors=None):
    u = rows(verts, normals, colors)
    return u[np.lexsort(u.T[::-1])] if u.shape[0] else u


def rows_in(u, ref_u):
    """Whether each row of u is a row of ref_u."""
    void = np.dtype((np.void, u.dtype.itemsize * u.shape[1]))
    return np.isin(np.ascontiguousarray(u).view(void).ravel(), np.ascontiguousarray(ref_u).view(void).ravel())
