"""numpy f32 statement of the ESDF read-out: tslam_esdf_query and tslam_esdf_extract_slice (csrc/tslam_esdf.cu).

This is the definition the kernels are held to, bit for bit (the library builds with -fmad=false, and every step
below is one correctly rounded f32 operation in the same order as the kernel's).

The state is the map as of one ESDF update, given as rows: `idx` int32[m,3] observed voxels (centred indices), `tsdf`
f32[m] their TSDF (gather()), `esdf` f32[m] their ESDF (esdf_gather(), rows matched by index).  A voxel is a valid
corner when it has a row whose TSDF is not NaN: unobserved voxels and observed voxels with a NaN TSDF (INERT) are
not, and neither is a voxel outside the volume.  `blocks` (optional) restricts the state to the voxels of those
16^3 blocks (block coordinates int[k,3]), e.g. the blocks present at the update.

Query, per point p (submap-local map frame, voxel i centred at i*vs):
    u = p / vs (f32 division), per axis
    invalid unless every u is finite and both corners floor(u), floor(u) + 1 lie inside the volume
    i0 = floor(u), f = u - i0
    lerp(a, b, t) = a + t*(b - a)
    dist   = lerp along x, then y, then z of the 8 corner values
    grad.x = the four x-differences E1yz - E0yz lerped along y, then z, divided by vs
    grad.y = the four y-differences lerped along x, then z, divided by vs
    grad.z = the four z-differences lerped along x, then y, divided by vs
invalid points read NaN in dist and grad.

Slice (cvt_ESDF_to_voxels_slice, dense_esdf.py:498-509): _index = (z + map_size_z/2)/vs in f32 with
map_size_z = f32(vs*Nz); every observed voxel with _index - 0.5 < k + Nz/2 < _index + 0.5 (k centred) is exported with
its ESDF and the position (i, j, k)*vs (global maps) or R (i, j, k)*vs + T (submap maps).
"""
import numpy as np

F = np.float32


def _key(i, j, k):
    """int64 key of centred voxel indices (|index| < 2^20)."""
    return ((i.astype(np.int64) + (1 << 20)) << 42) | ((j.astype(np.int64) + (1 << 20)) << 21) | (k.astype(np.int64) + (1 << 20))


class EsdfState:
    def __init__(self, idx, tsdf, esdf, N, Nz, vs, blocks=None):
        idx = np.asarray(idx, np.int32).reshape(-1, 3)
        tsdf = np.asarray(tsdf, F)
        esdf = np.asarray(esdf, F)
        assert idx.shape[0] == tsdf.shape[0] == esdf.shape[0]
        if blocks is not None:
            bk = _key(*np.asarray(blocks, np.int64).reshape(-1, 3).T)
            keep = np.isin(_key(*(idx.astype(np.int64) >> 4).T), bk)
            idx, tsdf, esdf = idx[keep], tsdf[keep], esdf[keep]
        self.idx, self.tsdf, self.esdf = idx, tsdf, esdf
        self.N, self.Nz, self.hN, self.hNz = int(N), int(Nz), int(N) // 2, int(Nz) // 2
        self.vs, self.vs_d = F(vs), float(vs)
        keys = _key(idx[:, 0], idx[:, 1], idx[:, 2])
        o = np.argsort(keys, kind="stable")
        self.keys, self.val, self.ok = keys[o], esdf[o], ~np.isnan(tsdf[o])

    def corner(self, i, j, k):
        """(value, valid) of voxels (i, j, k)."""
        key = _key(i, j, k)
        if self.keys.shape[0] == 0:
            return np.zeros(key.shape, F), np.zeros(key.shape, bool)
        p = np.minimum(np.searchsorted(self.keys, key), self.keys.shape[0] - 1)
        hit = self.keys[p] == key
        return np.where(hit, self.val[p], F(0)), hit & self.ok[p]


def lerp(a, b, t):
    return a + t * (b - a)


def query(st, xyz):
    """-> dist f32[n], grad f32[n,3], valid bool[n]."""
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    n = xyz.shape[0]
    dist = np.full(n, np.nan, F)
    grad = np.full((n, 3), np.nan, F)
    with np.errstate(all="ignore"):
        u = xyz / st.vs
        lo = np.array([-st.hN, -st.hN, -st.hNz], F)
        hi = np.array([st.N - st.hN - 1, st.N - st.hN - 1, st.Nz - st.hNz - 1], F)
        ok = np.isfinite(xyz).all(1) & ((u >= lo) & (u < hi)).all(1)   # tested before any float -> int conversion
    q = np.nonzero(ok)[0]
    uq = u[q]
    i0 = np.floor(uq).astype(np.int64)
    f = (uq - i0.astype(F)).astype(F)
    E = {}
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                v, good = st.corner(i0[:, 0] + dx, i0[:, 1] + dy, i0[:, 2] + dz)
                E[dx, dy, dz] = v
                ok[q] &= good
    fx, fy, fz = f[:, 0], f[:, 1], f[:, 2]
    c = {(y, z): lerp(E[0, y, z], E[1, y, z], fx) for y in (0, 1) for z in (0, 1)}
    d = lerp(lerp(c[0, 0], c[1, 0], fy), lerp(c[0, 1], c[1, 1], fy), fz)
    ax = {(y, z): E[1, y, z] - E[0, y, z] for y in (0, 1) for z in (0, 1)}
    gx = lerp(lerp(ax[0, 0], ax[1, 0], fy), lerp(ax[0, 1], ax[1, 1], fy), fz) / st.vs
    ay = {(x, z): E[x, 1, z] - E[x, 0, z] for x in (0, 1) for z in (0, 1)}
    gy = lerp(lerp(ay[0, 0], ay[1, 0], fx), lerp(ay[0, 1], ay[1, 1], fx), fz) / st.vs
    az = {(x, y): E[x, y, 1] - E[x, y, 0] for x in (0, 1) for y in (0, 1)}
    gz = lerp(lerp(az[0, 0], az[1, 0], fx), lerp(az[0, 1], az[1, 1], fx), fy) / st.vs
    good = ok[q]
    qq = q[good]
    dist[qq] = d[good]
    grad[qq] = np.stack([gx, gy, gz], 1)[good]
    return dist, grad, ok


def slice_rows(st, z, R=None, T=None):
    """-> xyz f32[m,3], esdf f32[m] of the exported voxels (row order unspecified).  R, T: pose of a submap map (None:
    global map)."""
    msz = F(st.vs_d * st.Nz)   # map_size_z = voxel_scale * Nz, computed in f64 and rounded once
    index = (F(z) + msz / F(2)) / st.vs
    ku = (st.idx[:, 2] + st.hNz).astype(F)
    sel = (index - F(0.5) < ku) & (ku < index + F(0.5))
    ijk = st.idx[sel].astype(F)
    p = ijk * st.vs
    if R is not None:
        R, T = np.asarray(R, F).reshape(3, 3), np.asarray(T, F).reshape(3)
        p = np.stack([((R[r, 0] * p[:, 0] + R[r, 1] * p[:, 1]) + R[r, 2] * p[:, 2]) + T[r] for r in range(3)], 1)
    return p.astype(F), st.esdf[sel]
