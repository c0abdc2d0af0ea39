"""numpy statement of tslam_tsdf_render (csrc/tslam_render.cu; DESIGN.md section 7, "Rendering").

Every f32 step below is one correctly rounded operation in the kernel's order (the library builds with -fmad=false), and
the interpolation, its validity and its gradient are tests/esdf_query_reference.py's query() on the state that
tests/submap_register_reference.py's Reading builds: the zero level registration and frame tracking align to.  The
kernel's shortcuts (memoised block lookups, stopping at the first hit or when the ray leaves the volume) change no
result, so this reference evaluates all K samples of every ray and takes the first crossing.

  ray      r = ((f32(i) - cx) / fx, (f32(j) - cy) / fy, 1); dir = ((R0 rx + R1 ry) + R2 1) + 0 per row (pose_apply, T = 0)
  samples  K = floor((z_max - z_min) / step) + 1 in f64 of the f32 parameters; z_k = z_min + f32(k) step; x_k = T + z_k dir
  hit      first k with samples k, k+1 valid, D_k > 0 >= D_{k+1}; a = D_k - D_{k+1}, f = D_k / a, z* = z_k + step f,
           x* = T + z* dir
  status   0 no hit, 1 hit with x*'s corners valid and |g| = sqrt((gx gx + gy gy) + gz gz) > 0, 2 any other hit
  normal   g / |g|; colour: each channel interpolated at x* like the TSDF (one EsdfState per channel)
"""
import numpy as np

import esdf_query_reference as eqr
import submap_register_reference as reg

F = np.float32


class Scene:
    """One submap as gather() returns it: idx int32[m,3], tsdf, w f32[m], and optionally col f32[m,3]."""

    def __init__(self, idx, tsdf, w, N, Nz, vs, col=None):
        self.rd = reg.Reading(idx, tsdf, w, N, Nz, vs)
        self.vs = F(vs)
        self.col = None
        if col is not None:
            idx, w, col = np.asarray(idx, np.int32).reshape(-1, 3), np.asarray(w, F), np.asarray(col, F).reshape(-1, 3)
            keep = w > 0
            z = np.zeros(int(keep.sum()), F)
            self.col = [eqr.EsdfState(idx[keep], z, col[keep, c], N, Nz, vs) for c in range(3)]


def from_gather(gathered, N, Nz, vs):
    """Scene of gather()'s (idx, tsdf, w, occ[, col])."""
    return Scene(*gathered[:3], N, Nz, vs, col=gathered[4] if len(gathered) > 4 else None)


def n_samples(z_min, z_max, step):
    return int(np.floor((float(F(z_max)) - float(F(z_min))) / float(F(step)))) + 1


def directions(R, K9, i, j):
    """f32 [m,3] local-frame directions of pixels (i, j) for camera rotation R (f64, rounded to f32)."""
    fx, fy, cx, cy = F(K9[0]), F(K9[4]), F(K9[2]), F(K9[5])
    R32 = np.asarray(R, np.float64).reshape(3, 3).astype(F)
    rx = (np.asarray(i).astype(F) - cx) / fx
    ry = (np.asarray(j).astype(F) - cy) / fy
    return np.stack([((R32[r, 0] * rx + R32[r, 1] * ry) + R32[r, 2] * F(1)) + F(0) for r in range(3)], 1).astype(F)


def render(sc, R, T, h, w, K9, z_min, z_max, step, pixels=None, color=False):
    """-> dict(depth f32[P], status u8[P], normal f32[P,3], color f32[P,3] (when asked)) for the pixels `pixels` (flat
    row-major indices j w + i; default every pixel of the h x w image)."""
    pixels = np.arange(h * w) if pixels is None else np.asarray(pixels, np.int64)
    P = pixels.shape[0]
    T32 = np.asarray(T, np.float64).reshape(3).astype(F)
    z_min, step = F(z_min), F(step)
    K = n_samples(z_min, z_max, step)
    z = (z_min + np.arange(K).astype(F) * step).astype(F)
    dirs = directions(R, K9, pixels % w, pixels // w)
    depth = np.zeros(P, F)
    status = np.zeros(P, np.uint8)
    normal = np.full((P, 3), np.nan, F)
    col = np.full((P, 3), np.nan, F)
    chunk = max(1, 2_000_000 // K)
    for a in range(0, P, chunk):
        d = dirs[a:a + chunk]
        m = d.shape[0]
        x = (T32[None, None, :] + z[None, :, None] * d[:, None, :]).astype(F)
        D, _, ok = eqr.query(sc.rd.st, x.reshape(-1, 3))
        D, ok = D.reshape(m, K), ok.reshape(m, K)
        with np.errstate(invalid="ignore"):
            cross = ok[:, :-1] & ok[:, 1:] & (D[:, :-1] > 0) & (D[:, 1:] <= 0)
        hit = cross.any(1)
        r = np.nonzero(hit)[0]
        k = cross[r].argmax(1)
        Dk, Dk1 = D[r, k], D[r, k + 1]
        f = (Dk / (Dk - Dk1)).astype(F)
        zs = (z[k] + step * f).astype(F)
        xs = (T32[None, :] + zs[:, None] * d[r]).astype(F)
        _, g, good = eqr.query(sc.rd.st, xs)
        with np.errstate(invalid="ignore"):
            gn = np.sqrt((g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2]).astype(F)
            one = good & (gn > 0)
        rows = a + r
        depth[rows] = zs
        status[rows] = np.where(one, 1, 2)
        with np.errstate(invalid="ignore", divide="ignore"):
            normal[rows[one]] = (g[one] / gn[one, None]).astype(F)
        if color:
            for c in range(3):
                col[rows[one], c] = eqr.query(sc.col[c], xs[one])[0]
    out = dict(depth=depth, status=status, normal=normal)
    if color:
        out["color"] = col
    return out
