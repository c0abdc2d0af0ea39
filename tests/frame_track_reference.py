"""numpy statement of frame tracking (tslam_tsdf_track_depth / tslam_tsdf_track_points, csrc/tslam_register.cu;
DESIGN.md section 7, "Frame tracking").

The two selection rules are restated here in the kernels' f32 operation order (every step one correctly rounded f32
operation; the library builds with -fmad=false).  What follows selection - residual, sums and the Levenberg-Marquardt
loop - is registration's with d = 0, so it is tests/submap_register_reference.py's register(), called, not restated.

  depth   sampled pixels (i, j) = (step ii, step jj), ii < w // step, jj < h // step, row-major; kept when d != 0 and
          not (f32(d) > dmax_mm or f32(d) < dmin_mm), dmin_mm / dmax_mm = f32(min_ray * 1000) / f32(max_ray * 1000);
          point dep = f32(d) / 1000, x = ((f32(i) - cx) dep) / fx, y = ((f32(j) - cy) dep) / fy
  points  input order; kept when x, y, z are finite and f32(min_ray) <= sqrt((x x + y y) + z z) < f32(max_ray)
"""
import numpy as np

import submap_register_reference as reg

F = np.float32


def select_depth(depth, K, step, min_ray, max_ray):
    """-> f32[n,3] sensor-frame points of one uint16 frame [h,w], in row-major sampled-pixel order."""
    depth = np.asarray(depth, np.uint16)
    h, w = depth.shape
    hh, ww = h // step, w // step
    fx, cx, fy, cy = F(K[0]), F(K[2]), F(K[4]), F(K[5])
    dmin, dmax = F(min_ray * 1000.0), F(max_ray * 1000.0)
    d = depth[:hh * step:step, :ww * step:step]
    df = d.astype(F)
    keep = (d != 0) & ~((df > dmax) | (df < dmin))
    jj, ii = np.nonzero(keep)                                   # row-major
    dep = df[jj, ii] / F(1000.0)
    x = (((ii * step).astype(F) - cx) * dep) / fx
    y = (((jj * step).astype(F) - cy) * dep) / fy
    return np.stack([x, y, dep], 1).astype(F)


def select_points(xyz, min_ray, max_ray):
    """-> f32[n,3] the kept points of a cloud f32[m,3], in input order."""
    p = np.asarray(xyz, F).reshape(-1, 3)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    with np.errstate(over="ignore", invalid="ignore"):
        r = np.sqrt((x * x + y * y) + z * z)
        keep = np.isfinite(p).all(1) & (r >= F(min_ray)) & (r < F(max_ray))
    return p[keep]


def reading(gathered, N, Nz, vs):
    """The map's submap as gather() returns it (idx, tsdf, w[, occ])."""
    idx, t, w = gathered[:3]
    return reg.Reading(idx, t, w, N, Nz, vs)


def track(rd, p, R0, T0, vs, huber=None, max_iters=20, min_points=100):
    """The solver of one frame: registration's, with d = 0 -> dict(R, T, S, cost_init, iterations, converged, status)."""
    return reg.register(rd, p, np.zeros(len(p), F), R0, T0, vs, huber=huber, max_iters=max_iters, min_points=min_points)


def normal_equations(rd, p, R, t, delta):
    return reg.normal_equations(rd, p, np.zeros(len(p), F), R, t, delta)


def abs_sums(rd, p, R, t, delta):
    return reg.abs_sums(rd, p, np.zeros(len(p), F), R, t, delta)
