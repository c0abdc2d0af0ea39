#!/usr/bin/env python3
"""How much a CTA-level merge saves the bucket kernel on the bench's frames (CPU only, no GPU).

k_bucket_depth runs one thread per sampled pixel; a warp covers an 8x4 tile of sampled pixels, a CTA a 32x8 tile.  Every
(warp tile, bucket) pair costs one global index probe and either an opener's stores or a set of reductions; merging
at CTA level first costs one per (CTA tile, bucket) pair instead.  This counts both, and the buckets (= rays), per frame
of the bench stream, with the kernel's f32 arithmetic (each operation rounded, as under -fmad=false).

  python tools/bucket_pairs.py [--frames 64] [--start 0]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

VS = 0.05
STEP = 2
MIN_RAY, MAX_RAY = 0.3, 10.0  # the bench handle's defaults (tsdf_handle.py)


def bucket_keys(d, R):
    """Bucket coordinates (bx, by, bz) of every valid sampled pixel of depth image d under rotation R, and its
    sampled-pixel coordinates (ii, jj)."""
    from taichislam_b200 import synthetic as syn
    f32 = np.float32
    hh, ww = d.shape[0] // STEP, d.shape[1] // STEP
    jj, ii = np.meshgrid(np.arange(hh), np.arange(ww), indexing="ij")
    dv = d[jj * STEP, ii * STEP]
    df = dv.astype(f32)
    ok = (dv != 0) & ~((df > f32(MAX_RAY * 1000.0)) | (df < f32(MIN_RAY * 1000.0)))
    dep = df / f32(1000.0)
    x = ((ii * STEP).astype(f32) - f32(syn.CX)) * dep / f32(syn.FX)
    y = ((jj * STEP).astype(f32) - f32(syn.CY)) * dep / f32(syn.FY)
    R = R.astype(f32)
    p = [(R[r, 0] * x + R[r, 1] * y) + R[r, 2] * dep for r in range(3)]
    b = [np.floor(np.abs(q / f32(VS)) + f32(0.5)).astype(np.int64) * np.sign(q).astype(np.int64) for q in p]  # roundf
    return ii[ok], jj[ok], b[0][ok], b[1][ok], b[2][ok]


def distinct_pairs(tile, bx, by, bz):
    key = ((bx + 4096) << 26) | ((by + 4096) << 13) | (bz + 4096)
    return int(np.unique(np.stack([tile, key], 1), axis=0).shape[0]), int(np.unique(key).shape[0])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--start", type=int, default=0)
    args = ap.parse_args()
    import bench
    depth, Rs, _ = bench.make_inputs(args.frames, args.start)
    warp, cta, rays, px = [], [], [], []
    for q in range(args.frames):
        ii, jj, bx, by, bz = bucket_keys(depth[q], Rs[q])
        wtile = ((jj // 4) << 20) | (ii // 8)
        ctile = ((jj // 8) << 20) | (ii // 32)
        w, r = distinct_pairs(wtile, bx, by, bz)
        c, _ = distinct_pairs(ctile, bx, by, bz)
        warp.append(w); cta.append(c); rays.append(r); px.append(int(ii.shape[0]))
    out = {"frames": args.frames, "valid_px_per_frame": float(np.mean(px)),
           "warp_tile_bucket_pairs_per_frame": float(np.mean(warp)), "cta_tile_bucket_pairs_per_frame": float(np.mean(cta)),
           "buckets_per_frame": float(np.mean(rays)), "cta_over_warp": float(np.sum(cta) / np.sum(warp))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
