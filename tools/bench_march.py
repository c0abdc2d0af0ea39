#!/usr/bin/env python3
"""Per-kernel CUDA-event times of the integrate launch (block-binned march) for the four scenes on one GPU.  Prints one
JSON line per scene.
Usage: python tools/bench_march.py [reps]"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.tsdf_handle import TsdfHandle

PEAK = 6564.2
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
for name, d in (("S2 sphere 4 m", syn.scene_sphere(4.0)), ("S1 plane 3 m", syn.scene_plane(3.0)), ("S3 sphere 8 m", syn.scene_sphere(8.0)),
                ("S4 noise 1.5-4.5 m", syn.scene_noise())):
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    dd = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(d, (64,) + d.shape)).view(np.int16)).cuda()
    for w in range(3):
        Rs, Ts = syn.stream_poses(64, start=64 * w)
        g.integrate_depth(dd, Rs, Ts)
    g.stats(clear=True)
    g.set_profiling(True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for r in range(reps):
        Rs, Ts = syn.stream_poses(64, start=64 * (3 + r))
        g.integrate_depth(dd, Rs, Ts)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    st = g.stats()
    k = g.kernel_ms2(reps).mean(axis=0)
    rays, upd = st["n_rays"] / reps, st["n_updates"] / reps
    alg = 17.0 * rays + 9.0 * upd
    out = {"scene": name, "frames_per_s": 64e3 / ms, "ms_per_64": ms, "rays": rays, "updates": upd,
           "kernel_ms": {"bucket": float(k[0]), "raymarch_total": float(k[1]), "commit": float(k[2]), "setup": float(k[3]),
                         "scan": float(k[4]), "fill": float(k[5]), "march": float(k[6])},
           "raymarch_alg_GBs": float(alg / (k[1] * 1e-3) / 1e9), "raymarch_frac": float(alg / (k[1] * 1e-3) / 1e9 / PEAK),
           "n_oob": st["n_oob"], "blocks": st["n_blocks"], "err": st["err_flags"]}
    try:
        ms_ = g.march_stats()
        out["march_stats_per_launch"] = {kk: v / reps for kk, v in ms_.items()}
    except Exception as ex:
        out["march_stats_per_launch"] = repr(ex)
    print(json.dumps(out), flush=True)
    g.close()
