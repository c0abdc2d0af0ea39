#!/usr/bin/env python3
"""ESDF query throughput on one GPU (tslam_esdf_query): 100 frames of the S2 stream into a 512^3 map, one ESDF update,
then 2^20-point batches timed with CUDA events after warm-up, for
  * uniform: points uniform over the observed voxels (a random observed voxel + a uniform offset inside it);
  * polylines: the same points reordered along a Z-order curve of their voxels and cut into 1024 runs of 1024
    points, so that consecutive queries are neighbours as along a planner's polylines (they share corner blocks).
Prints one JSON line: queries/s per pattern, the algorithmic bytes per query (12 B in, 16 B + 1 B out, 8 corners x
(4 B ESDF + 1 B class)) and the rate they imply, the card's name and power limit read in the same run.
Usage: python tools/bench_esdf_query.py [reps]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.tsdf_handle import TsdfHandle

BYTES_PER_QUERY = 12 + 16 + 1 + 8 * (4 + 1)
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
n = 1 << 20
vs = 0.05

g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
d = syn.scene_sphere(4.0)
Rs, Ts = syn.stream_poses(100)
g.integrate_depth(np.ascontiguousarray(np.broadcast_to(d, (100,) + d.shape)), Rs, Ts)
sw = g.esdf_update()
idx = g.gather()[0]
rng = np.random.default_rng(0)
uni = ((idx[rng.integers(0, idx.shape[0], n)] + rng.uniform(0.0, 1.0, size=(n, 3))) * vs).astype(np.float32)
vox = (np.floor(uni / np.float32(vs)).astype(np.int64) + 256) & 511   # (in-volume voxel of each point, 9 bits per axis)
morton = np.zeros(n, np.int64)
for b in range(9):
    for a in range(3):
        morton |= ((vox[:, a] >> b) & 1) << (3 * b + a)
order = np.argsort(morton, kind="stable").reshape(1024, 1024)
poly = uni[order[rng.permutation(1024)].reshape(n)]               # runs in random order, each run in curve order

out = {"map": "512^3, 100 S2-stream frames", "esdf_sweeps": sw, "observed_voxels": int(idx.shape[0]), "batch": n,
       "reps": reps, "bytes_per_query": BYTES_PER_QUERY}
for name, pts in (("uniform", uni), ("polylines", poly)):
    x = torch.from_numpy(pts).cuda()
    for _ in range(5):
        dist, grad, valid = g.esdf_query(x)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dist, grad, valid = g.esdf_query(x)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    out[name] = {"ms_per_batch": ms, "queries_per_s": n / (ms * 1e-3), "valid_frac": float(valid.float().mean()),
                 "alg_GBs": n * BYTES_PER_QUERY / (ms * 1e-3) / 1e9}
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                      str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
out["gpu"] = torch.cuda.get_device_name()
out["nvidia_smi_name_power_limit_max_sm_clock"] = smi
print(json.dumps(out), flush=True)
g.close()
