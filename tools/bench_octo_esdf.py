#!/usr/bin/env python3
"""Occupancy ESDF of the log-odds Octomap: scene_room depth frames streamed into a 512^3 map (0.05 m voxels,
max_ray_length = 5 m, recast_step 2, frames on the device, poses from synthetic.stream_poses), for D = 1 m and 2 m.
CUDA events around `steps` frames after `warmup` (every update synchronises the host once per sweep group, so the
window is wall time of the stream).  Per D it reports, per frame:
  * integrate only;
  * integrate + incremental tslam_octo_esdf_update (and the update's changed / suspect voxels and sweeps);
  * integrate + full update (mode 1) on an identical map - the two fields are then compared bit for bit;
and query throughput for 2^20 points drawn uniformly from the voxels known at the end, in that random order and
sorted in Z (Morton) order.  Card name and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_octo_esdf.py [steps] [warmup]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.octo_handle import OctoHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 40
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 5
LO = dict(l_hit=868, l_miss=-415, l_min=-2048, l_max=3595, l_occ=0)
VS = 0.05
dev = torch.device("cuda", torch.cuda.current_device())
depth = torch.from_numpy(syn.scene_room().astype(np.int16)).to(dev)
Rs, Ts = syn.stream_poses(warmup + steps)


def stream(D, mode):
    """mode None: integrate only; 0: + incremental update; 1: + full update -> (ms per frame, per-frame stats, handle)"""
    h = OctoHandle(512, 512, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH, logodds=LO)
    for q in range(warmup):
        h.integrate_depth(depth, Rs[q], Ts[q])
        if mode is not None:
            h.esdf_update(0, D, full=bool(mode))
    h.sync()
    stats = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for q in range(warmup, warmup + steps):
        h.integrate_depth(depth, Rs[q], Ts[q])
        if mode is not None:
            stats.append(h.esdf_update(0, D, full=bool(mode)))
    e1.record()
    h.sync()
    return e0.elapsed_time(e1) / steps, stats, h


def morton(c):
    c = (c - c.min(0)).astype(np.uint64)
    k = np.zeros(len(c), np.uint64)
    for b in range(10):
        for a in range(3):
            k |= ((c[:, a] >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b + a)
    return np.argsort(k, kind="stable")


def query_rate(h, pts, reps=20):
    x = torch.from_numpy(pts).to(dev)
    for _ in range(3):
        h.esdf_query(x)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        r = h.esdf_query(x)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    return {"ms": ms, "points_per_s": pts.shape[0] / (ms / 1000.0), "valid": float(r[2].float().mean())}


res = {"steps": steps, "warmup": warmup, "map": "512^3, 0.05 m, scene_room, max_ray_length 5 m"}
ms_int, _, h0 = stream(None, None)
h0.close()
res["integrate_ms_per_frame"] = ms_int
for D in (1.0, 2.0):
    ms_inc, st_inc, hi = stream(D, 0)
    ms_full, st_full, hf = stream(D, 1)
    ii, ie = hi.esdf_gather(0)
    fi, fe = hf.esdf_gather(0)
    oi, of = np.lexsort(ii.T[::-1]), np.lexsort(fi.T[::-1])
    same = bool(np.array_equal(ii[oi], fi[of]) and np.array_equal(ie[oi].view(np.int32), fe[of].view(np.int32)))
    mean = lambda k, s: float(np.mean([x[k] for x in s]))
    r = {"integrate_plus_incremental_ms_per_frame": ms_inc, "integrate_plus_full_ms_per_frame": ms_full,
         "incremental_update_ms_per_frame": ms_inc - ms_int, "full_update_ms_per_frame": ms_full - ms_int,
         "changed_voxels_per_frame": mean("changed", st_inc), "suspect_voxels_per_frame": mean("suspect", st_inc),
         "raise_sweeps_per_frame": mean("raise_sweeps", st_inc), "lower_sweeps_incremental": mean("lower_sweeps", st_inc),
         "lower_sweeps_full": mean("lower_sweeps", st_full), "known_voxels": int(ii.shape[0]), "incremental_equals_full": same}
    if D == 1.0:
        rng = np.random.default_rng(0)
        pick = ii[rng.integers(0, ii.shape[0], 1 << 20)]
        pts = ((pick + rng.random((1 << 20, 3))) * VS).astype(np.float32)
        r["query_uniform"] = query_rate(hi, pts)
        r["query_zorder"] = query_rate(hi, np.ascontiguousarray(pts[morton(pick)]))
    res[f"D_{D:g}m"] = r
    hi.close()
    hf.close()
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
