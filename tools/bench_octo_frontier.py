#!/usr/bin/env python3
"""Frontiers of the log-odds Octomap: scene_room depth frames streamed into a 512^3 map (0.05 m voxels,
max_ray_length = 5 m, recast_step 2, frames on the device, poses from synthetic.stream_poses).  CUDA events around
`steps` frames after `warmup` (every update synchronises the host a few times, so the window is wall time of the
stream).  Per frame it reports:
  * integrate only;
  * integrate + incremental tslam_octo_frontier_update;
  * integrate + full update (mode 1) on an identical map - the two frontier sets and cluster lists are then compared;
and the frontier voxels, clusters and blocks re-examined per frame.  Card name and power limit are read in the same
run.  One JSON line.
Usage: python tools/bench_octo_frontier.py [steps] [warmup]"""
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


def stream(mode):
    """mode None: integrate only; 0: + incremental update; 1: + full update -> (ms per frame, per-frame stats, handle)"""
    h = OctoHandle(512, 512, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH, logodds=LO)
    for q in range(warmup):
        h.integrate_depth(depth, Rs[q], Ts[q])
        if mode is not None:
            h.frontier_update(0, full=bool(mode))
    h.sync()
    stats = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for q in range(warmup, warmup + steps):
        h.integrate_depth(depth, Rs[q], Ts[q])
        if mode is not None:
            stats.append(h.frontier_update(0, full=bool(mode)))
    e1.record()
    h.sync()
    return e0.elapsed_time(e1) / steps, stats, h


def state(h):
    idx, cl = h.frontier_gather(0)
    o = np.lexsort(idx.T[::-1])
    return idx[o], cl[o], h.frontier_clusters(0)


res = {"steps": steps, "warmup": warmup, "map": "512^3, 0.05 m, scene_room, max_ray_length 5 m"}
ms_int, _, h0 = stream(None)
h0.close()
ms_inc, st_inc, hi = stream(0)
ms_full, st_full, hf = stream(1)
a, b = state(hi), state(hf)
same = all(np.array_equal(x, y) for x, y in zip(a, b))
mean = lambda k, s: float(np.mean([x[k] for x in s]))
res.update({"integrate_ms_per_frame": ms_int, "integrate_plus_incremental_ms_per_frame": ms_inc,
            "integrate_plus_full_ms_per_frame": ms_full, "incremental_update_ms_per_frame": ms_inc - ms_int,
            "full_update_ms_per_frame": ms_full - ms_int, "frontier_voxels_per_frame": mean("voxels", st_inc),
            "frontier_voxels_max": int(max(x["voxels"] for x in st_inc)), "clusters_per_frame": mean("clusters", st_inc),
            "blocks_reexamined_incremental": mean("blocks", st_inc), "blocks_reexamined_full": mean("blocks", st_full),
            "incremental_updates_full": int(sum(x["full"] for x in st_inc)), "known_voxels": int(hi.gather(0)[0].shape[0]),
            "incremental_equals_full": bool(same)})
hi.close()
hf.close()
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
