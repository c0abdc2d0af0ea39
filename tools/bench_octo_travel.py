#!/usr/bin/env python3
"""Travel cost on the log-odds Octomap: a 512^3 map (0.05 m voxels, max_ray_length = 5 m) after 40 scene_room frames on
the device, then
  * travel_update from the last camera cell with clearance 0 and 0.2 m (occupancy ESDF, D = 1 m): ms per update, sweeps,
    host flag reads, reachable and traversable cells; a full ESDF update in the same run for scale;
  * travel_query of 2^20 points (reachable cells, jittered inside the cell);
  * travel_path of 256 targets: the reachable cells nearest to randomly chosen frontier-cluster centroids.
CUDA events around `steps` calls after `warmup`.  Card name and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_octo_travel.py [steps] [warmup]"""
import json, math, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.octo_handle import OctoHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 3
LO = dict(l_hit=868, l_miss=-415, l_min=-2048, l_max=3595, l_occ=0)
VS = 0.05
ES_GROUP = 6  # sweeps per host flag read (tslam_esdf_common.cuh)
dev = torch.device("cuda", torch.cuda.current_device())
h = OctoHandle(512, 512, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH, logodds=LO)
depth = torch.from_numpy(syn.scene_room().astype(np.int16)).to(dev)
Rs, Ts = syn.stream_poses(40)
for q in range(40):
    h.integrate_depth(depth, Rs[q], Ts[q])
start = np.asarray(Ts[39], np.float32)
idx, L = h.gather(0)


def timed(fn):
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = fn()
    e1.record()
    h.sync()
    return e0.elapsed_time(e1) / steps, out


res = {"steps": steps, "warmup": warmup, "map": "512^3, 0.05 m, scene_room x 40 frames, max_ray_length 5 m",
       "known_voxels": int(idx.shape[0]), "start": start.tolist()}
ms, _ = timed(lambda: h.esdf_update(0, 1.0, full=True))
res["esdf_full_update_ms"] = ms
for cl in (0.0, 0.2):
    ms, st = timed(lambda: h.travel_update(0, start, clearance=cl))
    res[f"update_clearance_{cl}"] = dict(ms=ms, sweeps=st["sweeps"], host_flag_reads=math.ceil(st["sweeps"] / ES_GROUP),
                                         ms_per_sweep=ms / max(st["sweeps"], 1), reachable=st["reachable"],
                                         traversable=st["traversable"], start_ok=st["start_ok"])
# queries and paths against the clearance-0 field
st = h.travel_update(0, start)
ri, rG = h.travel_gather(0)
rng = np.random.default_rng(0)
n = 1 << 20
pts = ri[rng.integers(len(ri), size=n)].astype(np.float32) * np.float32(VS) + rng.uniform(-0.45, 0.45, (n, 3)).astype(np.float32) * np.float32(VS)
x = torch.from_numpy(pts.astype(np.float32)).to(dev)
ms, cost = timed(lambda: h.travel_query(x))
res["query"] = dict(points=n, ms=ms, points_per_s=n / ms * 1e3, finite=int(torch.isfinite(cost).sum().item()))
h.frontier_update(0)
rec = h.frontier_clusters(0)
cent = rec[:, 2:5] / rec[:, 1:2]
tg = cent[rng.integers(len(cent), size=256)]
near = np.array([ri[np.argmin(((ri - t) ** 2).sum(1))] for t in tg])
xt = torch.from_numpy(near.astype(np.float32) * np.float32(VS)).to(dev)
ms, (cells, ln) = timed(lambda: h.travel_path(xt, max_len=4096))
res["paths"] = dict(targets=256, ms=ms, mean_len=float(ln.double().mean().item()), max_len=int(ln.max().item()),
                    reached=int((ln > 0).sum().item()), clusters=int(rec.shape[0]))
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
