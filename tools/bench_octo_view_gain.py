#!/usr/bin/env python3
"""Viewpoint gain of the log-odds Octomap: a 512^3 map (0.05 m voxels, max_ray_length = 5 m, recast_step 2) after 40
scene_room frames on the device, then 256 views on FREE cells around the frontier-cluster centroids (random yaw, pitch
within +-0.3 rad).  CUDA events around `steps` batches after `warmup`, for
  * the unknown gain with the 640x480 depth camera at step 2 and at step 4, 5 m;
  * the frontier gain with the same camera at step 2 and the map's clusters.
Reported per batch: ms, rays/s, nominal cell visits/s (rays x max_range / vs: the walks stop
earlier at the first OCC cell or the volume boundary), frontier (view, voxel) pairs/s, and the bitmap scratch of one chunk.
Card name and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_octo_view_gain.py [steps] [warmup]"""
import json, math, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.octo_handle import OctoHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 3
LO = dict(l_hit=868, l_miss=-415, l_min=-2048, l_max=3595, l_occ=0)
VS = 0.05
N_VIEWS = 256
dev = torch.device("cuda", torch.cuda.current_device())
h = OctoHandle(512, 512, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH, logodds=LO)
depth = torch.from_numpy(syn.scene_room().astype(np.int16)).to(dev)
Rs, Ts = syn.stream_poses(40)
for q in range(40):
    h.integrate_depth(depth, Rs[q], Ts[q])
st = h.frontier_update(0)
rec = h.frontier_clusters(0)
idx, L = h.gather(0)
free = idx[L <= LO["l_occ"]].astype(np.int64)
cent = rec[:, 2:5] / rec[:, 1:2]
rng = np.random.default_rng(0)
# FREE cells nearest to randomly chosen cluster centroids (jittered by up to 0.5 m)
targets = cent[rng.integers(len(cent), size=N_VIEWS)] + rng.uniform(-10, 10, (N_VIEWS, 3))
near = np.array([free[np.argmin(((free - t) ** 2).sum(1))] for t in targets])
pos = torch.from_numpy((near.astype(np.float32) * np.float32(VS))).to(dev)


def rot(yaw, pitch):
    cy, sy, cp, sp = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch)
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, cp, -sp], [0, sp, cp]])
    return Rz @ Rx


R = torch.from_numpy(np.stack([rot(rng.uniform(-math.pi, math.pi), rng.uniform(-0.3, 0.3)) for _ in range(N_VIEWS)]).astype(np.float32)).to(dev)
CAM = dict(fx=syn.FX, fy=syn.FY, cx=syn.CX, cy=syn.CY, width=640, height=480, max_range=5.0)


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


def scratch_bytes(cam):
    ww, hh, step, dep = cam["width"] // cam["step"], cam["height"] // cam["step"], cam["step"], float(np.float32(cam["max_range"]))
    fx, fy, cx, cy = (float(np.float32(cam[k])) for k in ("fx", "fy", "cx", "cy"))
    r2 = max((((i - cx) * dep / fx) ** 2 + ((j - cy) * dep / fy) ** 2 + dep * dep) for i in (0, (ww - 1) * step) for j in (0, (hh - 1) * step))
    e = 2 * (math.ceil(math.sqrt(r2) / float(np.float32(VS))) + 2) + 1
    per = ((min(e, 512) ** 3 + 31) // 32) * 4
    chunk = max(1, min(N_VIEWS, (256 << 20) // per))
    return per, chunk, per * chunk


res = {"steps": steps, "warmup": warmup, "views": N_VIEWS, "map": "512^3, 0.05 m, scene_room x 40 frames, max_ray_length 5 m",
       "frontier_voxels": st["voxels"], "clusters": st["clusters"], "known_voxels": int(idx.shape[0])}
for step in (2, 4):
    cam = dict(CAM, step=step)
    ms, (valid, gain) = timed(lambda: h.view_gain_unknown(pos, R, cam))
    rays = N_VIEWS * (640 // step) * (480 // step)
    per, chunk, scratch = scratch_bytes(cam)
    visits = rays * (5.0 / VS)
    res[f"unknown_step{step}"] = {"ms_per_batch": ms, "rays_per_s": rays / ms * 1e3, "nominal_cell_visits_per_s": visits / ms * 1e3,
                                  "valid_views": int(valid.sum().item()), "mean_gain": float(gain.double().mean().item()),
                                  "bitmap_bytes_per_view": per, "views_per_chunk": chunk, "scratch_bytes": scratch}
cam = dict(CAM, step=2)
ms, (valid, total, per) = timed(lambda: h.view_gain_frontier(pos, R, cam))
pairs = N_VIEWS * st["voxels"]
res["frontier"] = {"ms_per_batch": ms, "pairs_per_s": pairs / ms * 1e3, "pairs": pairs,
                   "mean_visible": float(total.double().mean().item()), "row_sums_equal_totals": bool((per.sum(1) == total).all().item())}
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
