#!/usr/bin/env python3
"""Frontier viewpoints of the log-odds Octomap: a 512^3 map (0.05 m voxels, max_ray_length = 5 m, recast_step 2) after 40
scene_room frames, the 640x480 depth camera at step 2 and 5 m.  CUDA events around `steps` calls after `warmup`, for
  * frontier_viewpoints with 48 samples (radii 1, 1.5, 2 m x 16 angles) and 144 samples (x heights 0, +-0.5 m), at
    top_k 1 and 4;
  * beside it, the frontier gain of the same poses (every candidate whose cell is FREE) through view_gain_frontier,
    against all clusters' voxels;
  * one plan_exploration step split into its public calls, host clock around each (each ends in a synchronise):
    frontier update (incremental, nothing changed), viewpoints (48 samples, top_k 4), travel update + costs of the kept
    viewpoints, tour.
Card name and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_octo_viewpoints.py [steps] [warmup]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.mapping.taichi_octomap import Octomap

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 3
VS = 0.05
dev = torch.device("cuda", torch.cuda.current_device())
o = Octomap(map_scale=[25.6, 25.6], voxel_scale=VS, occupancy_model="logodds", max_ray_length=5.0, max_disp_particles=16)
o.set_dep_camera_intrinsic(syn.K_DEPTH)
o.set_base_pose_submap(0, np.eye(3), np.zeros(3))
h = o._h
assert h.N == 512
depth = syn.scene_room()
Rs, Ts = syn.stream_poses(40)
for q in range(40):
    o.recast_depth_to_map(Rs[q], Ts[q], depth, None)
st = o.frontier_update()
CAM = dict(fx=syn.FX, fy=syn.FY, cx=syn.CX, cy=syn.CY, width=640, height=480, step=2, max_range=5.0)
OFFS = {48: Octomap.viewpoint_offsets((1.0, 1.5, 2.0), 16, (0.0,)), 144: Octomap.viewpoint_offsets((1.0, 1.5, 2.0), 16, (0.0, 0.5, -0.5))}


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
       "camera": "640x480, step 2, 5 m", "frontier_voxels": st["voxels"], "clusters": st["clusters"]}
rec = h.frontier_clusters(0)
cen = (rec[:, 2:5].astype(np.float64) / rec[:, 1:2].astype(np.float64) * float(np.float32(VS))).astype(np.float32)
for S, offs in OFFS.items():
    off = torch.from_numpy(offs).to(dev)
    for k in (1, 4):
        ms, (count, sample, visible, pos, R) = timed(lambda: h.frontier_viewpoints(off, CAM, top_k=k))
        res[f"viewpoints_S{S}_top{k}"] = {"ms_per_call": ms, "candidates": int(st["clusters"]) * S, "kept_slots": int(count.sum().item()),
                                         "mean_best_visible": float(visible[:, 0].double().mean().item())}
    # the same candidate poses (those on FREE cells) through the frontier gain against every cluster's voxels
    p = (cen[:, None, :] + offs[None]).reshape(-1, 3).astype(np.float32)
    d = (np.repeat(cen, S, 0) - p)
    hh = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).astype(np.float32)
    with np.errstate(all="ignore"):
        ux, uy = d[:, 0] / hh, d[:, 1] / hh
    z = np.zeros_like(ux)
    Rc = np.stack([np.stack([uy, z, ux], -1), np.stack([-ux, z, uy], -1), np.stack([z, z - 1, z], -1)], -2).astype(np.float32)
    ok = np.isfinite(Rc).all((1, 2))
    occ, unk = h.query_points(p)
    ok &= ~occ & ~unk
    pt, Rt = torch.from_numpy(p[ok]).to(dev), torch.from_numpy(Rc[ok]).to(dev)
    ms, (valid, total, per) = timed(lambda: h.view_gain_frontier(pt, Rt, CAM))
    res[f"view_gain_frontier_S{S}"] = {"ms_per_call": ms, "views": int(ok.sum()), "pairs": int(ok.sum()) * int(st["voxels"])}

# plan_exploration, one step split into its public calls, from the FREE cell nearest the last camera position
idx, L = h.gather(0)
free = idx[L <= o.l_occ].astype(np.float64) * float(np.float32(VS))
start = free[np.argmin(((free - Ts[-1]) ** 2).sum(1))]
times = {}
for rep in range(warmup + 1):
    t0 = time.perf_counter()
    o.frontier_update()
    t1 = time.perf_counter()
    fv = o.frontier_viewpoints(640, 480, radii=(1.0, 1.5, 2.0), angles=16, top_k=4, max_range=5.0, step=2, update=False)
    t2 = time.perf_counter()
    o.travel_update(start)
    kept = np.arange(4)[None, :] < fv["count"][:, None]
    cost = o.travel_cost(fv["pos"][kept])
    t3 = time.perf_counter()
    c = np.full(kept.shape, np.inf, np.float32)
    c[kept] = cost
    ok = kept & np.isfinite(c)
    goals = np.nonzero(ok.any(1))[0]
    tour = o.exploration_tour(start, fv["pos"][goals, np.argmax(ok, 1)[goals]])
    t4 = time.perf_counter()
    times = {"frontier_update_ms": (t1 - t0) * 1e3, "viewpoints_ms": (t2 - t1) * 1e3, "travel_update_and_costs_ms": (t3 - t2) * 1e3,
             "tour_ms": (t4 - t3) * 1e3, "goals": int(goals.size), "tour_goals": int(tour["order"].size)}
res["plan_exploration_breakdown"] = times
t0 = time.perf_counter()
plan = o.plan_exploration(start, 640, 480, top_k=4, max_range=5.0, step=2)
res["plan_exploration_ms"] = (time.perf_counter() - t0) * 1e3
res["plan_clusters"] = int(plan["clusters"].size)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
