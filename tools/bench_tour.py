#!/usr/bin/env python3
"""Exploration tours (tslam_tour_open) on two kinds of matrix, for n in {16, 65, 257, 1024} and R in {1, 132, 528}:
  * "room": travel_multi_query of n starts on the map of bench_octo_travel_multi.py (512^3, 0.05 m, 40 scene_room frames,
    max_ray_length 5 m), starts taken as there: the last camera cell, the reachable cell nearest each frontier-cluster
    centroid, then random reachable cells; beside it the travel_multi_update that built the matrix;
  * "random": Euclidean distances between uniform points in a 10 m cube times noise in [1, 1.3), asymmetric.
Per case: ms per solve (CUDA events, after warm-up), passes (mean and max over restarts), move evaluations per second
(each restart evaluates passes + 1 steps of every move), the best cost against the nearest-neighbour tour and against
R = 1, and the numpy reference's host time (tests/tour_reference.py) for R = 1 where it finishes in reasonable time,
else for one step.  Card name and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_tour.py [steps] [warmup]"""
import json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.octo_handle import OctoHandle
from taichislam_b200.tour import solve_open_tour
import tour_reference as tr

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 1
LO = dict(l_hit=868, l_miss=-415, l_min=-2048, l_max=3595, l_occ=0)
VS = 0.05
NS = (16, 65, 257, 1024)
RS = (1, 132, 528)
dev = torch.device("cuda", torch.cuda.current_device())


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n, out


def moves(m):  # 2-opt pairs plus Or-opt (L, i, p) triples of one step
    return m * (m - 1) // 2 + sum((m - L + 1) * (m - L) for L in (1, 2, 3) if m - L + 1 > 0)


# the room map and its starts, as bench_octo_travel_multi.py takes them
h = OctoHandle(512, 512, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH, logodds=LO)
depth = torch.from_numpy(syn.scene_room().astype(np.int16)).to(dev)
Rs, Ts = syn.stream_poses(40)
for q in range(40):
    h.integrate_depth(depth, Rs[q], Ts[q])
cam = np.asarray(Ts[39], np.float32)
h.frontier_update(0)
rec = h.frontier_clusters(0)
cent = rec[:, 2:5] / rec[:, 1:2]
rng = np.random.default_rng(0)
h.travel_update(0, cam)
ri, _ = h.travel_gather(0)
nr = np.array([ri[np.argmin(((ri - c) ** 2).sum(1))] for c in cent])
pool = np.concatenate([nr, ri[rng.choice(len(ri), max(NS), replace=False)]])
ALL = np.concatenate([cam[None], pool.astype(np.float32) * np.float32(VS)]).astype(np.float32)

res = {"steps": steps, "warmup": warmup, "map": "512^3, 0.05 m, scene_room x 40 frames, max_ray_length 5 m",
       "clusters": int(rec.shape[0]), "threads_per_cta": 256}
for n in NS:
    starts = ALL[:n]
    upd = lambda: h.travel_multi_update(0, starts)
    for _ in range(warmup):
        upd()
    t_upd = float(np.median([timed(upd, 1)[0] for _ in range(steps)]))
    room = h.travel_multi_query(torch.from_numpy(starts).to(dev)).contiguous()
    xyz = rng.uniform(0, 10, (n, 3))
    rand = torch.from_numpy((np.linalg.norm(xyz[:, None] - xyz[None], axis=2) * rng.uniform(1.0, 1.3, (n, n))).astype(np.float32)).to(dev)
    rand.fill_diagonal_(0)
    for kind, C in (("room", room), ("random", rand)):
        r = {"n": n}
        if kind == "room":
            r["travel_multi_update_ms"] = t_upd
        nn = solve_open_tour(C, restarts=1, max_passes=0)
        m = nn["m"]
        r.update(m=m, moves_per_step=moves(m), nn_inf_legs=nn["inf_legs"], nn_cost=nn["cost"])
        best1 = None
        for R in RS:
            call = lambda: solve_open_tour(C, restarts=R, seed=1)
            for _ in range(warmup):
                call()
            ms, out = timed(call, steps)
            ev = float((out["passes"].astype(np.int64) + 1).sum()) * moves(m)
            if R == 1:
                best1 = out["cost"]
            r[f"R={R}"] = dict(ms=ms, passes_mean=float(out["passes"].mean()), passes_max=int(out["passes"].max()),
                               converged=int(out["converged"].sum()), move_evals_per_s=ev / (ms * 1e-3),
                               inf_legs=out["inf_legs"], cost=out["cost"], vs_nn=out["cost"] / nn["cost"] if nn["cost"] else None,
                               vs_R1=out["cost"] / best1 if best1 else None)
        Ch = C.cpu().numpy()
        if m <= 257:
            t0 = time.perf_counter()
            tr.solve(Ch, restarts=1)
            r["reference_R1_host_s"] = time.perf_counter() - t0
        else:
            Wi, Wq, _ = tr.weights(Ch)
            t = [0] + [g for g in range(1, n) if Wi[0, g] == 0]
            tr.deltas(t, Wi, Wq)
            t0 = time.perf_counter()
            tr.deltas(t, Wi, Wq)
            r["reference_one_step_host_s"] = time.perf_counter() - t0
        res[f"{kind} n={n}"] = r
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
