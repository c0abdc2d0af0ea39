#!/usr/bin/env python3
"""Trajectory optimisation against the occupancy ESDF (tslam_octo_esdf_trajectory) on the log-odds Octomap of scene_room
(512^3, 0.05 m, 40 frames, 5 m rays, as the other Octomap benches), ESDF max_dist 1 m.  Paths come from
travel_update_multi (clearance 0.2 m) between seeded traversable cells: 64 starts, each paired with reachable goals,
turned into control points at 0.1 m spacing and cut to at most 256 control points.  For T = 1, 64 and 1024 trajectories
per call: end-to-end ms per call (host clock around calls that end in a synchronise, after warm-up; min / median / max
over windows), ESDF samples per second inside the kernel (collision and check samples of all evaluations over the
call time), and the host-driven solve (tests/trajectory_reference.py with the GPU esdf_query, one round trip per
evaluation) for T = 1 and 64; and the fraction of trajectories whose dense check is all valid with min d >= c, before
(raw path as control points) and after.  Card name and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_trajectory.py [windows] [warmup]"""
import json, os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.octo_handle import OctoHandle
from taichislam_b200.trajectory import control_points
import trajectory_reference as tref

windows = int(sys.argv[1]) if len(sys.argv) > 1 else 5
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 1
LO = dict(l_hit=868, l_miss=-415, l_min=-2048, l_max=3595, l_occ=0)
VS, CL = 0.05, 0.2
SET = dict(max_iters=100, samples=4, check_samples=16, memory=8)
dev = torch.device("cuda", torch.cuda.current_device())

h = OctoHandle(512, 512, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH, logodds=LO)
depth = torch.from_numpy(syn.scene_room().astype(np.int16)).to(dev)
Rs, Ts = syn.stream_poses(40)
for q in range(40):
    h.integrate_depth(depth, Rs[q], Ts[q])
h.esdf_update(0, 1.0)
rng = np.random.default_rng(0)
h.travel_update(0, np.asarray(Ts[39], np.float32), CL)
ri, _ = h.travel_gather(0)                                  # traversable cells reachable from the last camera
starts = ri[rng.choice(len(ri), 64, replace=False)].astype(np.float32) * np.float32(VS)
h.travel_multi_update(0, starts, CL)
paths = []
while len(paths) < 1024:
    src = rng.integers(0, 64, 256).astype(np.int32)
    goal = ri[rng.choice(len(ri), 256)].astype(np.float32) * np.float32(VS)
    cells, ln = h.travel_multi_path(src, goal)
    for q in range(256):
        if ln[q] >= 8 and len(paths) < 1024:
            paths.append(control_points(cells[q, :ln[q]].astype(np.float64) * VS, 2 * VS)[:256])
paths = [np.concatenate([p[:-3], np.repeat(p[-4:-3], 3, 0)], 0) if len(p) == 256 else p for p in paths]


def call(qs, **kw):
    return h.esdf_trajectory(qs, CL, **dict(SET, **kw))


def samples_of(out, qs):
    """ESDF reads of a call: (N-3) K + 1 per evaluation, (N-3) C + 1 for the check"""
    return sum((len(q) - 3) * (SET["samples"] * o["evaluations"] + SET["check_samples"]) + 1 + o["evaluations"]
               for o, q in zip(out, qs))


res = {}
for T in (1, 64, 1024):
    qs = paths[:T]
    for _ in range(warmup):
        call(qs)
    ts = []
    reps = max(1, 64 // T)
    for _ in range(windows):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            out = call(qs)
        ts.append((time.perf_counter() - t0) * 1e3 / reps)
    before = call(qs, max_iters=0)
    r = dict(ms_min=min(ts), ms_median=float(np.median(ts)), ms_max=max(ts), ctrl_points=int(sum(len(q) for q in qs)),
             iterations_mean=float(np.mean([o["iterations"] for o in out])),
             evaluations_mean=float(np.mean([o["evaluations"] for o in out])),
             status=np.bincount([o["status"] for o in out], minlength=4).tolist(),
             esdf_samples_per_s=samples_of(out, qs) / (min(ts) * 1e-3),
             ok_before=float(np.mean([o["ok"] for o in before])), ok_after=float(np.mean([o["ok"] for o in out])))
    if T <= 64:
        fld = lambda x: h.esdf_query(np.ascontiguousarray(x, np.float32))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref = [tref.solve(q, fld, VS, clearance=CL, **SET) for q in qs]
        r["host_driven_ms"] = (time.perf_counter() - t0) * 1e3
        r["host_driven_same_bits"] = all(o["ctrl"].tobytes() == x["ctrl"].tobytes() for o, x in zip(out, ref))
    res[f"T{T}"] = r

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print(json.dumps(dict(bench="trajectory", card=card, clearance=CL, settings=SET, results=res)))
