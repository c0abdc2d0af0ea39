#!/usr/bin/env python3
"""SDF-to-SDF registration of TSDF submap pairs (tslam_tsdf_register): a 512^3 map (0.05 m voxels, max_ray_length 6 m)
with two overlapping scene_room submaps (the recovery scenario of tests/submap_register_reference.py: base poses 30
degrees and 0.7 m apart, two frames each).  For P = 1, 8 and 64 pairs (alternately 0 -> 1 and 1 -> 0, each from a start
perturbed by up to 0.1 m and 3 degrees):
  * end to end, host clock around `steps` synchronous calls after `warmup`, in `windows` separate windows (min / median
    / max over the windows): max_iters = 0 (point selection plus one evaluation of every pair) and a full solve
    (max_iters = 20); "ms per LM iteration, end to end" = (solve - selection call) / (evaluations - 1), which includes
    the host LM step, the per-iteration upload, the D2H copy of the sums and the synchronisation;
  * GPU time of the kernels alone, from torch.profiler (CUPTI), over one max_iters = 0 call (the one k_rg_eval launch
    covers every pair at its start pose) and over one full solve (mean per launch; later launches cover only the pairs
    still active): k_rg_eval, k_rg_final, and the selection kernels (count, CUB sort and scan, permute, fill);
  * points per second of the start-pose k_rg_eval launch, and its algorithmic bytes (16 B record per point, 8 corners x
    (8 B TSDF/weight + 1 B observed) per valid point).
Card name and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_submap_register.py [steps] [warmup] [windows]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
import submap_register_reference as ref
from taichislam_b200 import synthetic as syn
from taichislam_b200.tsdf_handle import TsdfHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 2
windows = int(sys.argv[3]) if len(sys.argv) > 3 else 5
VS = 0.05
h = TsdfHandle(512, 512, voxel_scale=VS, K=syn.K_DEPTH, max_ray_length=6.0, max_submaps=4)
for s, base, seeds in ((0, ref.ROOM_BASE_A, ref.ROOM_SEEDS_A), (1, ref.ROOM_BASE_B, ref.ROOM_SEEDS_B)):
    R, T = ref.local_pose(base)
    for sd in seeds:
        h.integrate_depth(syn.scene_room(seed=sd), R[None], T[None], submaps=[s])
h.sync()
Rab, tab = ref.true_relative(ref.ROOM_BASE_A, ref.ROOM_BASE_B)
Rba, tba = Rab.T, -Rab.T @ tab


def pairs(P):
    a, b, R0, T0 = [], [], [], []
    for p in range(P):
        Rt, tt = (Rab, tab) if p % 2 == 0 else (Rba, tba)
        R, T = ref.perturbed(Rt, tt, p % 3)
        a.append(p % 2); b.append(1 - p % 2); R0.append(R); T0.append(T)
    return a, b, np.array(R0), np.array(T0)


def timed(fn):
    """min / median / max over the windows of the mean ms per call, and the last output"""
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(windows):
        t0 = time.perf_counter()
        for _ in range(steps):
            out = fn()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3 / steps)
    return [min(ms), float(np.median(ms)), max(ms)], out


def kernel_ms(fn):
    """mean GPU ms per launch of each registration kernel over one call, from the profiler's CUDA activity"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    acc = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        name = e.name
        key = next((k for k in ("k_rg_eval", "k_rg_final", "k_rg_count", "k_rg_permute", "k_rg_fill") if k in name),
                   "cub" if "cub" in name.lower() else None)
        if key is None:
            continue
        n, t = acc.get(key, (0, 0.0))
        acc[key] = (n + 1, t + e.time_range.elapsed_us() / 1e3)
    return {k: {"launches": n, "ms_per_launch": t / n} for k, (n, t) in acc.items()}


res = {"steps": steps, "warmup": warmup, "windows": windows,
       "map": "512^3, 0.05 m, two scene_room submaps x 2 frames, max_ray_length 6 m", "band_m": 4 * VS, "huber_m": VS}
for P in (1, 8, 64):
    a, b, R0, T0 = pairs(P)
    sel = lambda: h.register(h, a, b, R0, T0, 4 * VS, max_iters=0)
    solve = lambda: h.register(h, a, b, R0, T0, 4 * VS, max_iters=20)
    ms0, o0 = timed(sel)
    ms1, o1 = timed(solve)
    kern0, kern = kernel_ms(sel), kernel_ms(solve)
    evals = 1 + int(o1["iterations"].max())
    pts = int(o0["n_points"].sum())
    valid = int(o0["n_valid"].sum())
    it_ms = [(ms1[i] - ms0[i]) / max(evals - 1, 1) for i in range(3)]
    ev = kern0.get("k_rg_eval", {"ms_per_launch": float("nan")})["ms_per_launch"]   # one launch, every pair at its start
    res[f"P{P}"] = {"points_per_pair": [int(v) for v in sorted(set(o0["n_points"].tolist()))], "valid_at_start": valid,
                    "ms_select_plus_one_evaluation_min_med_max": ms0, "ms_per_solve_min_med_max": ms1, "evaluations": evals,
                    "iterations_mean": float(o1["iterations"].mean()), "converged": int(o1["converged"].sum()),
                    "ms_per_lm_iteration_end_to_end_min_med_max": it_ms, "kernels_select_call": kern0, "kernels_solve": kern,
                    "k_rg_eval_ms_at_start": ev,
                    "k_rg_eval_points_per_s_at_start": pts / (ev * 1e-3), "bytes_per_evaluation_at_start": 16 * pts + 72 * valid,
                    "k_rg_eval_GB_per_s_at_start": (16 * pts + 72 * valid) / (ev * 1e-3) / 1e9}
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
