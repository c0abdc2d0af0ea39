#!/usr/bin/env python3
"""Frame tracking against the TSDF (tslam_tsdf_track_depth): a 512^3 map (0.05 m voxels, max_ray_length 6 m) built from
the 40 frames of the box-room trajectory (tests/track_world.py) at their true poses.  For n = 1, 8 and 64 frames of
640x480 at step 2 (other dropout seeds than the map's), each from a start perturbed by 3 cm and 2 degrees:
  * end to end, host clock around `steps` synchronous calls after `warmup`, in `windows` separate windows (min / median
    / max over the windows): max_iters = 0 (selection plus one evaluation of every frame) and a full solve
    (max_iters = 20); "ms per LM iteration, end to end" = (solve - selection call) / (evaluations - 1), which includes
    the host LM step, the per-iteration upload, the D2H copy of the sums and the synchronisation;
  * GPU time of the kernels alone, from torch.profiler (CUPTI) in runs of their own: over one max_iters = 0 call (the
    one k_rg_eval launch covers every frame at its start pose) and over one full solve (mean per launch):
    k_rg_eval, k_rg_final, the selection kernel k_tr_select (count and fill) and the CUB scan;
  * points per second of the start-pose k_rg_eval launch, and of the selection call end to end.
Card name and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_frame_track.py [steps] [warmup] [windows]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
import track_world as tw
from taichislam_b200 import synthetic as syn
from taichislam_b200.tsdf_handle import TsdfHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 2
windows = int(sys.argv[3]) if len(sys.argv) > 3 else 5
VS, STEP = 0.05, 2
h = TsdfHandle(512, 512, voxel_scale=VS, K=syn.K_DEPTH, max_ray_length=6.0, max_submaps=4)
for k in range(tw.N_FRAMES):
    R, t = tw.pose(k)
    h.integrate_depth(tw.render(R, t, seed=k), R[None], t[None])
h.sync()
rng = np.random.default_rng(1)
frames = [tw.render(*tw.pose(k % tw.N_FRAMES), seed=1000 + k) for k in range(64)]
starts = [tw.perturb(*tw.pose(k % tw.N_FRAMES), rng, dt=0.03, deg=2.0) for k in range(64)]


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
    """mean GPU ms per launch of each tracking kernel over one call, from the profiler's CUDA activity"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    acc = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        name = e.name
        key = next((k for k in ("k_rg_eval", "k_rg_final") if k in name), None)
        if key is None and "k_tr_select" in name:
            key = "k_tr_select_count" if ("Lb1" in name or "true" in name) else "k_tr_select_fill"
        if key is None and "cub" in name.lower():
            key = "cub_scan"
        if key is None:
            continue
        n, t = acc.get(key, (0, 0.0))
        acc[key] = (n + 1, t + e.time_range.elapsed_us() / 1e3)
    return {k: {"launches": n, "ms_per_launch": t / n} for k, (n, t) in acc.items()}


res = {"steps": steps, "warmup": warmup, "windows": windows, "step": STEP, "image": "640x480",
       "map": "512^3, 0.05 m, 40 box-room frames, max_ray_length 6 m", "huber_m": VS}
for n in (1, 8, 64):
    d = np.stack(frames[:n])
    R0, T0 = np.stack([s[0] for s in starts[:n]]), np.stack([s[1] for s in starts[:n]])
    sel = lambda: h.track_depth(d, R0, T0, step=STEP, max_iters=0)
    solve = lambda: h.track_depth(d, R0, T0, step=STEP, max_iters=20)
    ms0, o0 = timed(sel)
    ms1, o1 = timed(solve)
    kern0, kern = kernel_ms(sel), kernel_ms(solve)
    evals = 1 + int(o1["iterations"].max())
    pts = int(o0["n_points"].sum())
    it_ms = [(ms1[i] - ms0[i]) / max(evals - 1, 1) for i in range(3)]
    ev = kern0.get("k_rg_eval", {"ms_per_launch": float("nan")})["ms_per_launch"]
    res[f"n{n}"] = {"points_per_frame_mean": pts / n, "valid_at_start": int(o0["n_valid"].sum()),
                    "ms_select_plus_one_evaluation_min_med_max": ms0, "ms_per_solve_min_med_max": ms1,
                    "ms_per_frame_solve_median": ms1[1] / n, "evaluations": evals,
                    "iterations_mean": float(o1["iterations"].mean()), "converged": int(o1["converged"].sum()),
                    "ms_per_lm_iteration_end_to_end_min_med_max": it_ms, "kernels_select_call": kern0, "kernels_solve": kern,
                    "k_rg_eval_ms_at_start": ev, "k_rg_eval_points_per_s_at_start": pts / (ev * 1e-3),
                    "select_call_points_per_s_end_to_end": pts / (ms0[1] * 1e-3)}
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
