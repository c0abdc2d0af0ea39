#!/usr/bin/env python3
"""Rendering of the TSDF's zero level (tslam_tsdf_render): a 512^3 map (0.05 m voxels, max_ray_length 6 m) built from
the 40 frames of the box-room trajectory (tests/track_world.py) at their true poses.  For n = 1, 8 and 64 cameras of
640x480 at trajectory poses (z 0.3 .. 6 m, step = one voxel, normals on):
  * end to end, host clock around `steps` calls and a synchronise after `warmup`, in `windows` separate windows (min /
    median / max over the windows of the mean ms per call);
  * GPU time of k_render alone, from torch.profiler (CUPTI) in a run of its own (mean over `steps` launches);
  * rays per second, and evaluated samples per second, the samples of a ray taken from the output: the hit sample + 2
    (samples k and k + 1 of the crossing, counted from z_min), or K on a miss - an upper count, since the kernel stops
    once a ray leaves the volume.
k_render does per sample the 8-corner gather and trilinear interpolation that k_rg_eval does per point (DESIGN.md
section 7).  Card name and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_render.py [steps] [warmup] [windows]"""
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
VS, Z_MIN, Z_MAX = 0.05, 0.3, 6.0
h = TsdfHandle(512, 512, voxel_scale=VS, K=syn.K_DEPTH, max_ray_length=Z_MAX, min_ray_length=Z_MIN, max_submaps=4)
for k in range(tw.N_FRAMES):
    R, t = tw.pose(k)
    h.integrate_depth(tw.render(R, t, seed=k), R[None], t[None])
h.sync()
K = int(np.floor((float(np.float32(Z_MAX)) - float(np.float32(Z_MIN))) / float(np.float32(VS)))) + 1
poses = [tw.pose((3 * c) % tw.N_FRAMES) for c in range(64)]


def timed(fn):
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
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    ts = [e.time_range.elapsed_us() / 1e3 for e in prof.events() if e.device_type.name == "CUDA" and "k_render" in e.name]
    return {"launches": len(ts), "ms_per_launch": float(np.mean(ts)) if ts else float("nan")}


res = {"steps": steps, "warmup": warmup, "windows": windows, "image": "640x480", "z_range_m": [Z_MIN, Z_MAX], "step_m": VS,
       "samples_per_ray_K": K, "map": "512^3, 0.05 m, 40 box-room frames, max_ray_length 6 m"}
for n in (1, 8, 64):
    Rs, Ts = np.stack([p[0] for p in poses[:n]]), np.stack([p[1] for p in poses[:n]])
    call = lambda: h.render(Rs, Ts, syn.H, syn.W, syn.K_DEPTH, z_min=Z_MIN, z_max=Z_MAX, step=VS)
    ms, out = timed(call)
    kern = kernel_ms(call)
    depth, status = out[0].cpu().numpy().astype(np.float64), out[1].cpu().numpy()
    hit = status > 0
    ksamp = np.floor((depth - np.float32(Z_MIN)) / np.float32(VS)).astype(np.int64) + 2   # sample k of the crossing, + 2
    samples = float(np.where(hit, np.minimum(ksamp, K), K).sum())
    rays = n * syn.H * syn.W
    res[f"n{n}"] = {"ms_per_call_end_to_end_min_med_max": ms, "k_render": kern, "hit_fraction": float(hit.mean()),
                    "status1_fraction": float((status == 1).mean()), "samples_per_ray_mean": samples / rays,
                    "rays_per_s_end_to_end": rays / (ms[1] * 1e-3), "rays_per_s_kernel": rays / (kern["ms_per_launch"] * 1e-3),
                    "samples_per_s_kernel": samples / (kern["ms_per_launch"] * 1e-3)}
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
