#!/usr/bin/env python3
"""Kernel chain of one integrate launch, from torch.profiler (CUPTI): where the launch's time goes between kernels.

Runs the device-resident arm of bench.py - a 512^3 map, the S2 stream, 64-frame depth launches with commit, the same
three warm-up steps of 16 launches and profiling on as bench.py sets it (kernel_ms2) - then traces a few launches
in a run of their own.  Writes OUT/trace.json (Chrome trace) and OUT/summary.json, and prints the summary:

  kernels          per kernel name: launches, mean and total duration (us)
  gaps             idle time between consecutive kernels of a launch (k_bucket_depth opens a launch), per kernel pair
                   (mean, median, min, max; negative where a programmatic dependent launch starts before its predecessor ends)
  bookkeeping      kernels that do no voxel work (class/scan, generic march, resets, dirty-list compaction)
  share            (bookkeeping kernel time + all gaps inside the launches) / launch span, and each part alone

The card's name and power limit are read in the same run.
The first --skip traced launches (default 1) are left out of the statistics: the first launch after the synchronise
waits on the host, which enqueues it under the profiler for the first time.
Usage: python tools/trace_integrate.py [--out DIR] [--launches K] [--skip S] [--no-events]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH, LAUNCHES_PER_STEP, POOL_BATCHES = 64, 16, 4
BOOKKEEPING = ("k_seg_class", "k_seg_scan", "k_seg_class_scan", "k_march_generic", "k_march_reset", "k_reset_counters",
               "k_collect_dirty")


def base_name(name):
    """'void k_march_blocks<false, 320, 3>(TsBatch, ...)' -> 'k_march_blocks'"""
    s = name.split("(")[0]
    s = s.split("<")[0]
    return s.split()[-1] if s.split() else name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "trace_integrate"),
                    help="output directory (default: trace_integrate under the system temporary directory)")
    ap.add_argument("--launches", type=int, default=8)
    ap.add_argument("--skip", type=int, default=1, help="traced launches left out of the statistics at the start")
    ap.add_argument("--warmup", type=int, default=3, help="warm-up steps of 16 launches (bench.py's default)")
    ap.add_argument("--no-events", action="store_true", help="trace with profiling off (bench.py times its launches with it on)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from taichislam_b200 import synthetic as syn
    from taichislam_b200.tsdf_handle import TsdfHandle

    torch.cuda.set_device(0)
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    pool = []
    for b in range(POOL_BATCHES):
        d, _, _ = bench.make_inputs(BATCH, b * BATCH)
        pool.append(torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda())
    n_launches = args.warmup * LAUNCHES_PER_STEP + args.skip + args.launches
    Rs, Ts = syn.stream_poses(n_launches * BATCH, start=0)
    Rs = np.ascontiguousarray(Rs.astype(np.float32).reshape(n_launches, BATCH, 9))
    Ts = np.ascontiguousarray(Ts.astype(np.float32).reshape(n_launches, BATCH, 3))

    def launch(k):
        g.integrate_depth(pool[k % POOL_BATCHES], Rs[k], Ts[k], commit=True)

    k = 0
    for _ in range(args.warmup * LAUNCHES_PER_STEP):
        launch(k)
        k += 1
    g.set_profiling(not args.no_events)
    l0 = g.launch_count()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.skip + args.launches):
            launch(k)
            k += 1
        torch.cuda.synchronize()
    kernels_per_launch = (g.launch_count() - l0) / (args.skip + args.launches)
    os.makedirs(args.out, exist_ok=True)
    trace_path = os.path.join(args.out, "trace.json")
    prof.export_chrome_trace(trace_path)
    g.close()

    with open(trace_path) as f:
        tr = json.load(f)
    evs = [e for e in tr["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    evs.sort(key=lambda e: float(e["ts"]))
    seq = [(base_name(e["name"]) if e["cat"] == "kernel" else e["cat"], float(e["ts"]), float(e["dur"])) for e in evs]
    # split into launches: each one opens with the bucket kernel
    launches, cur = [], None
    for s in seq:
        if s[0] == "k_bucket_depth":
            cur = []
            launches.append(cur)
        if cur is not None:
            cur.append(s)
    launches = launches[args.skip:]
    per_kernel, gaps = {}, {}
    spans, book_us, gap_us, between = [], [], [], []
    for i, L in enumerate(launches):
        t0, t1 = L[0][1], max(s[1] + s[2] for s in L)
        spans.append(t1 - t0)
        book_us.append(sum(s[2] for s in L if s[0] in BOOKKEEPING))
        gsum = 0.0
        for a, b in zip(L, L[1:]):
            gap = max(0.0, b[1] - (a[1] + a[2]))
            gsum += gap
            gaps.setdefault(f"{a[0]} -> {b[0]}", []).append(b[1] - (a[1] + a[2]))
        gap_us.append(gsum)
        if i + 1 < len(launches):
            between.append(launches[i + 1][0][1] - t1)
        for s in L:
            per_kernel.setdefault(s[0], []).append(s[2])
    span = float(np.mean(spans)) if spans else float("nan")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    summary = {
        "gpu": torch.cuda.get_device_name(), "nvidia_smi_name_power_limit_max_sm_clock": smi,
        "profiling_events": not args.no_events, "launches_traced": len(launches),
        "kernels_per_launch": kernels_per_launch,
        "launch_chain": [s[0] for s in launches[0]] if launches else [],
        "kernels_us": {k_: {"n": len(v), "mean": float(np.mean(v)), "total": float(np.sum(v))} for k_, v in per_kernel.items()},
        "gaps_us": {k_: {"mean": float(np.mean(v)), "median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
                    for k_, v in gaps.items()},
        "launch_span_us": span,
        "bookkeeping_kernels_us": float(np.mean(book_us)) if book_us else None,
        "gaps_inside_launch_us": float(np.mean(gap_us)) if gap_us else None,
        "gap_between_launches_us": float(np.mean(between)) if between else None,
        "share_bookkeeping": float(np.mean(book_us)) / span if spans else None,
        "share_gaps": float(np.mean(gap_us)) / span if spans else None,
        "share_bookkeeping_plus_gaps": (float(np.mean(book_us)) + float(np.mean(gap_us))) / span if spans else None,
        "note": "gaps can be negative where programmatic dependent launch overlaps a kernel with its predecessor; "
                "negative gaps count as 0 in the shares",
    }
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary, indent=1))


if __name__ == "__main__":
    main()
