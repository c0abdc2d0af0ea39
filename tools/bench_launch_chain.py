#!/usr/bin/env python3
"""The bench's flagship launches with profiling OFF: what the launch chain itself costs, apart from the kernel stamps.

Runs the device-resident arm of bench.py - a 512^3 map, the S2 stream, 64-frame depth launches with commit, three
warm-up steps of 16 launches - but never switches profiling on, then times `--steps` steps of 16 launches (1600
launches by default) between two CUDA events, `--repeats` times on the same map.  Prints one JSON line: frames/s and
ms per launch of every repeat, the card's name, power limit and max SM clock read in the same run (DESIGN §5).

Usage: python tools/bench_launch_chain.py [--steps 100] [--warmup 3] [--repeats 3]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH, LAUNCHES_PER_STEP, POOL_BATCHES = 64, 16, 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from taichislam_b200 import synthetic as syn
    from taichislam_b200.tsdf_handle import TsdfHandle

    torch.cuda.set_device(0)
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    pool = []
    for b in range(POOL_BATCHES):
        d, _, _ = bench.make_inputs(BATCH, b * BATCH)
        pool.append(torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda())
    n_launches = (args.warmup + args.steps * args.repeats) * LAUNCHES_PER_STEP
    Rs, Ts = syn.stream_poses(n_launches * BATCH, start=0)
    Rs = np.ascontiguousarray(Rs.astype(np.float32).reshape(n_launches, BATCH, 9))
    Ts = np.ascontiguousarray(Ts.astype(np.float32).reshape(n_launches, BATCH, 3))
    k = 0

    def steps(n):
        nonlocal k
        for _ in range(n * LAUNCHES_PER_STEP):
            g.integrate_depth(pool[k % POOL_BATCHES], Rs[k], Ts[k], commit=True)
            k += 1

    steps(args.warmup)
    runs = []
    for _ in range(args.repeats):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        steps(args.steps)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        runs.append({"frames_per_s": args.steps * LAUNCHES_PER_STEP * BATCH / (ms * 1e-3),
                     "ms_per_launch": ms / (args.steps * LAUNCHES_PER_STEP)})
    g.sync()
    st = g.stats()
    g.close()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"profiling": False, "launches_per_repeat": args.steps * LAUNCHES_PER_STEP, "runs": runs,
                      "err_flags": st["err_flags"], "gpu": torch.cuda.get_device_name(),
                      "nvidia_smi_name_power_limit_max_sm_clock": smi}))


if __name__ == "__main__":
    main()
