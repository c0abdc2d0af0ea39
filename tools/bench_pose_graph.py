#!/usr/bin/env python3
"""Submap pose-graph optimisation (tslam_pose_graph_solve, pose_graph.optimize) on the seeded random-walk graphs of
tests/pose_graph_reference.py (odometry chain, a loop every 4 nodes to a node 2-24 steps back, 10 % false loops, 20 %
rank-3 loops) at 64, 256, 1024 and 4096 nodes, eps_t = 1e-8, eps_r = 1e-10.  Per size: the GPU solve end to end (host
clock around the call, which ends in a device synchronise; median, min and max over `windows` windows of `steps` calls
after `warmup` calls), LM evaluations, CG iterations per evaluation, and the numpy / scipy reference's host solve
(exact sparse LM steps) timed in the same run.  Then the loop-world flow of tests/test_gpu_pose_graph_mapping.py:
detect_loops for every submap, optimize_poses and the incremental fusion update it triggers, end to end.  With
--profile, a separate run records one solve per size under torch.profiler and reports the kernels' CUDA times.  Card name
and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_pose_graph.py [steps] [warmup] [windows] [--profile]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
import pose_graph_reference as P
from taichislam_b200 import pose_graph

args = [a for a in sys.argv[1:] if not a.startswith("--")]
steps = int(args[0]) if len(args) > 0 else 3
warmup = int(args[1]) if len(args) > 1 else 1
windows = int(args[2]) if len(args) > 2 else 3
profile = "--profile" in sys.argv
SIZES = (64, 256, 1024, 4096)
OPTS = dict(eps_t=1e-8, eps_r=1e-10)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q)


def timed(fn):
    for _ in range(warmup):
        fn()
    ws = []
    for _ in range(windows):
        t = time.perf_counter()
        for _ in range(steps):
            fn()
        ws.append((time.perf_counter() - t) * 1e3 / steps)
    return dict(median_ms=float(np.median(ws)), min_ms=float(min(ws)), max_ms=float(max(ws)))


def main():
    assert torch.cuda.is_available(), "bench_pose_graph needs a GPU"
    out = dict(card=card(), steps=steps, warmup=warmup, windows=windows, sizes={})
    for n in SIZES:
        R0, T0, fx, ed, *_ = P.random_walk_graph(n, seed=n)
        g = pose_graph.optimize(R0, T0, fx, ed, **OPTS)
        t = time.perf_counter()
        r = P.solve_edges(R0, T0, fx, ed, **OPTS)
        ref_ms = (time.perf_counter() - t) * 1e3
        row = dict(nodes=n, edges=int(len(ed["ij"])), gpu=timed(lambda: pose_graph.optimize(R0, T0, fx, ed, **OPTS)),
                   gpu_status=g["status_name"], gpu_evaluations=g["evaluations"], gpu_accepted=g["accepted"],
                   cg_iterations=g["cg_iterations"], cg_per_evaluation=g["cg_iterations"] / max(g["evaluations"], 1),
                   cg_residual=g["cg_residual"], reference_host_ms=ref_ms, reference_evaluations=r["evaluations"],
                   reference_status=int(r["status"]), max_dT_vs_reference=float(np.abs(g["T"] - r["T"]).max()))
        out["sizes"][n] = row
        print(json.dumps(row), file=sys.stderr)
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        kt = {}
        for n in SIZES:
            R0, T0, fx, ed, *_ = P.random_walk_graph(n, seed=n)
            with prof(activities=[ProfilerActivity.CUDA]) as p:
                pose_graph.optimize(R0, T0, fx, ed, **OPTS)
            ev = {}
            for e in p.key_averages():
                if e.device_type.name == "CUDA" or "k_pg" in e.key:
                    ev[e.key[:60]] = dict(count=e.count, total_ms=e.device_time_total / 1e3)
            kt[n] = ev
        out["kernels"] = kt
    else:
        import test_gpu_pose_graph_mapping as M
        sm, _ = M.run_loop_world()
        torch.cuda.synchronize()
        t = time.perf_counter()
        loops = {}
        for f in sorted(sm.submaps):
            loops.update(sm.detect_loops(f, min_gap=2))
        t1 = time.perf_counter()
        res = sm.optimize_poses(loops)  # includes the incremental fusion update of set_frame_poses
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        out["loop_world"] = dict(detect_ms=(t1 - t) * 1e3, optimise_and_fuse_ms=(t2 - t1) * 1e3, loops=len(loops),
                                 status=res["info"]["status_name"], evaluations=res["info"]["evaluations"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
