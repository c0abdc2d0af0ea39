#!/usr/bin/env python3
"""Loop detection between TSDF submaps (tslam_tsdf_place_describe, tslam_place_match, DenseTSDF.detect_loops) on a
collection of 256 submaps like tools/bench_fuse_update.py's: 2 frames (640x480, 0.05 m voxels, 3 m rays) of the box room
(tests/track_world.py) each, at base poses along a path of 0.15 m and about 3 degrees per submap.  Cases:
  * describe 256: every submap once; describe 1024: the 256 submaps four times over (a submap may be listed again);
  * match 1 x 255: the newest submap against the others; match 256 x 256: every submap against all;
  * verify: tslam_tsdf_register of the 1 x 255 shortlist (top_k = 8) from the coarse poses;
  * detect_loops: DenseTSDF.detect_loops end to end for the newest submap (describe, match, register).
Each figure is the median over `windows` windows of `steps` calls (host clock around calls that end in a device
synchronise), after `warmup` unrecorded calls of the same case; min and max of the windows too.  With --profile, a separate
run records one call of each case under torch.profiler and reports the kernels' CUDA times.  Card name and power limit are
read in the same run.  One JSON line.
Usage: python tools/bench_place.py [steps] [warmup] [windows] [--profile]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
import track_world as tw
from taichislam_b200 import place
from taichislam_b200 import synthetic as syn
from taichislam_b200.mapping.dense_tsdf import DenseTSDF

args = [a for a in sys.argv[1:] if not a.startswith("--")]
steps = int(args[0]) if len(args) > 0 else 5
warmup = int(args[1]) if len(args) > 1 else 2
windows = int(args[2]) if len(args) > 2 else 5
profile = "--profile" in sys.argv
VS, FRAMES, N_SUB = 0.05, 2, 256
UP = (0.0, -1.0, 0.0)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q)


def base_pose(s):
    a = 0.05 * s
    R = tw.rot([0, 1, 0], np.rad2deg(a)) @ tw.rot([1, 0, 0], 2.0 * np.sin(0.3 * s))
    return R, np.array([0.15 * s - 19.0, 0.2 * np.sin(0.1 * s), 5.0 * np.sin(0.05 * s)])


def build():
    dm = DenseTSDF(map_scale=[10.0, 10.0], voxel_scale=VS, max_ray_length=3.0, max_submap_num=N_SUB, max_blocks=600 * N_SUB,
                   max_disp_particles=1 << 16)
    dm.set_dep_camera_intrinsic(syn.K_DEPTH)
    renders = {}
    for s in range(N_SUB):
        if s:
            dm.switch_to_next_submap()
        Rb, tb = base_pose(s)
        dm.set_base_pose_submap(s, Rb, tb)
        for f in range(FRAMES):
            k = (s * 7 + f * 3) % tw.N_FRAMES
            if k not in renders:
                R, t = tw.pose(k)
                renders[k] = (R, t, tw.render(R, t, seed=k))
            R, t, d = renders[k]
            dm.recast_depth_to_map(Rb @ R, Rb @ t + tb, d, np.array([]))  # the frame at pose k of the submap's local frame
    dm.finalization_current_submap()
    return dm


def timed(fn):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(windows):
        t = time.perf_counter()
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t) * 1000.0 / steps)
    return dict(median_ms=float(np.median(out)), min_ms=float(min(out)), max_ms=float(max(out)))


def main():
    dm = build()
    h = dm._h
    S = list(range(N_SUB))
    L = place.level(UP)
    M = np.stack([L @ dm.base_pose(s)[0] for s in S])
    band = 4 * VS
    desc = h.place_describe(S, M, 8.0, 0.3, band)
    ids = np.arange(N_SUB, dtype=np.int64)
    q_last = [N_SUB - 1]
    mt = place.match(desc["sc"], desc["ring"], desc["bev"], desc["n_points"], ids, q_last, top_k=8, min_gap=2, min_points=200)
    pairs = [(N_SUB - 1, int(d), k) for k, d in enumerate(mt["match"][0]) if d >= 0]
    R0 = np.stack([place.coarse_pose(M[q], M[d], mt["yaw_deg"][0, k], mt["dx"][0, k], mt["dy"][0, k], 8.0)[0] for q, d, k in pairs])
    T0 = np.stack([place.coarse_pose(M[q], M[d], mt["yaw_deg"][0, k], mt["dx"][0, k], mt["dy"][0, k], 8.0)[1] for q, d, k in pairs])
    S4 = S * 4
    M4 = np.concatenate([M] * 4)
    cases = {
        "describe_256": lambda: h.place_describe(S, M, 8.0, 0.3, band),
        "describe_1024": lambda: h.place_describe(S4, M4, 8.0, 0.3, band),
        "match_1x255": lambda: place.match(desc["sc"], desc["ring"], desc["bev"], desc["n_points"], ids, q_last, top_k=8, min_gap=2),
        "match_256x256": lambda: place.match(desc["sc"], desc["ring"], desc["bev"], desc["n_points"], ids, S, top_k=8, min_gap=2),
        "verify_1x255_shortlist": lambda: h.register(h, [p[0] for p in pairs], [p[1] for p in pairs], R0, T0, band, max_iters=100,
                                                     min_points=200),
        "detect_loops_newest_of_256": lambda: dm.detect_loops(q_last, up=UP, min_gap=2),
    }
    res = dict(card=card(), n_submaps=N_SUB, points=int(desc["n_points"].sum()), verified_pairs=len(pairs), steps=steps,
               warmup=warmup, windows=windows)
    res["cases"] = {k: timed(f) for k, f in cases.items()}
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof
        kern = {}
        for k, f in cases.items():
            f()
            torch.cuda.synchronize()
            with prof(activities=[ProfilerActivity.CUDA]) as p:
                f()
                torch.cuda.synchronize()
            kern[k] = {e.key: round(e.device_time_total / 1000.0, 4) for e in p.key_averages() if e.device_time_total > 0}
        res["kernel_ms_profiled"] = kern
    print(json.dumps(res))


if __name__ == "__main__":
    main()
