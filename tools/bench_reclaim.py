#!/usr/bin/env python3
"""Reclaim of TSDF pool blocks (tslam_tsdf_reclaim, DESIGN.md section 7, "Reclaiming pool blocks").

(a) 256 box-room submaps (tests/track_world.py, 2 frames of 640x480 each, 0.05 m voxels, 3 m rays), placed along a path
    as in tools/bench_fuse_update.py, fused into an incremental global map.  32 updates each move 8 submaps by a
    loop-closure-sized correction (0.2 .. 0.5 m and 1 .. 3 degrees, a new one every update).  One global map reclaims its
    empty blocks after every update (what SubmapMapping(reclaim_empty=True) does), a second one does not: global
    n_blocks of both after every update, the reclaim's time after each update (host clock around the synchronising
    call), and the end-to-end time of a reclaim that drops nothing (median of 5 after 2 warm-up calls).  Both maps are
    checked equal on their observed voxels at the end.
(b) A 512^3 map (0.05 m voxels) after 1024 frames of the bench.py stream, then OUTSIDE at R m around the last pose:
    the time of that call, the blocks before / after, and a repeat that drops nothing (median of 5).
With --profile, one more run of (a) and (b) under torch.profiler (CUDA activities) gives the kernel times of
k_rc_classify / k_rc_move / k_rc_rebuild; the move kernel's achieved bytes/s is (moved blocks x bytes per block x 2,
read + write) over its kernel time, against the 3.35 TB/s HBM3 data-sheet figure of the H100 SXM.
Card name and power limit are read in the same run.  One JSON line per part.
Usage: python tools/bench_reclaim.py [--profile] [--updates 32] [--radius 3.0]"""
import argparse, json, os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import track_world as tw
from taichislam_b200 import synthetic as syn
from taichislam_b200.tsdf_handle import TsdfHandle

VS, FRAMES, N_SUB, N_MOVE = 0.05, 2, 256, 8
HBM_PEAK = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q)


def block_bytes(h, sums):
    """bytes of one pool block's planes that the move copies: acc tw obs occ (+ esdf, texture) + fusion sums"""
    b = 4096 * (8 + 8 + 1 + 1)
    if h.texture_enabled:
        b += 4096 * (8 + 16)
    if sums:
        b += 4096 * 8 * (6 if h.texture_enabled else 3)
    return b


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t0) * 1e3


def base_pose(s, d=np.zeros(3), yaw=0.0):
    a = 0.05 * s
    R = tw.rot([0, 1, 0], np.rad2deg(a) + yaw) @ tw.rot([1, 0, 0], 2.0 * np.sin(0.3 * s))
    return R, np.array([0.15 * s - 19.0, 0.2 * np.sin(0.1 * s), 5.0 * np.sin(0.05 * s)]) + d


def part_a(updates):
    src = TsdfHandle(200, 200, voxel_scale=VS, K=syn.K_DEPTH, max_ray_length=3.0, max_submaps=N_SUB, max_blocks=600 * N_SUB)
    for s in range(N_SUB):
        for f in range(FRAMES):
            R, t = tw.pose((s * 7 + f * 3) % tw.N_FRAMES)
            src.integrate_depth(tw.render(R, t, seed=(s * 7 + f * 3) % tw.N_FRAMES), R[None], t[None], submaps=[s])
    src.sync()
    maps = [TsdfHandle(2000, 400, voxel_scale=VS, is_global_map=True, max_submaps=N_SUB, max_blocks=1 << 17) for _ in range(2)]
    rng = np.random.default_rng(5)
    poses = {s: base_pose(s) for s in range(N_SUB)}
    for g in maps:
        for s, (R, T) in poses.items():
            g.set_submap_pose(s, R, T)
        g.fuse_update(src)
    nb0 = maps[0].stats()["n_blocks"]
    rec_ms, rec_stats, blocks = [], [], []
    for it in range(updates):
        for s in rng.choice(N_SUB, N_MOVE, replace=False):
            d = rng.normal(size=3)
            d *= rng.uniform(0.2, 0.5) / np.linalg.norm(d)
            poses[int(s)] = base_pose(int(s), d, float(rng.uniform(1.0, 3.0) * rng.choice([-1, 1])))
        for g in maps:
            for s, (R, T) in poses.items():
                g.set_submap_pose(s, R, T)
            st = g.fuse_update(src)
            assert not st["full"], st
        st, ms = timed(lambda: maps[0].reclaim(empty=True))
        rec_ms.append(ms)
        rec_stats.append(st)
        blocks.append([maps[0].stats()["n_blocks"], maps[1].stats()["n_blocks"]])
    idle = []
    for i in range(7):
        st, ms = timed(lambda: maps[0].reclaim(empty=True))
        assert st["dropped"] == 0
        if i >= 2:
            idle.append(ms)
    a, b = (as_rows(g) for g in maps)
    out = dict(part="a", submaps=N_SUB, updates=updates, moved_per_update=N_MOVE, blocks_after_first_fusion=nb0,
               blocks_with_reclaim=[x[0] for x in blocks], blocks_without_reclaim=[x[1] for x in blocks],
               reclaim_ms_dropping=dict(min=round(min(rec_ms[1:]), 3), median=round(float(np.median(rec_ms[1:])), 3), max=round(max(rec_ms[1:]), 3),
                                        first=round(rec_ms[0], 3)),
               dropped_per_update=[s["dropped"] for s in rec_stats], moved_blocks_per_update=[s["moved"] for s in rec_stats],
               reclaim_ms_nothing_dropped_median5=round(float(np.median(idle)), 3),
               block_bytes=block_bytes(maps[0], True), equal_observed_voxels=a == b, **card())
    for g in maps:
        g.close()
    src.close()
    return out


def as_rows(h):
    i, t, w, o = h.gather(0)
    k = np.lexsort(i.T[::-1])
    return [np.ascontiguousarray(x[k]).tobytes() for x in (i, t, w, o)]


def stream_depth(t):
    k = ((t % 256) * 7) % 11
    return syn.scene_sphere(4.0 + 0.04 * (k - 5))


def part_b(radius, n_frames=1024):
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    Rs, Ts = syn.stream_poses(n_frames, start=0)
    for b in range(0, n_frames, 64):
        d = np.stack([stream_depth(t) for t in range(b, b + 64)])
        g.integrate_depth(d, Rs[b:b + 64], Ts[b:b + 64], commit=True)
    g.sync()
    centre = np.asarray(Ts[-1], np.float64)
    st, ms = timed(lambda: g.reclaim(center=centre, radius=radius))
    idle = []
    for i in range(7):
        s2, m2 = timed(lambda: g.reclaim(center=centre, radius=radius))
        assert s2["dropped"] == 0
        if i >= 2:
            idle.append(m2)
    out = dict(part="b", grid="512^3", frames=n_frames, radius_m=radius, stats=st, reclaim_ms=round(ms, 3),
               reclaim_ms_nothing_dropped_median5=round(float(np.median(idle)), 3), block_bytes=block_bytes(g, False), **card())
    g.close()
    return out


def warm():
    """load the reclaim kernels and CUB once, on a small map"""
    h = TsdfHandle(128, 128, voxel_scale=VS, K=syn.K_DEPTH, max_ray_length=3.0, max_submaps=2, max_blocks=4096)
    R, t = tw.pose(0)
    h.integrate_depth(tw.render(R, t, seed=0), R[None], t[None], submaps=[0])
    h.reclaim(center=t, radius=1.0)
    h.close()


def profile(args, outdir):
    from torch.profiler import ProfilerActivity, profile as tprof
    with tprof(activities=[ProfilerActivity.CUDA]) as p:
        ra = part_a(min(args.updates, 8))
        rb = part_b(args.radius)
    kern = {}
    for e in p.key_averages():
        if "k_rc_" in e.key:
            kern[e.key] = dict(calls=e.count, total_ms=round(e.device_time_total / 1e3, 4))
    move_ms = sum(v["total_ms"] for k, v in kern.items() if k.startswith("k_rc_move("))
    moved = sum(ra["moved_blocks_per_update"]) * ra["block_bytes"] + rb["stats"]["moved"] * rb["block_bytes"]
    res = dict(part="profile", kernels=kern, move_kernel_ms=round(move_ms, 4), move_bytes=2 * moved,
               move_bytes_per_s=(2 * moved / (move_ms / 1e3)) if move_ms > 0 else None, hbm_datasheet_bytes_per_s=HBM_PEAK, **card())
    if res["move_bytes_per_s"]:
        res["share_of_datasheet"] = round(res["move_bytes_per_s"] / HBM_PEAK, 3)
    os.makedirs(outdir, exist_ok=True)
    p.export_chrome_trace(os.path.join(outdir, "bench_reclaim_trace.json"))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--updates", type=int, default=32)
    ap.add_argument("--radius", type=float, default=3.0)
    ap.add_argument("--out", default=tempfile.gettempdir(), help="directory of the --profile trace")
    args = ap.parse_args()
    warm()
    if args.profile:
        print(json.dumps(profile(args, args.out)), flush=True)
        return
    print(json.dumps(part_a(args.updates)), flush=True)
    print(json.dumps(part_b(args.radius)), flush=True)


if __name__ == "__main__":
    main()
