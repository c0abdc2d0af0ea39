#!/usr/bin/env python3
"""Incremental Octomap fusion (tslam_octo_fuse_update) against the rebuild (tslam_octo_fuse, fuse_from) on collections of
64 and 256 submaps, log-odds and hit counter.  Each submap holds 2 scene_room frames (640x480 at step 2, 0.05 m voxels,
5 m rays) at small pose offsets, and is placed in a 51 m x 51 m x 12.8 m global map along a path of 0.15 m and about
3 degrees per submap.  Per case, the host clock around the call (every call synchronises), `warmup` unrecorded calls
then `steps` recorded ones (min / median / max ms):
  * rebuild: fuse_from;   * full: fuse_update(full=True);
  * add one: the last submap back in after a call that left it out (only the addition is timed);
  * move 1 / move 8: that many submaps alternate between two poses 5 cm apart;
  * log-odds only: esdf_update (D = 1 m) and frontier_update of the global map after moving one submap, incremental
    against full (alternated).
Every case's map is checked equal, as sorted gather rows, to a rebuild at the same poses.  Card name and power limit
are read in the same run.  One JSON line per (model, size).
Usage: python tools/bench_octo_fuse_update.py [steps] [warmup] [sizes, comma separated]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.octo_handle import OctoHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 1
sizes = [int(x) for x in sys.argv[3].split(",")] if len(sys.argv) > 3 else [64, 256]
VS, FRAMES, N, NZ = 0.05, 2, 1024, 256
LO = dict(l_hit=868, l_miss=-415, l_min=-2048, l_max=3595, l_occ=0)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q)


def rot_z(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def base_pose(s, d=0.0):
    return rot_z(0.05 * s), np.array([0.15 * s - 19.0 + d, 0.2 * np.sin(0.1 * s), 0.3 * np.sin(0.05 * s)])


def handle(model, n_sub, max_blocks):
    return OctoHandle(N, NZ, K=2, voxel_scale=VS, min_occupy_thres=1, max_ray_length=5.0, Kcam=syn.K_DEPTH, max_submaps=n_sub,
                      max_blocks=max_blocks, logodds=LO if model == "logodds" else None)


def rows(h):
    r = h.gather(0)
    k = np.lexsort(r[0].T[::-1])
    return [np.ascontiguousarray(a[k]).tobytes() for a in r]


def timed(fn, prep=None):
    ts = []
    for q in range(warmup + steps):
        if prep:
            prep(q)
        torch.cuda.synchronize()
        t = time.perf_counter()
        out = fn(q)
        torch.cuda.synchronize()
        if q >= warmup:
            ts.append((time.perf_counter() - t) * 1e3)
    return dict(min=round(min(ts), 3), median=round(float(np.median(ts)), 3), max=round(max(ts), 3)), out


def run(model, n_sub, depth):
    src = handle(model, n_sub, 2500 * n_sub)
    rng = np.random.default_rng(n_sub)
    for s in range(n_sub):
        for f in range(FRAMES):
            a = rng.uniform(-0.4, 0.4, 3)
            src.integrate_depth(depth, rot_z(a[0]), np.array([a[1], a[2], 0.0]) * 0.5, submap=s)
    src.sync()
    dst = handle(model, n_sub, 1 << 19)
    poses = {s: base_pose(s) for s in range(n_sub)}
    for s, (R, T) in poses.items():
        dst.set_submap_pose(s, R, T)
    out = dict(model=model, submaps=n_sub, frames_per_submap=FRAMES, src_known_voxels=int(sum(src.gather(s)[0].shape[0] for s in range(n_sub))))

    def check(name):
        reb = handle(model, n_sub, 1 << 19)
        for s, (R, T) in poses.items():
            reb.set_submap_pose(s, R, T)
        reb.fuse_from(src)
        out.setdefault("checked_equal_to_rebuild", {})[name] = rows(dst) == rows(reb)

    reb = handle(model, n_sub, 1 << 19)
    for s, (R, T) in poses.items():
        reb.set_submap_pose(s, R, T)
    out["rebuild_ms"], _ = timed(lambda q: reb.fuse_from(src))
    out["global_voxels"] = int(reb.gather(0)[0].shape[0])
    del reb
    out["full_ms"], st = timed(lambda q: dst.fuse_update(src, full=True))
    check("full")
    inc_all = np.ones(n_sub, bool)
    inc_wo = inc_all.copy()
    inc_wo[-1] = False
    out["add_one_ms"], st = timed(lambda q: dst.fuse_update(src, include=inc_all), prep=lambda q: dst.fuse_update(src, include=inc_wo))
    out["add_one_stats"] = st
    check("add_one")

    def mover(k):
        sel = np.linspace(0, n_sub - 1, k).astype(int)

        def prep(q):
            for s in sel:
                poses[s] = base_pose(s, 0.05 * ((q + 1) % 2))
                dst.set_submap_pose(s, *poses[s])
        return prep
    for k in (1, 8):
        out[f"move_{k}_ms"], st = timed(lambda q: dst.fuse_update(src), prep=mover(k))
        out[f"move_{k}_stats"] = st
        check(f"move_{k}")
    if model == "logodds":
        dst.esdf_update(0, max_dist=1.0)
        dst.frontier_update(0)
        prep = mover(1)
        for name, fn in (("esdf", lambda full: dst.esdf_update(0, max_dist=1.0, full=full)),
                         ("frontier", lambda full: dst.frontier_update(0, full=full))):
            ti, tf = [], []
            for q in range(warmup + steps):
                for full, acc in ((False, ti), (True, tf)):
                    prep(2 * q + int(full))
                    dst.fuse_update(src)
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    fn(full)
                    torch.cuda.synchronize()
                    if q >= warmup:
                        acc.append((time.perf_counter() - t) * 1e3)
            out[f"{name}_after_move_1_ms"] = dict(incremental=round(float(np.median(ti)), 3), full=round(float(np.median(tf)), 3),
                                                  incremental_min_max=[round(min(ti), 3), round(max(ti), 3)],
                                                  full_min_max=[round(min(tf), 3), round(max(tf), 3)])
    return out


def main():
    torch.cuda.init()
    info = card()
    depth = syn.scene_room()
    for model in ("logodds", "hits"):
        for n in sizes:
            r = run(model, n, depth)
            r.update(info, steps=steps, warmup=warmup)
            print(json.dumps(r), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
