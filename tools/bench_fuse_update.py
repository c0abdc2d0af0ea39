#!/usr/bin/env python3
"""Incremental global fusion (tslam_tsdf_fuse_update) against the rebuild (tslam_tsdf_fuse, fuse_from) on submap
collections of 64 and 256 submaps.  Each submap holds 2 frames (640x480, 0.05 m voxels, 3 m rays) of the box room
(tests/track_world.py) at poses of its trajectory, and is placed in the 100 m x 100 m x 20 m global map at a pose along a
path of 0.15 m and about 3 degrees per submap, as SubmapMapping places keyframe submaps.  Per case, the host clock around the call (every call synchronises),
`warmup` unrecorded calls then `steps` recorded ones (min / median / max ms), and the tslam_mesh_update that follows
each call (incremental mesh):
  * rebuild: fuse_from;
  * full: fuse_update(full=True);
  * add one: the last submap back in after a call that left it out (only the addition is timed);
  * move 1 / move 8 / move all: that many submaps alternate between two poses 5 cm apart (move all selects the
    rebuild by the cost rule).
Every case's map is checked equal, as gather() rows, to a fresh handle's full update (the rebuild: its voxel set).  Card name and power limit are
read in the same run.  One JSON line per collection size.
Usage: python tools/bench_fuse_update.py [steps] [warmup] [sizes, comma separated]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
import track_world as tw
from taichislam_b200 import synthetic as syn
from taichislam_b200.mesh_handle import MeshCache
from taichislam_b200.tsdf_handle import TsdfHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 1
sizes = [int(x) for x in sys.argv[3].split(",")] if len(sys.argv) > 3 else [64, 256]
VS, FRAMES = 0.05, 2


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q)


renders = {}


def frame(k):
    if k not in renders:
        R, t = tw.pose(k)
        renders[k] = (R, t, tw.render(R, t, seed=k))
    return renders[k]


def base_pose(s, d=0.0):
    a = 0.05 * s
    R = tw.rot([0, 1, 0], np.rad2deg(a)) @ tw.rot([1, 0, 0], 2.0 * np.sin(0.3 * s))
    return R, np.array([0.15 * s - 19.0 + d, 0.2 * np.sin(0.1 * s), 5.0 * np.sin(0.05 * s)])


def rows(h):
    i, t, w, o = h.gather(0)
    k = np.lexsort(i.T[::-1])
    return [np.ascontiguousarray(a[k]).tobytes() for a in (i, t, w, o)]


def run(n_sub):
    src = TsdfHandle(200, 200, voxel_scale=VS, K=syn.K_DEPTH, max_ray_length=3.0, max_submaps=n_sub, max_blocks=600 * n_sub)
    for s in range(n_sub):
        for f in range(FRAMES):
            R, t, d = frame((s * 7 + f * 3) % tw.N_FRAMES)
            src.integrate_depth(d, R[None], t[None], submaps=[s])
    src.sync()
    blocks = src.stats()["n_blocks"]
    voxels = sum(src.count_active(s) for s in range(n_sub))
    dst = TsdfHandle(2000, 400, voxel_scale=VS, is_global_map=True, max_submaps=n_sub, max_blocks=65536)
    poses = {s: base_pose(s) for s in range(n_sub)}
    for s, (R, T) in poses.items():
        dst.set_submap_pose(s, R, T)
    mesh = MeshCache(dst)
    cap = 1 << 22
    v = torch.empty((3 * cap, 3), dtype=torch.float32, device="cuda")
    nrm = torch.empty_like(v)

    def mesh_ms():
        t0 = time.perf_counter()
        mesh.update_into(0.1, cap, v, nrm)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    def fresh_rows():
        g = TsdfHandle(2000, 400, voxel_scale=VS, is_global_map=True, max_submaps=n_sub, max_blocks=65536)
        for s, (R, T) in poses.items():
            g.set_submap_pose(s, R, T)
        g.fuse_update(src)
        r = rows(g)
        g.close()
        return r

    out = {}

    def case(name, prepare, call):
        fuse, msh, stats = [], [], None
        for it in range(warmup + steps):
            prepare(it)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st = call(it)
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) * 1e3
            dm = mesh_ms()
            if it >= warmup:
                fuse.append(dt)
                msh.append(dm)
                stats = st
        a, b = rows(dst), fresh_rows()
        ok = a == b if name != "rebuild" else a[0] == b[0]  # fuse_from differs in the low bits: its voxel set is compared
        out[name] = dict(ms=[round(min(fuse), 3), round(float(np.median(fuse)), 3), round(max(fuse), 3)],
                         mesh_ms=[round(min(msh), 3), round(float(np.median(msh)), 3), round(max(msh), 3)], stats=stats, equal_to_fresh=ok)

    nothing = lambda it: None  # noqa: E731
    case("rebuild", nothing, lambda it: dst.fuse_from(src))
    case("full", nothing, lambda it: dst.fuse_update(src, full=True))
    inc_all = np.ones(n_sub, bool)
    inc_but_last = inc_all.copy()
    inc_but_last[-1] = False
    case("add_one", lambda it: dst.fuse_update(src, include=inc_but_last), lambda it: dst.fuse_update(src, include=inc_all))

    def mover(k):
        chosen = np.linspace(0, n_sub - 1, k).astype(int) if k < n_sub else np.arange(n_sub)

        def prep(it):
            for s in chosen:
                poses[int(s)] = base_pose(int(s), 0.05 * ((it + 1) % 2))
                dst.set_submap_pose(int(s), *poses[int(s)])
        return prep

    for k, name in ((1, "move_1"), (8, "move_8"), (n_sub, "move_all")):
        case(name, mover(k), lambda it: dst.fuse_update(src))
    res = dict(submaps=n_sub, frames_per_submap=FRAMES, src_blocks=blocks, src_voxels=int(voxels), dst_blocks=dst.stats()["n_blocks"],
               cases=out, **card())
    mesh.close()
    dst.close()
    src.close()
    return res


for n in sizes:
    print(json.dumps(run(n)), flush=True)
