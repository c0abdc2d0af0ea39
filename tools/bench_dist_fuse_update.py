#!/usr/bin/env python3
"""Incremental fusion of the tiled global map (TiledGlobalMap.update_fused_submaps' phases, driven for a LocalGroup by
run_local_update_fused_submaps) against the tiled rebuild (run_local_fusion), at world 4 on ONE GPU.  The submaps are
those of tools/bench_fuse_update.py: 2 box-room frames each (640x480, 0.05 m voxels, 3 m rays), placed along a path of
0.15 m and about 3 degrees per submap in a 100 m x 100 m x 20 m map; submap s belongs to rank s % 4, so neighbouring
submaps live on different ranks and the path crosses the tile seams.  The four virtual ranks run one after another in
this process, so a time is the sum of every rank's work plus the host-side routing, not the time of four GPUs.
Per case, the host clock around the synchronised call, `warmup` unrecorded calls then `steps` recorded ones (min /
median / max ms), with the blocks and bytes routed to the owners:
  * rebuild: run_local_fusion (float sums, every submap splatted, all-to-all, commit);
  * full: run_local_update_fused_submaps(full=True);
  * add one: the last submap back in after a call that left it out (only the addition is timed);
  * move 1 / move 8: that many submaps alternate between two poses 5 cm apart.
After the cases the union of the tiles is checked, as gather() rows, against one map's tslam_tsdf_fuse_update of all
submaps.  Card name and power limit are read in the same run.  One JSON line per collection size.
Usage: python tools/bench_dist_fuse_update.py [steps] [warmup] [sizes, comma separated]"""
import json, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
import track_world as tw
from taichislam_b200 import synthetic as syn
from taichislam_b200.distributed import LocalGroup, TiledGlobalMap, run_local_fusion, run_local_update_fused_submaps
from taichislam_b200.tsdf_handle import TsdfHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 1
sizes = [int(x) for x in sys.argv[3].split(",")] if len(sys.argv) > 3 else [64, 256]
VS, FRAMES, WORLD = 0.05, 2, 4


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q)


class Map:
    """What TiledGlobalMap and the fusion phases read of a DenseTSDF, over a bare TsdfHandle."""

    def __init__(self, h):
        self._h, self.enable_texture = h, False

    def _flush(self):
        pass


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


def rows(parts):
    i, t, w, o = (np.concatenate([p[c] for p in parts]) for c in range(4))
    k = np.lexsort(i.T[::-1])
    return [np.ascontiguousarray(a[k]).tobytes() for a in (i, t, w, o)]


def run(n_sub):
    per_rank = (n_sub + WORLD - 1) // WORLD
    subs = [Map(TsdfHandle(200, 200, voxel_scale=VS, K=syn.K_DEPTH, max_ray_length=3.0, max_submaps=n_sub, max_blocks=600 * per_rank + 1024))
            for _ in range(WORLD)]
    for s in range(n_sub):
        for f in range(FRAMES):
            R, t, d = frame((s * 7 + f * 3) % tw.N_FRAMES)
            subs[s % WORLD]._h.integrate_depth(d, R[None], t[None], submaps=[s])
    for m in subs:
        m._h.sync()
    grp = LocalGroup(WORLD)
    glos = [Map(TsdfHandle(2000, 400, voxel_scale=VS, is_global_map=True, max_submaps=n_sub, max_blocks=32768)) for _ in range(WORLD)]
    tiled = [TiledGlobalMap(g, grp, r, WORLD) for r, g in enumerate(glos)]
    poses = {s: base_pose(s) for s in range(n_sub)}

    def set_poses(ss):
        for s in ss:
            for g in glos:
                g._h.set_submap_pose(s, *poses[s])

    set_poses(range(n_sub))
    out = {}

    def case(name, prepare, call):
        ms, stats = [], None
        for it in range(warmup + steps):
            prepare(it)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st = call()
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) * 1e3
            if it >= warmup:
                ms.append(dt)
                stats = st
        if stats is None:  # the rebuild reports its exchange per rank
            stats = dict(foreign_blocks_sent=sum(t.last_exchange["fusion_blocks_sent"] for t in tiled),
                         bytes_sent=sum(t.last_exchange["fusion_bytes_sent"] for t in tiled))
        out[name] = dict(ms=[round(min(ms), 3), round(float(np.median(ms)), 3), round(max(ms), 3)], stats=stats)

    nothing = lambda it: None  # noqa: E731
    case("rebuild", nothing, lambda: run_local_fusion(tiled, subs))
    case("full", nothing, lambda: run_local_update_fused_submaps(tiled, subs, full=True))
    inc_all = np.ones(n_sub, bool)
    inc_but_last = inc_all.copy()
    inc_but_last[-1] = False
    case("add_one", lambda it: run_local_update_fused_submaps(tiled, subs, include=inc_but_last),
         lambda: run_local_update_fused_submaps(tiled, subs, include=inc_all))

    def mover(k):
        chosen = [int(s) for s in np.linspace(0, n_sub - 1, k).astype(int)]

        def prep(it):
            for s in chosen:
                poses[s] = base_pose(s, 0.05 * ((it + 1) % 2))
            set_poses(chosen)
        return prep

    for k, name in ((1, "move_1"), (8, "move_8")):
        case(name, mover(k), lambda: run_local_update_fused_submaps(tiled, subs))
    # the union of the tiles against one map's update of all submaps
    one_src = TsdfHandle(200, 200, voxel_scale=VS, K=syn.K_DEPTH, max_ray_length=3.0, max_submaps=n_sub, max_blocks=600 * n_sub)
    for s in range(n_sub):
        one_src.scatter(s, *subs[s % WORLD]._h.gather(s))
    one = TsdfHandle(2000, 400, voxel_scale=VS, is_global_map=True, max_submaps=n_sub, max_blocks=65536)
    for s, (R, T) in poses.items():
        one.set_submap_pose(s, R, T)
    one.fuse_update(one_src)
    equal = rows([g._h.gather(0) for g in glos]) == rows([one.gather(0)])
    res = dict(submaps=n_sub, world=WORLD, frames_per_submap=FRAMES, tiles=list(tiled[0].tiles), blocks_per_rank=[g._h.stats()["n_blocks"] for g in glos],
               single_map_blocks=one.stats()["n_blocks"], equal_to_single_map=equal, cases=out, **card())
    for h in [one, one_src] + [m._h for m in subs + glos]:
        h.close()
    return res


for n in sizes:
    print(json.dumps(run(n)), flush=True)
