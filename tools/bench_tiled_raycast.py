#!/usr/bin/env python3
"""Cost of the per-sample owner test of the tiled raycast on one GPU: 100 frames of the S2 stream into a 512^3 map, then
the same 2^20 rays (origins in observed free space, uniform directions, 4 m) marched by tslam_tsdf_raycast and by
tslam_tsdf_raycast_tiled at world 1 (one tile: nothing is handed over, so both march every ray to its end), each
timed with CUDA events over many batches after warm-up.  The two answers are checked to be bit-identical.  Prints one
JSON line with the times, the mean samples per ray, the card's name and its power limit read in the same run.
Usage: python tools/bench_tiled_raycast.py [reps]"""
import ctypes as C, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import _capi as capi
from taichislam_b200 import synthetic as syn
from taichislam_b200.tsdf_handle import TsdfHandle

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 200
n = 1 << 20
vs, max_dist = 0.05, 4.0

g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
d = syn.scene_sphere(4.0)
Rs, Ts = syn.stream_poses(100)
g.integrate_depth(np.ascontiguousarray(np.broadcast_to(d, (100,) + d.shape)), Rs, Ts)
idx, t, _, _ = g.gather()
free = idx[t >= np.float32(1.8 * vs)]
rng = np.random.default_rng(0)
pos = ((free[rng.integers(0, free.shape[0], n)] + rng.uniform(-0.45, 0.45, size=(n, 3))) * vs).astype(np.float32)
dirs = rng.normal(size=(n, 3)).astype(np.float32)
dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)

L, h, st = g.L, g.h, capi.stream_ptr()
p, dr = torch.from_numpy(pos).cuda(), torch.from_numpy(dirs).cuda()
rays = torch.zeros((n, 8), dtype=torch.float32, device="cuda")
rays[:, :3], rays[:, 3:6], rays[:, 6] = p, dr, max_dist
tiles = (C.c_int32 * 3)(1, 1, 1)
out = {}
for name in ("plain", "tiled"):
    hit = torch.empty(n, dtype=torch.uint8, device="cuda")
    xyz = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    ln = torch.empty(n, dtype=torch.float32, device="cuda")
    dest = torch.empty(n, dtype=torch.int32, device="cuda")
    if name == "plain":
        def call():
            capi.check(L.tslam_tsdf_raycast(h, 0, n, capi.tptr(p), capi.tptr(dr), max_dist, capi.tptr(hit), capi.tptr(xyz), capi.tptr(ln), st))
    else:
        def call():
            capi.check(L.tslam_tsdf_raycast_tiled(h, tiles, 0, 1, 0, n, capi.tptr(rays), capi.tptr(dest), capi.tptr(hit), capi.tptr(xyz),
                                                  capi.tptr(ln), st))
    for _ in range(10):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    out[name] = {"ms_per_batch": ms, "rays_per_s": n / (ms * 1e-3)}
    out[name + "_answer"] = (hit.cpu().numpy(), xyz.cpu().numpy().view(np.uint32), ln.cpu().numpy().view(np.uint32))
    if name == "tiled":
        assert int((dest >= 0).sum()) == 0, "a ray was handed over at world 1"
a, b = out.pop("plain_answer"), out.pop("tiled_answer")
assert all(np.array_equal(x, y) for x, y in zip(a, b)), "tiled answers differ from the plain raycast"
lens = b[2].view(np.float32)
res = {"map": "512^3, 100 S2-stream frames", "rays": n, "max_dist_m": max_dist, "reps": reps,
       "mean_samples_per_ray": float(np.mean(np.floor(lens / vs + 0.5) + 1)), "hit_frac": float(a[0].mean()),
       "plain": out["plain"], "tiled_world1": out["tiled"], "tiled_over_plain": out["tiled"]["ms_per_batch"] / out["plain"]["ms_per_batch"]}
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                      str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit_max_sm_clock"] = smi
print(json.dumps(res), flush=True)
g.close()
