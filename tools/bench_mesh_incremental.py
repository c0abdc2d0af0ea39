#!/usr/bin/env python3
"""Incremental marching cubes against the one-shot mesh on the same map: tslam_mc_generate2(step=1) and
tslam_mesh_update timed with CUDA events (warm), each update checked bit-identical to the one-shot mesh.
Cases: (a) nothing changed; (b) one more S2 frame after 100 into a 512^3 map; (c) one 32-frame launch; (d) one frame on
the several-thousand-block map of tools/bench_paths.py (sphere R = 9.5 m seen from three rings of poses); (e) the first
call (full rebuild + cache fill).  Reports ms, the four block counts (pool, stamped, touched, remeshed), triangles and
the cache's device bytes per triangle, with the card's name and power limit read in the same run.  One JSON line.
Usage: python tools/bench_mesh_incremental.py [reps]"""
import ctypes as C, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np, torch
from taichislam_b200 import _capi as capi
from taichislam_b200 import synthetic as syn
from taichislam_b200.mesh_handle import MeshCache
from taichislam_b200.tsdf_handle import TsdfHandle
from util_rot import rot_xyz

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
THRES, CAP = 0.25, 1 << 23
dev = torch.device("cuda", torch.cuda.current_device())
bufs = {k: torch.empty((3 * CAP, 3), dtype=torch.float32, device=dev) for k in ("v1", "n1", "v2", "n2")}


def events(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    r = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), r


def one_shot(g):
    n = C.c_int64(0)
    capi.check(g.L.tslam_mc_generate2(g.h, 1, THRES, CAP, capi.tptr(bufs["v1"]), capi.tptr(bufs["n1"]), None, C.byref(n), capi.stream_ptr()))
    return int(n.value)


def update(c):
    n, rc = c.update_into(THRES, CAP, bufs["v2"], bufs["n2"])
    capi.check(rc)
    return n


def same(n):
    k = 3 * n
    return bool(torch.equal(bufs["v1"][:k].view(torch.int32), bufs["v2"][:k].view(torch.int32)) and
                torch.equal(bufs["n1"][:k].view(torch.int32), bufs["n2"][:k].view(torch.int32)))


def one_shot_ms(g):
    for _ in range(2):
        one_shot(g)
    ts = [events(lambda: one_shot(g))[0] for _ in range(reps)]
    return float(np.median(ts))


def case(g, c, change, label):
    """reps x (change the map, untimed; then one timed update), then the one-shot mesh of the final state"""
    ts, st = [], []
    for r in range(reps):
        change(r)
        g.commit()
        ms, n = events(lambda: update(c))
        ts.append(ms)
        st.append(c.stats)
    ref = one_shot(g)
    ok = ref == n and same(n)
    return {"case": label, "update_ms_median": float(np.median(ts)), "update_ms": ts, "one_shot_ms": one_shot_ms(g),
            "blocks_stamped_touched_remeshed": list(st[-1]), "triangles": n, "bit_identical": ok}


res = {"reps": reps, "thres": THRES, "cases": []}
# 512^3 map, 100 S2 frames
g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
d = syn.scene_sphere(4.0)
Rs, Ts = syn.stream_poses(260)
g.integrate_depth(np.ascontiguousarray(np.broadcast_to(d, (100,) + d.shape)), Rs[:100], Ts[:100])
torch.cuda.synchronize()
free0 = torch.cuda.mem_get_info()[0]
c = MeshCache(g)
ms, n = events(lambda: update(c))
cache_bytes = free0 - torch.cuda.mem_get_info()[0]
one_shot(g)
res["cases"].append({"case": "e first call (full rebuild + cache fill), 512^3 after 100 S2 frames", "update_ms": ms, "one_shot_ms": one_shot_ms(g),
                     "blocks_stamped_touched_remeshed": list(c.stats), "triangles": n, "bit_identical": same(n),
                     "cache_bytes": int(cache_bytes), "cache_bytes_per_triangle": cache_bytes / max(n, 1)})
res["cases"].append(case(g, c, lambda r: None, "a nothing changed"))
res["cases"].append(case(g, c, lambda r: g.integrate_depth(d, Rs[100 + r][None], Ts[100 + r][None]), "b one more S2 frame after 100, 512^3"))
res["cases"].append(case(g, c, lambda r: g.integrate_depth(np.ascontiguousarray(np.broadcast_to(d, (32,) + d.shape)), Rs[110 + 32 * r % 80:110 + 32 * r % 80 + 32],
                                                           Ts[110 + 32 * r % 80:110 + 32 * r % 80 + 32]), "c one 32-frame launch, 512^3"))
c.close(); g.close()
# several-thousand-block map (tools/bench_paths.py)
gb = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True, max_blocks=20000)
d9 = syn.scene_sphere(9.5)
for ring, pitch in enumerate((-0.9, 0.0, 0.9)):
    Rr = np.stack([rot_xyz(pitch, 0.0, 2 * np.pi * k / 48) for k in range(48)])
    gb.integrate_depth(np.broadcast_to(d9, (48,) + d9.shape), Rr, np.zeros((48, 3)))
cb = MeshCache(gb)
update(cb)
res["cases"].append(case(gb, cb, lambda r: gb.integrate_depth(d9, rot_xyz(0.0, 0.0, 0.05 + 0.1 * r)[None], np.zeros((1, 3))),
                         f"d one frame on the R = 9.5 m three-ring map ({cb.stats[0]} blocks)"))
# the final device-to-device copy into the caller's arrays (verts + normals of this mesh), the most that writing them
# directly from the emit / copy kernels could save
nt = res["cases"][-1]["triangles"]
src = torch.empty((2, 3 * nt, 3), dtype=torch.float32, device=dev)
dst = torch.empty_like(src)
for _ in range(3):
    dst.copy_(src)
res["final_copy_ms_at_d"] = float(np.median([events(lambda: dst.copy_(src))[0] for _ in range(reps)]))
del src, dst
cb.close(); gb.close()
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                      str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit_max_sm_clock"] = smi
print(json.dumps(res), flush=True)
