#!/usr/bin/env python3
"""Log-odds Octomap against the hit counter on the same frames: depth frames streamed into a 512^3 Octomap
(map_scale 25.6 m, 0.05 m voxels, max_ray_length = 5 m, recast_step 2), both modes in one run, CUDA events around
`steps` frames after `warmup`.  Scenes: synthetic.scene_room and S1 (plane at 3 m), poses from synthetic.stream_poses,
frames already on the device.  Reports frames/s for both modes, and for log-odds the tslam_octo_get_stats counts per
frame, miss-cell visits/s and algorithmic bytes/s, next to the card's name and power limit read in the same run.

Algorithmic bytes per log-odds frame: 2 B per sampled pixel, the 16 B ray record written and read (32 B per ray), one
4 B mark-word test per miss-cell visit, and per updated voxel its 4 + 4 B log-odds read and write plus its two mark bits
read and cleared (0.5 B).

On each finished map the readers are timed too (ms per call, CUDA events over `READER_REPS` calls after one warm-up
call, inputs on the device, seeded): tslam_octo_query_points on 2^20 points uniform in the 8 m cube around the mean
sensor position, tslam_octo_raycast on 2^20 rays of 4 m from the sensor positions in uniform directions,
tslam_octo_query_near_occupy at voxel 3 on the same 2^20 points, tslam_octo_extract2 at levels 1 and 2 (with the
zeroing of its device counter), and tslam_octo_fuse of the map into a global map of the same kind (its reset included).
One JSON line.
Usage: python tools/bench_octo_logodds.py [steps] [warmup]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import _capi as capi
from taichislam_b200 import synthetic as syn
from taichislam_b200.octo_handle import OctoHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 100
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 10
LO = dict(l_hit=868, l_miss=-415, l_min=-2048, l_max=3595, l_occ=0)
dev = torch.device("cuda", torch.cuda.current_device())


READER_REPS = 20
NQ = 1 << 20


def timed_ms(call):
    call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(READER_REPS):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / READER_REPS


def readers(h, Ts, logodds):
    L, st, p = h.L, capi.stream_ptr(), capi.tptr
    rng = np.random.default_rng(0)
    pts = torch.from_numpy((Ts.mean(0) + rng.uniform(-4.0, 4.0, size=(NQ, 3))).astype(np.float32)).to(dev)
    org = torch.from_numpy(Ts[rng.integers(0, len(Ts), NQ)].astype(np.float32)).to(dev)
    dr = rng.normal(size=(NQ, 3))
    dr = torch.from_numpy((dr / np.linalg.norm(dr, axis=1, keepdims=True)).astype(np.float32)).to(dev)
    u8 = lambda *shape: torch.empty(shape, dtype=torch.uint8, device=dev)
    f32 = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
    flags, near, hit, xyz, ln = u8(NQ), u8(NQ), u8(NQ), f32(NQ, 3), f32(NQ)
    ms = {"query_points": timed_ms(lambda: capi.check(L.tslam_octo_query_points(h.h, 0, NQ, p(pts), p(flags), st))),
          "raycast_4m": timed_ms(lambda: capi.check(L.tslam_octo_raycast(h.h, 0, NQ, p(org), p(dr), 4.0, p(hit), p(xyz), p(ln), st))),
          "query_near_voxel3": timed_ms(lambda: capi.check(L.tslam_octo_query_near_occupy(h.h, 0, NQ, p(pts), 3, p(near), st)))}
    out = {"hit_frac": float(hit.float().mean()), "occupied_frac": float((flags & 1).float().mean()),
           "near_frac": float(near.float().mean())}
    for level in (1, 2):
        cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        capi.check(L.tslam_octo_extract2(h.h, 0, level, 0, p(f32(1, 3)), None, p(cnt), st))
        rows = int(cnt.item())
        buf = f32(max(rows, 1), 3)

        def export():
            cnt.zero_()
            capi.check(L.tslam_octo_extract2(h.h, 0, level, rows, p(buf), None, p(cnt), st))
        ms[f"export_level{level}"] = timed_ms(export)
        out[f"export_level{level}_rows"] = rows
    gl = OctoHandle(512, 512, K=2, voxel_scale=0.05, max_ray_length=5.0, Kcam=syn.K_DEPTH, logodds=LO if logodds else None)
    gl.set_submap_pose(0, np.eye(3), np.zeros(3))
    ms["fuse_into_global"] = timed_ms(lambda: gl.fuse_from(h))
    gl.sync()
    gl.close()
    out["ms_per_call"] = ms
    return out


def run(scene, logodds):
    h = OctoHandle(512, 512, K=2, voxel_scale=0.05, max_ray_length=5.0, Kcam=syn.K_DEPTH, logodds=LO if logodds else None)
    d = torch.from_numpy(scene.astype(np.int16)).to(dev)
    Rs, Ts = syn.stream_poses(warmup + steps)
    for q in range(warmup):
        h.integrate_depth(d, Rs[q], Ts[q])
    h.sync()
    if logodds:
        h.stats(clear=True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for q in range(warmup, warmup + steps):
        h.integrate_depth(d, Rs[q], Ts[q])
    e1.record()
    h.sync()
    ms = e0.elapsed_time(e1)
    out = {"frames_per_s": steps / (ms / 1000.0), "ms_per_frame": ms / steps}
    if logodds:
        st = h.stats()
        px = (scene.shape[0] // 2) * (scene.shape[1] // 2)
        per = {k: v / steps for k, v in st.items()}
        b = 2 * px + 32 * per["rays"] + 4 * per["miss_visits"] + 8.5 * per["updated_voxels"]
        out.update({"per_frame": per, "miss_visits_per_s": per["miss_visits"] * out["frames_per_s"],
                    "algorithmic_bytes_per_frame": b, "algorithmic_GB_per_s": b * out["frames_per_s"] / 1e9})
    out["readers"] = readers(h, np.asarray(Ts[: warmup + steps], dtype=np.float64), logodds)
    h.close()
    return out


res = {"steps": steps, "warmup": warmup, "reader_reps": READER_REPS, "reader_n": NQ}
for name, scene in (("room", syn.scene_room()), ("S1_3m", syn.scene_plane(3.0))):
    res[name] = {"hits": run(scene, False), "logodds": run(scene, True)}
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
