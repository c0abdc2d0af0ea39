#!/usr/bin/env python3
"""Many-source travel costs on the log-odds Octomap: the map of bench_octo_travel.py (512^3, 0.05 m voxels, 40
scene_room frames on the device, max_ray_length = 5 m), then for S in {1, 16, 64, 256} starts - the last camera cell,
the reachable cell nearest each frontier-cluster centroid, topped up with random reachable cells:
  * travel_multi_update with clearance 0 and 0.2 m (occupancy ESDF, D = 1 m): ms per update, sweeps, B_t (submap blocks
    with a traversable cell) and the state bytes those imply;
  * the same S starts as S sequential travel_update calls, alternated with the batched update in the same run;
  * travel_multi_query of the S starts (the S x S matrix);
  * travel_multi_path of 256 (source, target) pairs, targets near frontier-cluster centroids.
CUDA events around `steps` calls after `warmup`.  Card name and power limit are read in the same run.  One JSON line.
Usage: python tools/bench_octo_travel_multi.py [steps] [warmup]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.octo_handle import OctoHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 2
LO = dict(l_hit=868, l_miss=-415, l_min=-2048, l_max=3595, l_occ=0)
VS = 0.05
MAX_BLOCKS = 1 << 18  # OctoHandle's default pool
dev = torch.device("cuda", torch.cuda.current_device())
h = OctoHandle(512, 512, K=2, voxel_scale=VS, max_ray_length=5.0, Kcam=syn.K_DEPTH, logodds=LO)
depth = torch.from_numpy(syn.scene_room().astype(np.int16)).to(dev)
Rs, Ts = syn.stream_poses(40)
for q in range(40):
    h.integrate_depth(depth, Rs[q], Ts[q])
h.esdf_update(0, 1.0, full=True)
cam = np.asarray(Ts[39], np.float32)
idx, L = h.gather(0)
h.frontier_update(0)
rec = h.frontier_clusters(0)
cent = rec[:, 2:5] / rec[:, 1:2]
rng = np.random.default_rng(0)
ALL, near = {}, None
for cl in (0.0, 0.2):  # starts reachable from the camera cell at each clearance, so every batched row is a real wave
    h.travel_update(0, cam, clearance=cl)
    ri, _ = h.travel_gather(0)
    nr = np.array([ri[np.argmin(((ri - c) ** 2).sum(1))] for c in cent])
    near = nr if near is None else near
    pool = np.concatenate([nr, ri[rng.choice(len(ri), 256, replace=False)]])
    ALL[cl] = np.concatenate([cam[None], pool.astype(np.float32) * np.float32(VS)]).astype(np.float32)

# B_t: blocks with a traversable cell (FREE in the volume; with clearance also ESDF >= clearance)
e_i, e_E = h.esdf_gather(0)
b_t = {0.0: np.unique(idx[L <= LO["l_occ"]] >> 3, axis=0).shape[0], 0.2: np.unique(e_i[e_E >= 0.2] >> 3, axis=0).shape[0]}


def state_bytes(S, nt):  # DESIGN section 7: 68 B per pool block + 2160 B per slot + 2052 B per (slot, source)
    return MAX_BLOCKS * 68 + nt * 2160 + S * nt * 2052


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        out = fn()
    e1.record()
    h.sync()
    return e0.elapsed_time(e1) / n, out


res = {"steps": steps, "warmup": warmup, "map": "512^3, 0.05 m, scene_room x 40 frames, max_ray_length 5 m",
       "known_voxels": int(idx.shape[0]), "clusters": int(rec.shape[0]), "B_t": {str(k): int(v) for k, v in b_t.items()}}
for S in (1, 16, 64, 256):
    r = {}
    for cl in (0.0, 0.2):
        starts = ALL[cl][:S]
        batched = lambda: h.travel_multi_update(0, starts, clearance=cl)
        seq = lambda: [h.travel_update(0, p, clearance=cl) for p in starts]
        for _ in range(warmup):
            batched(); seq()
        tb, ts = [], []
        for _ in range(steps):  # alternated, so both see the same state of the card
            tb.append(timed(batched, 1)[0])
            ts.append(timed(seq, 1)[0])
        st = batched()
        r[f"clearance_{cl}"] = dict(batched_ms=float(np.median(tb)), sequential_ms=float(np.median(ts)),
                                    ratio=float(np.median(tb) / np.median(ts)), sweeps=st["sweeps"],
                                    traversable=st["traversable"], B_t=b_t[cl], state_bytes=state_bytes(S, b_t[cl]),
                                    start_ok=int(st["start_ok"].sum()), mean_reachable=float(st["reachable"].mean()))
    # readers against the clearance-0 fields
    starts = ALL[0.0][:S]
    st = h.travel_multi_update(0, starts)
    xs = torch.from_numpy(starts).to(dev)
    for _ in range(warmup):
        h.travel_multi_query(xs)
    ms, M = timed(lambda: h.travel_multi_query(xs), steps)
    r["matrix"] = dict(ms=ms, finite=int(torch.isfinite(M).sum().item()), asymmetric=int(((M != M.T) & torch.isfinite(M)).sum().item()))
    src = torch.from_numpy(rng.integers(S, size=256).astype(np.int32)).to(dev)
    tg = torch.from_numpy(near[rng.integers(len(near), size=256)].astype(np.float32) * np.float32(VS)).to(dev)
    for _ in range(warmup):
        h.travel_multi_path(src, tg)
    ms, (cells, ln) = timed(lambda: h.travel_multi_path(src, tg, max_len=4096), steps)
    r["paths"] = dict(pairs=256, ms=ms, mean_len=float(ln.double().mean().item()), max_len=int(ln.max().item()),
                      reached=int((ln > 0).sum().item()))
    res[f"S={S}"] = r
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
