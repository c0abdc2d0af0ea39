#!/usr/bin/env python3
"""Log-odds Octomap against the hit counter on the same frames: depth frames streamed into a 512^3 Octomap
(map_scale 25.6 m, 0.05 m voxels, max_ray_length = 5 m, recast_step 2), both modes in one run, CUDA events around
`steps` frames after `warmup`.  Scenes: synthetic.scene_room and S1 (plane at 3 m), poses from synthetic.stream_poses,
frames already on the device.  Reports frames/s for both modes, and for log-odds the tslam_octo_get_stats counts per
frame, miss-cell visits/s and algorithmic bytes/s, next to the card's name and power limit read in the same run.

Algorithmic bytes per log-odds frame: 2 B per sampled pixel, the 16 B ray record written and read (32 B per ray), one
4 B mark-word test per miss-cell visit, and per updated voxel its 4 + 4 B log-odds read and write plus its two mark bits
read and cleared (0.5 B).  One JSON line.
Usage: python tools/bench_octo_logodds.py [steps] [warmup]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.octo_handle import OctoHandle

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 100
warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 10
LO = dict(l_hit=868, l_miss=-415, l_min=-2048, l_max=3595, l_occ=0)
dev = torch.device("cuda", torch.cuda.current_device())


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
    h.close()
    return out


res = {"steps": steps, "warmup": warmup}
for name, scene in (("room", syn.scene_room()), ("S1_3m", syn.scene_plane(3.0))):
    res[name] = {"hits": run(scene, False), "logodds": run(scene, True)}
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                     capture_output=True, text=True).stdout.strip()
res["gpu"] = torch.cuda.get_device_name()
res["nvidia_smi_name_power_limit"] = smi
print(json.dumps(res), flush=True)
