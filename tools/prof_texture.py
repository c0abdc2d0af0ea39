#!/usr/bin/env python3
"""Workload for an ncu capture of textured integrate (k_bucket_depth with colour sums, k_raymarch) and of the page-locked
frame queue (k_gather_rows).
    ncu --set full --clock-control none -k regex:'k_raymarch|k_gather_rows|k_bucket_depth' -s 6 -c 5 -o gpurun_out/prof_tex python tools/prof_texture.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.tsdf_handle import TsdfHandle
from taichislam_b200.mapping import DenseTSDF

g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True, texture_enabled=True)
g.set_color_intrinsics([1, 0, 0, 0, 1, 0, 0, 0, 1], True)
d = syn.scene_sphere(4.0)
dd = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(d, (64,) + d.shape)).view(np.int16)).cuda()
tex = torch.from_numpy(np.stack([syn.texture_gradient(q) for q in range(4)] * 16)).cuda()
Rs, Ts = syn.stream_poses(64)
for _ in range(3):                      # launches 0-5: bucket + raymarch (commit is k_commit_tma, not captured)
    g.integrate_depth(dd, Rs, Ts, texture=tex)
g.sync()
m = DenseTSDF(map_scale=[25.6, 25.6], voxel_scale=0.05, is_global_map=True)
m.set_dep_camera_intrinsic(syn.K_DEPTH)
m.set_base_pose_submap(0, np.eye(3), np.zeros(3))
host = torch.from_numpy(np.stack([d] * 64).view(np.int16)).pin_memory().numpy().view(np.uint16)
e = np.array([])
for q in range(64):                     # gather_rows x4 + bucket + binned march per 32 frames
    m.recast_depth_to_map(Rs[q], Ts[q], host[q], e)
print(m.frame_counters())
