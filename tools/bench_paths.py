#!/usr/bin/env python3
"""Time every path of SURVEY.md section 8 on one GPU (CUDA events, warm) and print a markdown table.
Not the headline bench (bench.py).  Usage: python tools/bench_paths.py > paths.md"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from taichislam_b200 import synthetic as syn
from taichislam_b200.tsdf_handle import TsdfHandle
from taichislam_b200.octo_handle import OctoHandle

PEAK = 6564.2  # GB/s, MEASURED_PEAKS.json


def timed(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


rows = []
# --- integrate, per scene (64-frame batches, device-resident) ---
for name, d in (("S1 plane 3 m", syn.scene_plane(3.0)), ("S2 sphere 4 m", syn.scene_sphere(4.0)), ("S3 sphere 8 m", syn.scene_sphere(8.0)),
                ("S4 noise 1.5-4.5 m", syn.scene_noise())):
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    dd = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(d, (64,) + d.shape)).view(np.int16)).cuda()
    Rs, Ts = syn.stream_poses(64)
    g.stats(clear=True)
    g.set_profiling(True)
    ms = timed(lambda: g.integrate_depth(dd, Rs, Ts), reps=5, warm=2)
    st = g.stats()
    km = g.kernel_ms2(5).mean(axis=0)
    calls = 7
    per_frame = (2.0 * st["n_px"] + 24.0 * st["n_valid"] + 17.0 * st["n_rays"] + 9.0 * st["n_updates"]) / (calls * 64)
    rows.append((f"integrate {name} -> 512^3", f"{64e3 / ms:,.0f} frames/s", f"{ms:.3f} ms / 64 frames",
                 f"{st['n_rays'] / calls / 64:,.0f} rays, {st['n_updates'] / calls / 64 / 1e6:.2f} M updates, {per_frame / 1e6:.1f} MB algorithmic per frame -> "
                 f"{per_frame * 64 / ms / 1e6:,.0f} GB/s = {per_frame * 64 / ms / 1e6 / PEAK * 100:.1f} % of HBM peak; kernels: bucket {km[0]:.3f}, "
                 f"set-up+walk+scan {km[3] + km[4]:.3f}, place {km[5]:.3f}, block march {km[6]:.3f}, commit {km[2]:.3f} ms"))
    g.close()

# --- C2: marching cubes after 100 stream frames ---
g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
d = syn.scene_sphere(4.0)
for b in range(2):
    Rs, Ts = syn.stream_poses(50, start=50 * b)
    g.integrate_depth(np.broadcast_to(d, (50,) + d.shape), Rs, Ts)
dev = torch.device("cuda")
cap = 1 << 21
v = torch.empty((3 * cap, 3), dtype=torch.float32, device=dev); nrm = torch.empty_like(v)
import ctypes as C
from taichislam_b200 import _capi as capi
ntri = C.c_int64(0)
def mc():
    capi.check(g.L.tslam_mc_generate(g.h, 1, 0.25, cap, capi.tptr(v), capi.tptr(nrm), C.byref(ntri), capi.stream_ptr()))
ms = timed(mc)
nblk = g.stats()["n_blocks"]
bytes_mc = 3.0 * nblk * 4096 + 72.0 * ntri.value
rows.append(("C2 marching cubes (512^3 map after 100 frames)", f"{ntri.value / ms * 1e3 / 1e6:,.1f} M triangles/s", f"{ms:.3f} ms",
             f"{ntri.value:,} triangles from {nblk} blocks; {bytes_mc / 1e6:.1f} MB algorithmic -> {bytes_mc / ms / 1e6:,.0f} GB/s"))
# --- C4: ESDF: full recompute, then incremental updates after every further frame of the stream ---
torch.cuda.synchronize(); t0 = time.perf_counter()
st_full = g.esdf_update2(0, full=True)
torch.cuda.synchronize(); ms = 1e3 * (time.perf_counter() - t0)
nvox = g.count_active()
rows.append(("C4 ESDF full recompute (same map)", f"{nvox / ms * 1e3 / 1e6:,.1f} M voxels/s", f"{ms:.2f} ms",
             f"{nvox:,} observed voxels, {st_full['lower_sweeps']} sweeps"))
inc_ms, inc_stats = [], []
for q in range(8):
    Rq, Tq = syn.stream_poses(1, start=100 + q)
    g.integrate_depth(d, Rq, Tq)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    si = g.esdf_update2(0)
    torch.cuda.synchronize(); inc_ms.append(1e3 * (time.perf_counter() - t0)); inc_stats.append(si)
rows.append(("C4 ESDF incremental update after one more frame", f"{np.mean(inc_ms[2:]):.2f} ms / frame", f"{min(inc_ms):.2f} - {max(inc_ms):.2f} ms",
             f"changed {np.mean([x['changed'] for x in inc_stats]):,.0f} / suspect {np.mean([x['suspect'] for x in inc_stats]):,.0f} voxels per update, "
             f"raise sweeps {inc_stats[-1]['raise_sweeps']}, lower sweeps {inc_stats[-1]['lower_sweeps']} (every frame moves the TSDF of "
             f"the whole visible band, so the wave covers the view, not just a rim)"))
# --- surface export / gather ---
xyz = torch.empty((1 << 22, 3), dtype=torch.float32, device=dev); rgb = torch.empty_like(xyz); cnt = torch.zeros(1, dtype=torch.int32, device=dev)
def surf():
    cnt.zero_(); g.extract_surface(0, xyz, rgb, cnt)
ms = timed(surf)
rows.append(("surface export (cvt_TSDF_surface_to_voxels)", f"{nvox / ms * 1e3 / 1e6:,.0f} M voxels scanned/s", f"{ms:.3f} ms", f"{int(cnt.item()):,} surface voxels"))
g.close()

# --- C3: octomap ---
o = OctoHandle(1024, 1024, K=2, voxel_scale=0.05, min_occupy_thres=2)
pts = torch.from_numpy(syn.octo_cloud(100000, seed=1)).cuda()
R, T = np.eye(3), np.zeros(3)
ms = timed(lambda: o.integrate_points(pts, R, T), reps=20, warm=3)
rows.append(("C3 Octomap 100k-point cloud -> 1024^3 hit counts", f"{100000 / ms * 1e3 / 1e9:.2f} G points/s", f"{ms * 1e3:.1f} us / frame",
             f"20 B/point algorithmic -> {2.0e6 / ms / 1e6:,.0f} GB/s"))
o.close()

# --- fusion: 8 submaps -> global ---
sub = TsdfHandle(256, 256, K=syn.K_DEPTH, max_submaps=16)
glo = TsdfHandle(1024, 1024, is_global_map=True, max_submaps=16)
d = syn.scene_sphere(3.0)
from math import cos, sin
for s in range(8):
    a = 0.7 * s
    Rb = np.array([[cos(a), -sin(a), 0], [sin(a), cos(a), 0], [0, 0, 1.0]])
    glo.set_submap_pose(s, Rb, np.array([3.0 * (s % 4) - 4.0, 4.0 * (s // 4) - 2.0, 0.1 * s]))
    Rs, Ts = syn.stream_poses(10, start=10 * s)
    sub.integrate_depth(np.broadcast_to(d, (10,) + d.shape), Rs, Ts, submaps=[s] * 10)
nsrc = sum(sub.count_active(s) for s in range(8))
ms = timed(lambda: glo.fuse_from(sub), reps=3, warm=1)
rows.append(("D1 submap -> global fusion (8 submaps)", f"{nsrc / ms * 1e3 / 1e6:,.0f} M source voxels/s", f"{ms:.2f} ms",
             f"{nsrc:,} observed source voxels x 7 corners; 90 B/voxel algorithmic -> {90.0 * nsrc / ms / 1e6:,.0f} GB/s"))

# --- texture: coloured integrate (k_raymarch: colour-word atomicMax next to every reduction) + coloured MC ---
gt = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True, texture_enabled=True)
gt.set_color_intrinsics([1, 0, 0, 0, 1, 0, 0, 0, 1], True)
d = syn.scene_sphere(4.0)
dd = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(d, (64,) + d.shape)).view(np.int16)).cuda()
rng = np.random.default_rng(0)
tex = torch.from_numpy(rng.integers(1, 255, (64, 480, 640, 3)).astype(np.uint8)).cuda()
Rs, Ts = syn.stream_poses(64)
ms = timed(lambda: gt.integrate_depth(dd, Rs, Ts, texture=tex), reps=5, warm=2)
rows.append(("textured integrate S2 sphere 4 m -> 512^3 (depth + uint8 RGB image)", f"{64e3 / ms:,.0f} frames/s", f"{ms:.3f} ms / 64 frames",
             "colour sums in the bucket pass, 64-bit colour-word atomicMax per sample (1 CTA/SM: 128 KB window)"))
vc = torch.empty((3 * cap, 3), dtype=torch.float32, device=dev)
def mcc():
    capi.check(gt.L.tslam_mc_generate2(gt.h, 1, 0.25, cap, capi.tptr(v), capi.tptr(nrm), capi.tptr(vc), C.byref(ntri), capi.stream_ptr()))
ms = timed(mcc)
rows.append(("coloured marching cubes (vertexInterp_color)", f"{ntri.value / ms * 1e3 / 1e6:,.1f} M triangles/s", f"{ms:.3f} ms", f"{ntri.value:,} triangles"))
gt.close()

# --- marching cubes where bandwidth matters: a map of several thousand blocks (sphere R = 9.5 m seen from three rings of poses) ---
gb = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True, max_blocks=20000)
d9 = syn.scene_sphere(9.5)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from util_rot import rot_xyz
for ring, pitch in enumerate((-0.9, 0.0, 0.9)):
    Rs = np.stack([rot_xyz(pitch, 0.0, 2 * np.pi * k / 48) for k in range(48)])
    gb.integrate_depth(np.broadcast_to(d9, (48,) + d9.shape), Rs, np.zeros((48, 3)))
nblk_b = gb.stats()["n_blocks"]
capb = 1 << 23
vb = torch.empty((3 * capb, 3), dtype=torch.float32, device=dev); nb_ = torch.empty_like(vb)
ntb = C.c_int64(0)
def mcb():
    capi.check(gb.L.tslam_mc_generate(gb.h, 1, 0.25, capb, capi.tptr(vb), capi.tptr(nb_), C.byref(ntb), capi.stream_ptr()))
ms = timed(mcb, reps=3, warm=1)
bytes_b = 3.0 * nblk_b * 4096 + 72.0 * ntb.value
rows.append((f"marching cubes on a {nblk_b}-block map", f"{ntb.value / ms * 1e3 / 1e6:,.1f} M triangles/s", f"{ms:.3f} ms",
             f"{ntb.value:,} triangles; {bytes_b / 1e6:.1f} MB algorithmic -> {bytes_b / ms / 1e6:,.0f} GB/s = {bytes_b / ms / 1e6 / PEAK * 100:.1f} % of HBM peak"))
gb.close()

print("| path | throughput | time | detail |\n|---|---|---|---|")
for r in rows:
    print("| " + " | ".join(r) + " |")
