#!/usr/bin/env python3
"""BASELINE config 5: multi-submap TSDF fusion spatially sharded across the GPUs of one box.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29533 tools/bench_c5.py

64 submaps (20 frames of the S2 scene each, base poses on an 8x8 grid, 6 m pitch), integrated submap-sharded
(rank r owns submaps r, r+W, ...), fused into a 2048^3 x 0.05 m global volume tiled over the ranks (2x2x2 for 8):
foreign blocks travel in one NCCL all-to-all, the boundary layer is exchanged as ghost blocks, marching cubes runs
locally and the triangle soup is all-gathered.  Then the tiled ESDF of the fused map (exchange rounds of boundary-block
ESDF until no rank sends) and routed ESDF queries (2^20 uniform points per rank, answered by the owning ranks), a
routed raycast (2^16 rays per rank, 4 m, handed across tile seams; rounds and forwarded rays reported beside the
time) and one TopoGraphGen run on the tiled map, all ranks in lockstep.  Last, the incremental tiled fusion
(TiledGlobalMap.update_fused_submaps): its first update (a full one), then one submap moved 5 cm (incremental: only
that submap's integer deltas travel to the tile owners).
Prints one JSON line on rank 0, with the GPU model and its power limit beside the figures."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist


def _power_limit(dev):
    """Enforced power limit of the GPU in W (read only), or None where NVML cannot say."""
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(dev)) / 1000.0
    except Exception:
        return None


def main():
    rank = int(os.environ.get("RANK", "0")); local = int(os.environ.get("LOCAL_RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from taichi_slam.mapping import DenseTSDF, MarchingCubeMesher
    from taichislam_b200 import synthetic as syn
    from taichislam_b200.distributed import TiledGlobalMap, submap_owner, factor_tiles
    n_sub, frames_per = 64, 20
    sub = DenseTSDF(map_scale=[25.6, 25.6], voxel_scale=0.05, max_submap_num=64, max_disp_particles=1024, max_blocks=60000)
    sub.set_dep_camera_intrinsic(syn.K_DEPTH)
    glo = DenseTSDF(map_scale=[102.4, 102.4], voxel_scale=0.05, is_global_map=True, max_submap_num=64, max_disp_particles=1024,
                    max_blocks=120000)
    d = syn.scene_sphere(4.0)
    pinned = torch.from_numpy(d.view(np.int16)).pin_memory().numpy().view(np.uint16)
    mine = [s for s in range(n_sub) if submap_owner(s, world) == rank]
    for s in range(n_sub):
        gx, gy = s % 8, s // 8
        a = 0.3 * s
        Rb = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]])
        Tb = np.array([6.0 * (gx - 3.5), 6.0 * (gy - 3.5), 0.0])
        glo.set_base_pose_submap(s, Rb, Tb)
    torch.cuda.synchronize(); dist.barrier()
    t0 = time.perf_counter()
    for s in mine:
        sub.active_submap_id[None] = s
        sub.set_base_pose_submap(s, np.eye(3), np.zeros(3))
        for q in range(frames_per):
            R, T = syn.stream_pose(q * 7)
            sub.recast_depth_to_map(R, T, pinned, np.array([]))
    sub._flush(); torch.cuda.synchronize(); dist.barrier()
    t_int = time.perf_counter() - t0
    tiled = TiledGlobalMap(glo, dist, rank, world)
    tiled.fuse_submaps_tiled(sub)  # warm (NCCL channels, allocations)
    torch.cuda.synchronize(); dist.barrier()
    t0 = time.perf_counter()
    tiled.fuse_submaps_tiled(sub)
    torch.cuda.synchronize(); dist.barrier()
    t_fuse = time.perf_counter() - t0
    x = dict(tiled.last_exchange)
    mesher = MarchingCubeMesher(glo, 3000000, tsdf_surface_thres=0.25)
    t0 = time.perf_counter()
    mv, mn, counts = tiled.generate_mesh_all_gather(mesher)
    torch.cuda.synchronize(); dist.barrier()
    t_mesh = time.perf_counter() - t0
    x.update(tiled.last_exchange)
    t0 = time.perf_counter()
    es = tiled.esdf_update()  # (the mesh's halo exchange is current: no TSDF halo inside)
    torch.cuda.synchronize(); dist.barrier()
    t_esdf = time.perf_counter() - t0
    rng = np.random.default_rng(rank)
    pts = torch.from_numpy(rng.uniform([-51.2, -51.2, -2.0], [51.2, 51.2, 6.0], size=(1 << 20, 3)).astype(np.float32)).cuda()
    tiled.esdf_query(pts)  # warm
    torch.cuda.synchronize(); dist.barrier()
    t0 = time.perf_counter()
    reps = 5
    for _ in range(reps):
        dq, gq, vq = tiled.esdf_query(pts)
    torch.cuda.synchronize(); dist.barrier()
    t_query = (time.perf_counter() - t0) / reps
    # routed raycast: 2^16 rays per rank from uniform origins in the surveyed slab, 4 m long, handed across tile seams
    rp = rng.uniform([-48.0, -48.0, -1.0], [48.0, 48.0, 4.0], size=(1 << 16, 3)).astype(np.float32)
    rd = rng.normal(size=(1 << 16, 3)).astype(np.float32)
    rd /= np.linalg.norm(rd, axis=1, keepdims=True)
    tiled.raycast(rp, rd, 4.0)  # warm
    torch.cuda.synchronize(); dist.barrier()
    t0 = time.perf_counter()
    tiled.raycast(rp, rd, 4.0)
    torch.cuda.synchronize(); dist.barrier()
    t_ray = time.perf_counter() - t0
    rq = dict(tiled.last_query)
    # one TopoGraphGen run on the tiled map, every rank in lockstep (its queries are collectives)
    from taichi_slam.mapping import TopoGraphGen
    topo = TopoGraphGen(tiled)
    t0 = time.perf_counter()
    n_nodes = topo.generate_topo_graph(np.array([0.0, 0.0, 1.0]), max_nodes=20)
    torch.cuda.synchronize(); dist.barrier()
    t_topo = time.perf_counter() - t0
    # incremental tiled fusion: the first update is full, then one submap moves 5 cm
    t0 = time.perf_counter()
    tiled.update_fused_submaps(sub)
    torch.cuda.synchronize(); dist.barrier()
    t_upd_full = time.perf_counter() - t0
    a = 0.0
    glo.set_base_pose_submap(0, np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]]),
                             np.array([6.0 * (0 - 3.5) + 0.05, 6.0 * (0 - 3.5), 0.0]))
    t0 = time.perf_counter()
    upd = tiled.update_fused_submaps(sub)
    torch.cuda.synchronize(); dist.barrier()
    t_upd_move = time.perf_counter() - t0
    esx = torch.tensor([es["blocks_sent"], es["bytes_sent"], int(vq.sum().item())], dtype=torch.float64, device="cuda")
    dist.all_reduce(esx)
    own = torch.tensor([glo.count_active(), sum(sub._h.count_active(s) for s in mine), x["fusion_blocks_sent"], x.get("halo_blocks_sent", 0),
                        glo._h.stats()["n_blocks"]], dtype=torch.float64, device="cuda")
    dist.all_reduce(own)
    if rank == 0:
        print(json.dumps({"config": "C5 multi-submap fusion, 2048^3 effective volume", "n_gpus": world, "tiles": list(factor_tiles(world)),
                          "submaps": n_sub, "frames": n_sub * frames_per, "integrate_s": t_int, "integrate_frames_per_s": n_sub * frames_per / t_int,
                          "fuse_ms": 1e3 * t_fuse, "source_voxels": int(own[1].item()), "global_voxels": int(own[0].item()),
                          "fusion_blocks_exchanged": int(own[2].item()), "fusion_exchange_MB": own[2].item() * (8 + 4096 * 10) / 1e6,
                          "halo_blocks_exchanged": int(own[3].item()), "mesh_ms_incl_halo_and_allgather": 1e3 * t_mesh,
                          "triangles": int(sum(counts)), "triangles_per_rank": counts, "global_blocks": int(own[4].item()),
                          "esdf_ms": 1e3 * t_esdf, "esdf_rounds": es["rounds"], "esdf_halo_blocks": int(esx[0].item()),
                          "esdf_halo_MB": esx[1].item() / 1e6, "query_points_per_rank": 1 << 20, "query_ms": 1e3 * t_query,
                          "query_Gpoints_per_s": world * (1 << 20) / t_query / 1e9, "query_valid": int(esx[2].item()),
                          "raycast_rays_per_rank": 1 << 16, "raycast_ms": 1e3 * t_ray, "raycast_rounds": rq["rounds"],
                          "raycast_rays_forwarded": rq["rays_forwarded"], "topo_ms": 1e3 * t_topo, "topo_nodes": int(n_nodes),
                          "update_full_ms": 1e3 * t_upd_full, "update_move1_ms": 1e3 * t_upd_move, "update_move1_reason": upd["reason"],
                          "update_move1_blocks_sent": upd["foreign_blocks_sent"], "update_move1_MB_sent": upd["bytes_sent"] / 1e6,
                          "gpu": torch.cuda.get_device_name(local), "power_limit_W": _power_limit(local)}))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
