"""Multi-GPU (NCCL) test of the tiled incremental fusion: TiledGlobalMap.update_fused_submaps on 2 ranks, a first
update and then a move, each equal bit for bit to one map's tslam_tsdf_fuse_update of all submaps, with the same
reason on every rank.  Needs >= 2 GPUs; skipped otherwise."""
import os
import socket

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _inputs():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from taichislam_b200 import synthetic as syn
    from util import rot_xyz
    d = syn.scene_sphere(2.5, 240, 320)
    K = [syn.FX / 2, 0, syn.CX / 2, 0, syn.FY / 2, syn.CY / 2, 0, 0, 1]
    poses = {s: (rot_xyz(0.1 * s + 0.05, 0.2 - 0.07 * s, 0.3 * s + 0.1), np.array([1.5 * (s % 2) - 0.7, 1.2 * (s // 2) - 0.6, 0.3 * s - 0.4]))
             for s in range(4)}
    return d, K, poses


def _maps(K):
    from taichi_slam.mapping import DenseTSDF
    sub = DenseTSDF(map_scale=[6.4, 6.4], voxel_scale=0.05, max_ray_length=3.0, max_submap_num=8, max_disp_particles=1024,
                    max_image_pixels=240 * 320)
    sub.set_dep_camera_intrinsic(K)
    glo = DenseTSDF(map_scale=[12.8, 12.8], voxel_scale=0.05, is_global_map=True, max_submap_num=8, max_disp_particles=1024)
    return sub, glo


def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from taichislam_b200.distributed import TiledGlobalMap, all_gather_ragged, submap_owner
        d, K, poses = _inputs()
        sub, glo = _maps(K)
        for s, (R, T) in poses.items():
            glo.set_base_pose_submap(s, R, T)
            if submap_owner(s, world) != rank:
                continue
            sub.active_submap_id[None] = s
            sub.set_base_pose_submap(s, np.eye(3), np.zeros(3))
            sub.recast_depth_to_map(np.eye(3), np.zeros(3), d, np.array([]))
        tiled = TiledGlobalMap(glo, dist, rank, world)
        out = []
        for step in range(2):
            if step == 1:
                R, T = poses[1]
                glo.set_base_pose_submap(1, R, T + np.array([0.04, 0.0, 0.0]))
            st = tiled.update_fused_submaps(sub)
            g = glo._h.gather_device(0)
            parts = [all_gather_ragged(dist, a, world)[0].cpu().numpy() for a in g]
            out.append((st, parts))
        # every rank's submaps, gathered for the single-map check on rank 0
        mine = {s: sub._h.gather(s) for s in poses if submap_owner(s, world) == rank}
        got = [None] * world
        dist.all_gather_object(got, mine)
        if rank == 0:
            q.put(("ok", out, {k: v for m in got for k, v in m.items()}))
        dist.barrier()
    except Exception:  # pragma: no cover
        import traceback
        q.put(("err", rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_nccl_update_fused_submaps_matches_one_map():
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from fuse_update_reference import same_values
    from taichislam_b200.tsdf_handle import TsdfHandle
    from util import as_dict_rows
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = q.get(timeout=600)
    for p in ps:
        p.join(timeout=120)
    assert res[0] == "ok", res
    _, out, gathered = res
    (st0, rows0), (st1, rows1) = out
    assert st0["reason"] == "first call" and st0["foreign_blocks_sent"] > 0
    assert st1["reason"] == "incremental" and st1["moved"] == 1
    _, K, poses = _inputs()
    src = TsdfHandle(128, 128, voxel_scale=0.05, max_submaps=8)
    for s, g in gathered.items():
        src.scatter(s, *g)
    for step, rows in enumerate((rows0, rows1)):
        one = TsdfHandle(256, 256, voxel_scale=0.05, is_global_map=True, max_submaps=8)
        for s, (R, T) in poses.items():
            one.set_submap_pose(s, R, T + (np.array([0.04, 0.0, 0.0]) if step == 1 and s == 1 else 0.0))
        one.fuse_update(src)
        a, b = as_dict_rows(*rows), as_dict_rows(*one.gather(0))
        assert len(a) == len(b) and all(same_values(x, y) for x, y in zip(a, b)), step
        one.close()
