"""Multi-GPU (NCCL) test of the tiled ESDF: esdf_update, routed esdf_query and the slice all-gather on 2 ranks ==
one map holding both tiles, bit for bit.  Needs >= 2 GPUs; skipped otherwise."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    import sys
    import torch
    import torch.distributed as dist
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_gpu_multi import _build_inputs, _make_maps
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from taichislam_b200.distributed import TiledGlobalMap, all_gather_ragged, submap_owner
        d, K, poses = _build_inputs()
        sub, glo = _make_maps(K)
        for s, (R, T) in poses.items():
            glo.set_base_pose_submap(s, R, T)
            if submap_owner(s, world) != rank:
                continue
            sub.active_submap_id[None] = s
            sub.set_base_pose_submap(s, np.eye(3), np.zeros(3))
            sub.recast_depth_to_map(np.eye(3), np.zeros(3), d, np.array([]))
        tiled = TiledGlobalMap(glo, dist, rank, world)
        tiled.fuse_submaps_tiled(sub)
        st = tiled.esdf_update()
        rows = [all_gather_ragged(dist, a, world)[0].cpu().numpy() for a in glo._h.gather_device(0)]
        ei, ee = glo._h.esdf_gather(0)
        eia = all_gather_ragged(dist, torch.from_numpy(ei).cuda(), world)[0].cpu().numpy()
        eea = all_gather_ragged(dist, torch.from_numpy(ee).cuda(), world)[0].cpu().numpy()
        rng = np.random.default_rng(rank)
        pts = rng.uniform(-3.3, 3.3, size=(1 << 16, 3)).astype(np.float32)
        dq, gq, vq = tiled.esdf_query(torch.from_numpy(pts).cuda())
        sx, sv = tiled.esdf_slice_all_gather(0.1)
        out = (st, rows, eia, eea, pts, dq.cpu().numpy(), gq.cpu().numpy(), vq.cpu().numpy(), sx.cpu().numpy(), sv.cpu().numpy())
        parts = [None] * world
        dist.all_gather_object(parts, out)
        if rank == 0:
            q.put(("ok", parts))
        dist.barrier()
    except Exception:  # pragma: no cover
        import traceback
        q.put(("err", rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_tiled_esdf_and_queries_match_single_gpu():
    import torch
    import torch.multiprocessing as mp
    from test_gpu_multi import _free_port
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
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
    parts = res[1]
    st, rows, eia, eea = parts[0][:4]
    assert st["rounds"] >= 1 and st["blocks_sent"] > 0
    from taichi_slam.mapping import DenseTSDF
    from util import as_dict_rows
    ref = DenseTSDF(map_scale=[12.8, 12.8], voxel_scale=0.05, is_global_map=True, max_submap_num=8, max_disp_particles=1024)
    ref._h.scatter(0, *rows)
    ref._h.esdf_update2(0, full=True)
    si, se = as_dict_rows(*ref._h.esdf_gather(0))
    gi, ge = as_dict_rows(eia, eea)
    assert np.array_equal(gi, si) and np.array_equal(ge.view(np.uint32), se.view(np.uint32))
    for p in parts:
        pts, dq, gq, vq = p[4:8]
        d, g, v = ref._h.esdf_query(pts)
        assert np.array_equal(dq.view(np.uint32), d.view(np.uint32)) and np.array_equal(gq.view(np.uint32), g.view(np.uint32))
        assert np.array_equal(vq, v) and v.any()
    n, sx, sv = ref._h.esdf_slice(0.1)
    a = np.concatenate([parts[0][8], parts[0][9][:, None]], 1)
    b = np.concatenate([sx, sv[:, None]], 1)
    a, b = a[np.lexsort(a.T[::-1])], b[np.lexsort(b.T[::-1])]
    assert n > 0 and np.array_equal(a.view(np.uint32), b.view(np.uint32))
