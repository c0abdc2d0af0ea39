"""Multi-GPU (NCCL) test of the planner queries on the tiled map: routed raycast, point and near-occupancy queries on 2
ranks == one map holding both tiles, bit for bit, and TopoGraphGen run in lockstep on both ranks builds the single
map's graph on each.  Needs >= 2 GPUs; skipped otherwise."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    import sys
    import torch
    import torch.distributed as dist
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_gpu_dist_query import _global_map, _graph
    from topo_world import START_A, two_rooms
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from taichi_slam.mapping import TopoGraphGen
        from taichislam_b200.distributed import TiledGlobalMap
        idx, t, w, occ = two_rooms()
        tiled = TiledGlobalMap(_global_map(), dist, rank, world, balance=False)
        own = np.array([tiled.owner_of_block(*b) for b in idx >> 4])
        tiled.m._h.scatter(0, idx[own == rank], t[own == rank], w[own == rank], occ[own == rank])
        rng = np.random.default_rng(rank)
        n = 1 << 14 if rank == 0 else 1 << 10
        pos = (rng.uniform(-1.0, 1.0, size=(n, 3)) * np.array([3.5, 1.8, 1.0]) + np.array([0.0, 0.0, 0.8])).astype(np.float32)
        dirs = rng.normal(size=(n, 3)).astype(np.float32)
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        ray = tiled.raycast(pos, dirs, 3.0)
        st = dict(tiled.last_query)
        occ_q, un_q = tiled.is_pos_occupy(pos), tiled.is_pos_unobserved(pos)
        near = tiled.is_near_pos_occupy(pos, 3)          # (exchanges the halo first)
        topo = TopoGraphGen(tiled, coll_det_num=64, max_raycast_dist=2.5)
        nn = topo.generate_topo_graph(START_A, max_nodes=12)
        out = (pos, dirs, ray, st, occ_q, un_q, near, nn, _graph(topo))
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


def test_tiled_queries_and_topo_graph_match_single_gpu():
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
    res = q.get(timeout=900)
    for p in ps:
        p.join(timeout=120)
    assert res[0] == "ok", res
    from taichi_slam.mapping import TopoGraphGen
    from test_gpu_dist_query import _global_map, _graph
    from topo_world import START_A, two_rooms
    ref = _global_map()
    ref._h.scatter(0, *two_rooms())
    single = TopoGraphGen(ref, coll_det_num=64, max_raycast_dist=2.5)
    nn = single.generate_topo_graph(START_A, max_nodes=12)
    g = _graph(single)
    for pos, dirs, ray, st, occ_q, un_q, near, n_topo, graph in res[1]:
        want = ref.raycast(pos, dirs, 3.0)
        assert np.array_equal(ray[0], want[0]) and np.array_equal(ray[1].view(np.uint32), want[1].view(np.uint32))
        assert np.array_equal(ray[2].view(np.uint32), want[2].view(np.uint32))
        assert 1 <= st["rounds"] <= 2 and st["rays_forwarded"] > 0
        assert np.array_equal(occ_q, ref.is_pos_occupy(pos)) and np.array_equal(un_q, ref.is_pos_unobserved(pos))
        assert np.array_equal(near, ref.is_near_pos_occupy(pos, 3))
        assert n_topo == nn >= 2 and graph == g
