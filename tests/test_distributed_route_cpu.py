"""World-size-2 gloo test (CPU) of the query routing of taichislam_b200/distributed.py: rows go out to the rank each
names, are answered there, and the answers come back in the caller's row order."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from taichislam_b200 import distributed as D


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rng = np.random.default_rng(rank)
        n = 1000 + 37 * rank
        rows = torch.from_numpy(rng.normal(size=(n, 3)).astype(np.float32))
        dest = torch.from_numpy(rng.integers(0, world, size=n))
        if rank == 1:
            dest[:] = 0  # one rank sends everything one way
        seen = []

        def answer(pts):  # the answering rank stamps its rank; the payload identifies the row
            seen.append(pts.shape[0])
            return (pts * 2.0 + rank * 1000.0, torch.full((pts.shape[0],), rank, dtype=torch.uint8))

        a, who = D.routed_answers(dist, rows, dest, world, answer)
        assert torch.equal(who.long(), dest), "answered by the wrong rank"
        assert torch.equal(a, rows * 2.0 + dest[:, None].float() * 1000.0), "answers out of the caller's order"
        # no rows at all on one rank
        e, _ = D.routed_answers(dist, rows[:0] if rank == 0 else rows, dest[:0] if rank == 0 else dest, world, answer)
        assert e.shape[0] == (0 if rank == 0 else n)
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc()))
    finally:
        dist.destroy_process_group()


def test_gloo_world2_routed_answers_come_back_in_caller_order():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in ps:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res


def test_route_order_groups_rows_by_destination():
    dest = torch.tensor([2, 0, 1, 0, 2, 2, 1])
    order, counts = D.route_order(dest, 4)
    assert counts.tolist() == [2, 2, 3, 0]
    assert dest[order].tolist() == [0, 0, 1, 1, 2, 2, 2]
    assert order.tolist() == [1, 3, 2, 6, 0, 4, 5]  # stable
    x = torch.arange(7) * 10
    assert torch.equal(D.route_restore(order, x[order]), x)
