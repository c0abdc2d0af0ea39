"""The plan merge of the tiled incremental fusion (taichislam_b200.distributed.merge_fuse_plans) as a pure function of
the ranks' plan rows, and once over a gloo world of 2 the way TiledGlobalMap.update_fused_submaps gathers them."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from taichislam_b200 import _capi as capi
from taichislam_b200 import distributed as D

S = 8


def row(reason=0, cost=0, cost_full=0, present=(), include=None):
    p = np.zeros(S, np.int64)
    p[list(present)] = 1
    inc = np.ones(S, np.int64) if include is None else np.asarray(include, np.int64)
    return np.concatenate([[reason, cost, cost_full], p, inc])


def test_incremental_when_every_rank_is():
    assert D.merge_fuse_plans([row(0, 3, 10, [0, 2]), row(0, 4, 12, [1, 3])]) == 0
    assert D.merge_fuse_plans([row(0, 0, 0)]) == 0                     # world 1, nothing to do


def test_full_everywhere_when_one_rank_is_full_with_the_smallest_reason():
    assert D.merge_fuse_plans([row(0, 1, 10, [0]), row(5, 0, 12, [1])]) == 5
    assert D.merge_fuse_plans([row(8, 0, 1), row(7, 0, 1), row(0, 0, 1), row(4, 0, 1)]) == 4
    assert D.merge_fuse_plans([row(8), row(1)]) == 1
    assert capi.TILED_FUSE_REASONS[7] == "tile cuts changed" and capi.TILED_FUSE_REASONS[8] == "sums not valid"


def test_cost_rule_uses_the_sums_over_the_ranks():
    # each rank alone would stay incremental (rank 1 is over on its own, but the sums are not)
    assert D.merge_fuse_plans([row(0, 2, 10), row(0, 14, 12)]) == 0
    assert D.merge_fuse_plans([row(0, 11, 10), row(0, 12, 12)]) == 6
    assert D.merge_fuse_plans([row(0, 10, 10), row(0, 12, 12)]) == 0   # equal cost stays incremental, as on one map


def test_a_submap_on_two_ranks_is_refused():
    with pytest.raises(ValueError, match=r"submaps \[3\] have blocks on several ranks"):
        D.merge_fuse_plans([row(0, present=[1, 3]), row(0, present=[3, 4])])
    with pytest.raises(ValueError, match="several ranks"):                 # also when a rank is full anyway
        D.merge_fuse_plans([row(1, present=[0]), row(0, present=[0])])


def test_include_must_match():
    inc = np.ones(S, np.int64)
    inc2 = inc.copy()
    inc2[5] = 0
    assert D.merge_fuse_plans([row(include=inc), row(include=inc)]) == 0
    with pytest.raises(ValueError, match=r"include differs between ranks \(submaps \[5\]\)"):
        D.merge_fuse_plans([row(include=inc), row(include=inc2)])


def test_malformed_rows_are_refused():
    with pytest.raises(ValueError, match="plan rows"):
        D.merge_fuse_plans(np.zeros((2, 4), np.int64))
    with pytest.raises(ValueError, match="plan rows"):
        D.merge_fuse_plans(np.zeros(19, np.int64))


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
        cases = [  # (rank 0's row, rank 1's row, expected reason or None for a refusal)
            (row(0, 3, 10, [0]), row(0, 4, 10, [1]), 0),
            (row(0, 3, 10, [0]), row(7, 0, 10, [1]), 7),
            (row(0, 11, 10, [0]), row(0, 12, 12, [1]), 6),
            (row(0, 0, 10, [0, 1]), row(0, 0, 10, [1]), None),
            (row(0, 0, 10, [0], include=[1] * S), row(0, 0, 10, [1], include=[0] + [1] * (S - 1)), None),
        ]
        for r0, r1, want in cases:
            mine = torch.as_tensor(r0 if rank == 0 else r1)
            parts = [torch.empty_like(mine) for _ in range(world)]
            dist.all_gather(parts, mine)
            rows = torch.stack(parts).numpy()
            try:
                got = D.merge_fuse_plans(rows)
            except ValueError:
                got = None
            assert got == want, (r0, r1, got, want)
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_gloo_world2_every_rank_merges_the_same_plan():
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
