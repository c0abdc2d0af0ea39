"""The hand-over bound of the routed raycast on a tiled map, on CPU: along a ray the tile of its samples is monotone on
each axis (numpy f32 statement of the kernel's sample and cell, ray_tiles.py), so a batch needs at most tx+ty+tz-2
hand-over rounds.  And the host round loop of taichislam_b200.distributed (raycast_rounds) driven under gloo with a
numpy stand-in for the march gives every rank the answers of one uninterrupted march, in its own row order."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import ray_tiles as rt
from taichislam_b200 import distributed as D

F = np.float32
N, NZ = 256, 256


def _rays(rng, n, vs, N=N, NZ=NZ):
    """Origins across the volume, directions with negative components, lengths over several tiles, plus rays on the
    .5 rounding tie at block boundaries, axis-aligned rays, and non-finite rays."""
    h = N // 2 * vs
    pos = rng.uniform(-h, h, size=(n, 3)).astype(F)
    dir = rng.normal(size=(n, 3)).astype(F)
    dir /= np.linalg.norm(dir, axis=1, keepdims=True)
    b = rng.integers(-N // 32, N // 32, size=(n // 4, 3))
    pos[: n // 4] = ((b * 16).astype(F) - F(0.5)) * F(vs)          # exactly on the tie of a block boundary (vs = 2^-k)
    dir[: n // 8] = 0.0
    ax = rng.integers(0, 3, size=n // 8)
    dir[np.arange(n // 8), ax] = rng.choice([-1.0, 1.0], size=n // 8)  # axis-aligned, in the tie planes
    bad = np.array([[np.nan, 0, 0], [np.inf, 0, 0], [-np.inf, 0, 0], [0, 0, 0]], F)
    pos = np.concatenate([pos, bad[:2], np.zeros((4, 3), F)])
    dir = np.concatenate([dir, np.ones((2, 3), F), bad])
    return pos, dir


def _balanced_cuts(rng, world):
    hist = np.zeros((3, 1024), np.int64)
    for a in range(3):
        hist[a, 512 - 8 + rng.integers(0, 6): 512 + 8 - rng.integers(0, 6)] = rng.integers(1, 100, size=1)
    hist[:, 512 - 8:512 + 8] += rng.integers(0, 50, size=(3, 16))
    return D.balanced_tiling(hist, world)


@pytest.mark.parametrize("world", [2, 4, 8, 12])
@pytest.mark.parametrize("balanced", [False, True])
@pytest.mark.parametrize("vs", [0.0625, 0.05])
def test_tile_of_a_ray_is_monotone_per_axis_and_within_the_bound(world, balanced, vs):
    rng = np.random.default_rng(world * 10 + balanced)
    if balanced:
        tiles, cuts = _balanced_cuts(rng, world)
        assert cuts is not None
    else:
        tiles = D.factor_tiles(world)
        cuts = rt.default_cuts(N, NZ, tiles)
    pos, dir = _rays(rng, 1500, vs)
    bound = sum(tiles) - 2
    worst = 0
    for run in rt.tile_runs(pos, dir, 6.0, vs, N, NZ, cuts, tiles):
        if len(run) == 0:
            continue
        d = np.diff(run, axis=0)
        assert np.all((d >= 0).all(0) | (d <= 0).all(0)), "tile not monotone on an axis"
        changes = int(np.count_nonzero(np.any(d != 0, axis=1)))
        assert changes <= sum(t - 1 for t in tiles)
        worst = max(worst, changes + 1)      # + the hand-over into the first sample's tile
    assert worst <= bound
    assert worst >= 2                        # the rays do cross tiles


def test_roundf_and_cells_follow_the_gpu():
    assert rt.roundf(np.array([0.5, -0.5, 1.5, 2.5, 0.49999997, -2.5], F)).tolist() == [1, -1, 2, 3, 0, -3]
    assert rt.cells(np.array([np.nan, np.inf, -np.inf, 1e30], F), 0.05).tolist() == [0, 2 ** 31 - 1, -2 ** 31, 2 ** 31 - 1]
    assert rt.tile_owner(rt.default_cuts(256, 256, (2, 2, 2)), (2, 2, 2), np.array([[-8, -8, -8], [0, 0, 0], [-1, 0, -1], [99, -99, 0]])).tolist() == [0, 7, 2, 5]


# ---- the host round loop under gloo, with the numpy march standing in for the kernel ----------------------------
VS = 0.0625
NS = 128


def _occupied(c):
    """A sparse pseudo-random occupancy of the cells (same on every rank)."""
    h = (c[:, 0] * 73856093) ^ (c[:, 1] * 19349663) ^ (c[:, 2] * 83492791)
    return (h % 997) < 4


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _batch(rank, world):
    rng = np.random.default_rng(100 + rank)
    n = 0 if rank == world - 1 else 600 + 17 * rank   # one rank asks nothing
    pos, dir = _rays(rng, n, VS, NS, NS) if n else (np.zeros((0, 3), F), np.zeros((0, 3), F))
    return pos, dir, 5.0


def _rows(pos, dir, max_dist, rank, world):
    rays = torch.zeros((len(pos), 8), dtype=torch.float32)
    rays[:, :3], rays[:, 3:6], rays[:, 6] = torch.from_numpy(pos), torch.from_numpy(dir), float(max_dist)
    return rays, torch.arange(len(pos), dtype=torch.int64) * world + rank


def _worker(rank, world, tiles, cuts, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        pos, dir, md = _batch(rank, world)
        rays, tags = _rows(pos, dir, md, rank, world)
        march = rt.march_stand_in(_occupied, VS, NS, NS, cuts, tiles, rank)
        (ans,), st = D.raycast_rounds(D._DistRouter(dist, world, torch.device("cpu")), [march], [rays], [tags], world, sum(tiles) - 2)
        one = rt.march_stand_in(_occupied, VS, NS, NS, rt.default_cuts(NS, NS, (1, 1, 1)), (1, 1, 1), 0)
        r1, _ = _rows(pos, dir, md, 0, 1)
        d1, want = one(r1)
        assert (d1 < 0).all()
        assert np.array_equal(ans.numpy().view(np.uint32), want.numpy().view(np.uint32)), "answers differ from one march"
        q.put((rank, "ok", st))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, traceback.format_exc(), None))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_gloo_round_loop_equals_one_uninterrupted_march(world):
    tiles = D.factor_tiles(world)
    cuts = rt.default_cuts(NS, NS, tiles)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, world, tiles, cuts, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = [q.get(timeout=300) for _ in range(world)]
    for p in ps:
        p.join(timeout=60)
    assert all(r[1] == "ok" for r in res), res
    stats = [r[2] for r in res]
    assert all(s == stats[0] for s in stats)               # every rank counts the same rounds
    assert 1 <= stats[0]["rounds"] <= sum(tiles) - 2 and stats[0]["rays_forwarded"] > 0


def test_round_loop_raises_past_its_bound():
    """A march that never finishes a ray (a bug the bound exists to catch) makes the loop raise, not spin."""
    def march(rays):
        return torch.ones(rays.shape[0], dtype=torch.int64), torch.zeros((rays.shape[0], 5))
    rays, tags = _rows(np.zeros((3, 3), F), np.ones((3, 3), F), 1.0, 0, 2)
    rays2, tags2 = _rows(np.zeros((0, 3), F), np.ones((0, 3), F), 1.0, 1, 2)
    with pytest.raises(RuntimeError, match="after 2 rounds"):
        D.raycast_rounds(D._LocalRouter(2), [march, march], [rays, rays2], [tags, tags2], 2, 2)
