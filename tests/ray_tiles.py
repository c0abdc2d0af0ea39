"""numpy f32 statement of the planner raycast's samples and of the tiling (raycast_sample / raycast_steps, which
k_raycast and k_tsdf_raycast_tiled share, ts_query_cell, tile_coord / tile_owner of csrc/tslam_dist.cu): sample j of
a ray is len = f32(j) * vs, x = dir * len + pos (two roundings: the library builds with -fmad=false), cell =
(int)roundf(x / vs) with roundf half away from zero and the float -> int conversion of the GPU (NaN -> 0,
saturating).  Used for the round bound of the hand-over (test_tiled_raycast_cpu.py) and as a stand-in march for the
host round loop under gloo."""
import numpy as np

F = np.float32


def roundf(u):
    """C roundf: nearest integer, ties away from zero (u - trunc(u) is exact in f32)."""
    u = np.asarray(u, F)
    t = np.trunc(u)
    with np.errstate(invalid="ignore"):
        return (t + np.where(np.abs(u - t) >= F(0.5), np.sign(u), F(0.0))).astype(F)


def f2i(v):
    """(int) of an integral f32 on the GPU (cvt.rzi.s32.f32): NaN -> 0, out of range saturates."""
    v = np.asarray(v, np.float64)
    return np.where(np.isnan(v), 0.0, np.clip(v, -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)


def cells(x, vs):
    with np.errstate(invalid="ignore", over="ignore"):
        return f2i(roundf(np.asarray(x, F) / F(vs)))


def samples(pos, dir, j, vs):
    """(x f32[n,3], len f32[n]) of sample j[n] of rays pos / dir f32[n,3]."""
    ln = (np.asarray(j).astype(F) * F(vs)).astype(F)
    with np.errstate(invalid="ignore", over="ignore"):
        x = (np.asarray(dir, F) * ln[:, None]).astype(F) + np.asarray(pos, F)
    return x.astype(F), ln


def in_bounds(c, N, Nz):
    lo = np.array([-(N // 2), -(N // 2), -(Nz // 2)])
    hi = np.array([N - N // 2, N - N // 2, Nz - Nz // 2])
    return np.all((c >= lo) & (c < hi), axis=-1)


def default_cuts(N, Nz, tiles):
    """fill_tiling's equal slices: block-coordinate cuts per axis."""
    out = []
    for a, (n, t) in enumerate(zip((N, N, Nz), tiles)):
        lo, hi = (-(n // 2)) >> 4, (n - n // 2 - 1) >> 4
        ext = (hi - lo + 1 + t - 1) // t
        out.append([lo + k * ext for k in range(t + 1)])
    return out


def tile_coords(cuts, tiles, b):
    """tile_coord per axis of block coordinates b int[...,3] -> int[...,3] (blocks beyond the cuts: the end tiles)."""
    return np.stack([np.searchsorted(np.asarray(cuts[a][1:tiles[a]]), b[..., a], side="right") for a in range(3)], -1)


def tile_owner(cuts, tiles, b):
    tc = tile_coords(cuts, tiles, b)
    return (tc[..., 0] * tiles[1] + tc[..., 1]) * tiles[2] + tc[..., 2]


def tile_runs(pos, dir, max_dist, vs, N, Nz, cuts, tiles):
    """Per ray, the tile coordinates int[k,3] of its in-volume samples in march order, up to the first sample outside
    the volume or the last step (a hit would only end it earlier)."""
    pos, dir = np.asarray(pos, F), np.asarray(dir, F)
    with np.errstate(invalid="ignore", over="ignore"):
        steps = f2i(np.trunc(F(max_dist) / F(vs)))
    out = []
    for i in range(len(pos)):
        j = np.arange(max(int(steps), 0))
        x, _ = samples(np.broadcast_to(pos[i], (len(j), 3)), np.broadcast_to(dir[i], (len(j), 3)), j, vs)
        c = cells(x, vs)
        inb = in_bounds(c, N, Nz)
        stop = int(np.argmin(inb)) if not inb.all() else len(j)
        out.append(tile_coords(cuts, tiles, c[:stop] >> 4))
    return out


def march_stand_in(occupied, vs, N, Nz, cuts, tiles, rank):
    """k_tsdf_raycast_tiled in numpy over an occupancy predicate occupied(cells int[n,3]) -> bool[n], for rays
    f32[n,8] (a torch CPU tensor; the next sample j is written back) -> (dest int64[n], answer f32[n,5])."""
    import torch

    def march(rays_t):
        r = rays_t.numpy()
        n = len(r)
        j = r[:, 7].view(np.int32).astype(np.int64)
        with np.errstate(invalid="ignore", over="ignore"):
            steps = f2i(np.trunc(r[:, 6] / F(vs)))
        dest = np.full(n, -1, np.int64)
        ans = np.zeros((n, 5), F)
        live = j < steps
        while live.any():
            i = np.nonzero(live)[0]
            x, ln = samples(r[i, :3], r[i, 3:6], j[i], vs)
            ans[i, 1:4], ans[i, 4] = x, ln
            c = cells(x, vs)
            inb = in_bounds(c, N, Nz)
            own = tile_owner(cuts, tiles, c >> 4)
            away = inb & (own != rank)
            hit = ~inb | (~away & occupied(c))
            dest[i[away]] = own[away]
            ans[i[hit], 0] = 1.0
            live[i[away | hit]] = False
            j[i[~(away | hit)]] += 1
            live &= j < steps
        r[:, 7] = j.astype(np.int32).view(F)
        return torch.from_numpy(dest), torch.from_numpy(ans)

    return march
