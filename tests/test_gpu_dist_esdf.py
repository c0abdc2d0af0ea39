"""Tiled ESDF on ONE GPU: `world` virtual ranks in one process (taichislam_b200.distributed.run_local_esdf*), the
all-to-all replaced by slicing.  The tiled field, its gather, slice and routed queries must be bit-identical to one map
holding every tile (tslam_esdf_update2 full recompute); the spiral corridor carries one wave across a tile cut k times."""
import ctypes as C
import gc

import numpy as np
import pytest

import esdf_spiral as sp
from taichislam_b200 import _capi as capi
from util import as_dict_rows

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def release_maps():
    """Maps of several GB each live in reference cycles: collect before and after each case (test_gpu_dist_local.py)."""
    gc.collect()
    yield
    gc.collect()


def _global_map(**kw):
    from taichi_slam.mapping import DenseTSDF
    kw.setdefault("map_scale", [12.8, 12.8])
    return DenseTSDF(voxel_scale=0.05, is_global_map=True, max_submap_num=8, max_disp_particles=1024, **kw)


def _fused(world, balance, keep_submaps=False):
    """The scene of test_gpu_dist_local.py, fused by run_local_fusion; the submap maps are released afterwards unless
    kept (then returned too)."""
    from test_gpu_dist_local import _inputs, _integrate, _maps
    from taichislam_b200.distributed import LocalGroup, TiledGlobalMap, run_local_fusion, submap_owner
    d, K, poses = _inputs()
    grp = LocalGroup(world)
    subs, glos, tiled = [], [], []
    for r in range(world):
        sub, glo = _maps(K, False)
        _integrate(sub, glo, poses, d, False, only={s for s in poses if submap_owner(s, world) == r})
        subs.append(sub); glos.append(glo)
        tiled.append(TiledGlobalMap(glo, grp, r, world, balance=balance))
    run_local_fusion(tiled, subs)
    if keep_submaps:
        return tiled, subs
    del subs
    gc.collect()
    return tiled


def _single_map(tiled, **kw):
    """One map holding every tile: the union of the ranks' observed rows, scattered into a fresh global map."""
    parts = [t.m._h.gather(0) for t in tiled]
    ref = _global_map(**kw)
    ref._h.scatter(0, *(np.concatenate([p[c] for p in parts]) for c in range(4)))
    ref._h.esdf_update2(0, full=True)
    return ref


def _esdf_rows(handles):
    rows = [h.esdf_gather(0) for h in handles]
    return as_dict_rows(np.concatenate([r[0] for r in rows]), np.concatenate([r[1] for r in rows]))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _assert_same_answers(got, ref):
    for g, r in zip(got, ref):
        if g.dtype == np.float32:
            assert np.array_equal(_bits(g), _bits(r))
        else:
            assert np.array_equal(g, r)


def _seams(t, N=256):
    """Per axis, the block coordinates b whose tile differs from that of b + 1."""
    out = []
    for a in range(3):
        s = []
        for b in range(-N // 32, N // 32 - 1):
            c0, c1 = [0, 0, 0], [0, 0, 0]
            c0[a], c1[a] = b, b + 1
            if t.owner_of_block(*c0) != t.owner_of_block(*c1):
                s.append(b)
        out.append(s)
    return out


def _query_points(t, n_uniform, seed, N=256):
    """Uniform points over (a little beyond) the volume, points whose corner cube straddles a seam on 1, 2 and 3 axes,
    and non-finite / far points."""
    rng = np.random.default_rng(seed)
    h = N // 2 * sp.VS
    p = [rng.uniform(-h - 0.1, h + 0.1, size=(n_uniform, 3))]
    seams = _seams(t, N)
    for axes in ([0], [1], [2], [0, 1], [0, 2], [1, 2], [0, 1, 2]):
        if not all(seams[a] for a in axes):
            continue
        q = rng.uniform(-2.0, 2.0, size=(20000, 3))
        for a in axes:
            b = rng.choice(seams[a], size=len(q))
            q[:, a] = ((b + 1) * 16 - 1 + rng.uniform(0.0, 1.0, size=len(q))) * sp.VS  # low corner: last voxel below the cut
        p.append(q)
    p.append(np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1e30, 0, 0], [0, 0, -h - 1.0], [h, 0.0, 0.0]]))
    return np.concatenate(p).astype(np.float32)


def _slice_rows(xyz, val):
    rows = np.concatenate([xyz, val[:, None]], 1)
    return rows[np.lexsort(rows.T[::-1])]


@pytest.mark.parametrize("world,balance", [(2, True), (2, False), (4, True), (4, False), (8, True), (8, False)])
def test_tiled_esdf_equals_single_map(world, balance):
    from taichislam_b200.distributed import run_local_esdf, run_local_esdf_query
    tiled = _fused(world, balance)
    st = run_local_esdf(tiled)
    assert st["rounds"] >= 1 and st["blocks_sent"] > 0 and st["bytes_sent"] == st["blocks_sent"] * (8 + 4096 * 4)
    ref = _single_map(tiled)
    gi, ge = _esdf_rows([t.m._h for t in tiled])
    si, se = _esdf_rows([ref._h])
    assert len(si) > 10000 and np.array_equal(gi, si) and np.array_equal(_bits(ge), _bits(se))
    # queries: every rank asks its own points, answered by the owners
    pts = [_query_points(t, 1 << 20, 100 + r) for r, t in enumerate(tiled)]
    got = run_local_esdf_query(tiled, pts)
    n_seam_valid = 0
    for r, (p, g) in enumerate(zip(pts, got)):
        want = ref._h.esdf_query(p)
        _assert_same_answers(g, want)
        assert want[2][: 1 << 20].mean() > 0.01
        n_seam_valid += int(want[2][1 << 20:].sum())
    assert n_seam_valid > 100
    # the torch path answers the same
    import torch
    gt = run_local_esdf_query(tiled, [torch.from_numpy(p[:4096]).cuda() for p in pts])
    _assert_same_answers([a.cpu().numpy() for a in gt[0]], ref._h.esdf_query(pts[0][:4096]))
    # slice: the union of the ranks' parts is the single map's slice
    for k in np.quantile(si[:, 2], [0.1, 0.5, 0.9]).astype(int):
        z = float(k) * sp.VS
        parts = [t.m._h.esdf_slice(z)[1:] for t in tiled]
        n, sx, sv = ref._h.esdf_slice(z)
        got = _slice_rows(np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]))
        assert n == len(sx) > 0 and np.array_equal(_bits(got), _bits(_slice_rows(sx, sv)))
    # a rank-local ESDF (plain update: ghosts relaxed from their TSDF as if owned, no exchange) only bounds the exact
    # field - never nearer the surface; whether it differs depends on the scene (the spiral test shows that it can)
    for t in tiled:
        t.m._h.esdf_update2(0)
    li, le = _esdf_rows([t.m._h for t in tiled])
    assert np.array_equal(li, si)
    assert np.all(le[se > 0] >= se[se > 0]) and np.all(le[se < 0] <= se[se < 0]) and np.all(le[se == 0] == 0)
    # ... and after it the ghost corners read invalid again: seam points answered by their owner lose their answer
    seam = [p[1 << 20:] for p in pts]
    after = run_local_esdf_query(tiled, seam)
    before = [ref._h.esdf_query(s)[2] for s in seam]
    assert sum(int(a[2].sum()) for a in after) < sum(int(b.sum()) for b in before)


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_spiral_crosses_the_seam_k_times(oracle_lib, sign):
    from oracle.oracle import OracleTSDF
    from taichislam_b200.distributed import LocalGroup, TiledGlobalMap, run_local_esdf, run_local_esdf_query
    k = 4
    idx, t, w, occ = sp.spiral_rows(k, sign)
    grp = LocalGroup(2)
    tiled = [TiledGlobalMap(_global_map(max_ray_length=sp.MAX_RAY), grp, r, 2) for r in range(2)]
    for tm in tiled:
        tm.set_tiling(sp.SPIRAL_TILES, sp.SPIRAL_CUTS)
    own = np.array([tiled[0].owner_of_block(*b) for b in idx // 16])
    assert set(own) == {0, 1}
    for r, tm in enumerate(tiled):
        tm.m._h.scatter(0, idx[own == r], t[own == r], w[own == r], occ[own == r])
    st = run_local_esdf(tiled)
    assert st["rounds"] >= k + 1, st
    ref = _single_map(tiled, max_ray_length=sp.MAX_RAY)
    gi, ge = _esdf_rows([tm.m._h for tm in tiled])
    si, se = _esdf_rows([ref._h])
    o = OracleTSDF(map_scale=sp.MAP_SCALE, voxel_scale=sp.VS, max_ray_length=sp.MAX_RAY, is_global_map=True)
    o.scatter(0, idx, t, w, occ)
    o.esdf_update()
    oi, oe = as_dict_rows(*o.esdf_gather())
    assert len(gi) == len(idx)
    assert np.array_equal(gi, si) and np.array_equal(_bits(ge), _bits(se))
    assert np.array_equal(gi, oi) and np.array_equal(_bits(ge), _bits(oe))
    # without the exchange the wave never reaches the corridor beyond the first crossing
    for tm in tiled:
        tm.m._h.esdf_update2(0)
    li, le = _esdf_rows([tm.m._h for tm in tiled])
    assert np.array_equal(li, si) and np.count_nonzero(_bits(le) != _bits(se)) > len(idx) // 2
    assert np.all(sign * le >= sign * se)
    run_local_esdf(tiled)
    # queries along the corridor (corner cubes straddling the cut included)
    p = ((idx[:-1].astype(np.float32) + np.float32(0.5) * (idx[1:] - idx[:-1])) * np.float32(sp.VS)).astype(np.float32)
    got = run_local_esdf_query(tiled, [p, p[::-1].copy()])
    _assert_same_answers(got[0], ref._h.esdf_query(p))
    _assert_same_answers(got[1], ref._h.esdf_query(p[::-1].copy()))


def _key(bx, by, bz, s=0):
    return (s << 30) | ((bx + 512) << 20) | ((by + 512) << 10) | (bz + 512)


def test_tiled_esdf_state():
    import torch
    from taichislam_b200.distributed import _route, run_local_esdf, run_local_fusion
    tiled, subs = _fused(2, True, keep_submaps=True)
    h0 = tiled[0].m._h
    # begin .. end: both readers refuse
    run_local_esdf(tiled)
    for t in tiled:
        t.esdf_begin(0)
    with pytest.raises(capi.TslamError) as e:
        h0.esdf_query(np.zeros((4, 3), np.float32))
    assert e.value.code == capi.E_INVALID
    with pytest.raises(capi.TslamError):
        h0.esdf_slice(0.1)
    # unpacking a key that is not a ghost block of this rank: TSLAM_E_INVALID, nothing written
    rows_before = as_dict_rows(*h0.esdf_gather(0))
    gi = rows_before[0]
    bx, by, bz = (int(v) for v in np.floor_divide(gi[len(gi) // 2], 16))
    assert tiled[0].owner_of_block(bx, by, bz) == 0
    keys = torch.tensor([_key(bx, by, bz), _key(7, 7, 7)], dtype=torch.int64, device="cuda")
    esdf = torch.full((2, 4096), 123.0, dtype=torch.float32, device="cuda")
    rc = h0.L.tslam_esdf_ghost_unpack(h0.h, 2, capi.tptr(keys), capi.tptr(esdf), capi.stream_ptr())
    assert rc == capi.E_INVALID
    rows_after = as_dict_rows(*h0.esdf_gather(0))
    assert np.array_equal(rows_before[0], rows_after[0]) and np.array_equal(_bits(rows_before[1]), _bits(rows_after[1]))
    for t in tiled:
        t.esdf_end()
    h0.esdf_query(np.zeros((4, 3), np.float32))  # readable again
    # a TSDF halo import invalidates the tiled field; so does a later fusion
    packed = [t.halo_pack() for t in tiled]
    routed, _ = _route([p[1] for p in packed], [p[0] for p in packed], 2)
    for t, bufs in zip(tiled, routed):
        t.halo_unpack(bufs)
    with pytest.raises(capi.TslamError):
        h0.esdf_query(np.zeros((4, 3), np.float32))
    run_local_esdf(tiled)
    h0.esdf_query(np.zeros((4, 3), np.float32))
    run_local_fusion(tiled, subs)
    with pytest.raises(capi.TslamError):
        h0.esdf_query(np.zeros((4, 3), np.float32))
    st = run_local_esdf(tiled)  # (runs the TSDF halo exchange the fusion made stale)
    assert st["rounds"] >= 1
    h0.esdf_query(np.zeros((4, 3), np.float32))
    # after end, the unpack / relax / pack calls refuse
    assert h0.L.tslam_esdf_tiled_relax(h0.h, None, capi.stream_ptr()) == capi.E_INVALID
    assert h0.L.tslam_esdf_tiled_end(h0.h) == capi.E_INVALID


def test_tiled_esdf_argument_checks():
    from taichislam_b200.distributed import run_local_esdf
    tiled = _fused(2, True)
    run_local_esdf(tiled)
    h = tiled[0].m._h
    L, st = h.L, capi.stream_ptr()
    tiles = (C.c_int32 * 3)(*tiled[0].tiles)
    one = np.zeros(4, np.float32)
    assert L.tslam_tiling_owner_points(h.h, tiles, 2, -1, capi.np_ptr(one), capi.np_ptr(one), st) == capi.E_INVALID
    assert L.tslam_tiling_owner_points(h.h, tiles, 2, 1, None, capi.np_ptr(one), st) == capi.E_INVALID
    assert L.tslam_tiling_owner_points(h.h, tiles, 3, 0, None, None, st) == capi.E_INVALID   # tiling does not match the world
    assert L.tslam_esdf_ghost_unpack(h.h, -1, None, None, st) == capi.E_INVALID
    assert L.tslam_esdf_ghost_unpack(h.h, 1, None, None, st) == capi.E_INVALID
    assert L.tslam_esdf_halo_count(h.h, tiles, 0, 2, None, st) == capi.E_INVALID
    cnt = np.zeros(2, np.int32)
    assert L.tslam_esdf_halo_count(h.h, tiles, 0, 2, capi.np_ptr(cnt), st) == capi.E_INVALID  # no tiled ESDF in progress
    assert L.tslam_esdf_halo_pack(h.h, tiles, 0, 2, capi.np_ptr(cnt), 4, None, None, st) == capi.E_INVALID
