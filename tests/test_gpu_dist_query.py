"""Planner queries on the tiled global map, on ONE GPU: `world` virtual ranks in one process
(taichislam_b200.distributed.run_local_raycast / _query_points / _near_occupy, LocalGroupMap), the all-to-all replaced
by slicing.  Every answer must be bit-identical to the same call on one DenseTSDF holding the union of the tiles; the
raycast hands rays across tile seams in at most tx+ty+tz-2 rounds; TopoGraphGen on the tiled map builds the graph of
the single map."""
import ctypes as C
import gc

import numpy as np
import pytest

from taichislam_b200 import _capi as capi
from topo_world import START_A, two_rooms

pytestmark = pytest.mark.gpu

F = np.float32
VS = 0.05
H = 128 * VS  # half extent of the 256^3 volume


@pytest.fixture(autouse=True)
def release_maps():
    """Maps of several GB each live in reference cycles: collect before and after each case (test_gpu_dist_local.py)."""
    gc.collect()
    yield
    gc.collect()


def _global_map():
    from taichi_slam.mapping import DenseTSDF
    return DenseTSDF(map_scale=[12.8, 12.8], voxel_scale=VS, is_global_map=True, max_submap_num=8, max_disp_particles=1024)


def _exchange_halo(tiled):
    from taichislam_b200.distributed import _route
    packed = [t.halo_pack() for t in tiled]
    routed, _ = _route([p[1] for p in packed], [p[0] for p in packed], len(tiled))
    for t, bufs in zip(tiled, routed):
        t.halo_unpack(bufs)


def _rooms(world, balance):
    """two_rooms scattered into the ranks by block owner (default cuts or cuts balanced on its blocks), halo exchanged."""
    from taichislam_b200.distributed import LocalGroup, TiledGlobalMap, balanced_tiling
    idx, t, w, occ = two_rooms()
    grp = LocalGroup(world)
    tiled = [TiledGlobalMap(_global_map(), grp, r, world, balance=False) for r in range(world)]
    if balance:
        hist = np.zeros((3, 1024), np.int64)
        for a in range(3):
            np.add.at(hist[a], (idx[:, a] >> 4) + 512, 1)
        tiles, cuts = balanced_tiling(hist, world)
        for tm in tiled:
            tm.set_tiling(tiles, cuts)
    own = np.array([tiled[0].owner_of_block(*b) for b in idx >> 4])
    for r, tm in enumerate(tiled):
        tm.m._h.scatter(0, idx[own == r], t[own == r], w[own == r], occ[own == r])
    _exchange_halo(tiled)
    return tiled


def _scene(kind, world, balance):
    if kind == "rooms":
        return _rooms(world, balance)
    from test_gpu_dist_esdf import _fused
    tiled = _fused(world, balance)
    _exchange_halo(tiled)
    return tiled


def _single_map(tiled):
    """One map holding every tile: the union of the ranks' observed rows, scattered into a fresh global map."""
    parts = [t.m._h.gather(0) for t in tiled]
    ref = _global_map()
    ref._h.scatter(0, *(np.concatenate([p[c] for p in parts]) for c in range(4)))
    return ref


def _bits(a):
    return np.ascontiguousarray(a, F).view(np.uint32)


def _same_rays(got, want):
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(_bits(got[1]), _bits(want[1])) and np.array_equal(_bits(got[2]), _bits(want[2]))


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


def _free_cells(ref, n, rng):
    """Positions of observed free voxels (TSDF >= 1.8 vs) of the single map, jittered within the voxel."""
    idx, t, _, _ = ref._h.gather(0)
    free = idx[t >= F(1.8 * VS)]
    pick = free[rng.integers(0, len(free), size=n)]
    return ((pick + rng.uniform(-0.45, 0.45, size=(n, 3))) * VS).astype(F)


def _unit(rng, n):
    d = rng.normal(size=(n, 3)).astype(F)
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(F)


def _seam_points(t, rng, n):
    """Points next to the seams: on 1, 2 or 3 cut planes at once (diagonal tiles), on both sides and on the .5 tie."""
    seams = _seams(t)
    out = []
    for axes in ([0], [1], [2], [0, 1], [0, 2], [1, 2], [0, 1, 2]):
        if not all(seams[a] for a in axes):
            continue
        q = rng.uniform(-2.5, 2.5, size=(n, 3))
        for a in axes:
            b = rng.choice(seams[a], size=n)
            q[:, a] = ((b + 1) * 16 + rng.choice([-1.5, -1.0, -0.5, 0.0, 0.5], size=n)) * VS  # cells either side and the tie
        out.append(q)
    return np.concatenate(out).astype(F)


def _ray_cases(t, ref, rng, n):
    """(pos, dir) of rank r's raycast: origins in observed free space and across the volume, rays lying in seam planes
    and crossing them axis-aligned, rays from the .5 tie, from outside the volume and with non-finite values."""
    pos = [_free_cells(ref, n // 2, rng), rng.uniform(-H, H, size=(n // 4, 3)).astype(F)]
    dir = [_unit(rng, n // 2), _unit(rng, n // 4)]
    sp = _seam_points(t, rng, 512)
    ax = np.zeros((len(sp), 3), F)
    ax[np.arange(len(sp)), rng.integers(0, 3, size=len(sp))] = rng.choice([-1.0, 1.0], size=len(sp))
    pos += [sp, sp]
    dir += [ax, _unit(rng, len(sp))]
    bad_p = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0.1, 0.1, 0.1], [0.1, 0.1, 0.1], [0.1, 0.1, 0.1], [H + 1, 0, 0], [-H - 1, 0.2, 0],
                      [H - 0.01, 0, 0], [0.1, 0.1, 0.1]], F)
    bad_d = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 0], [np.nan, 0, 0], [np.inf, 0, 0], [-1, 0, 0], [1, 0, 0], [1, 0, 0], [0, -np.inf, 1]], F)
    pos.append(bad_p)
    dir.append(bad_d)
    return np.concatenate(pos).astype(F), np.concatenate(dir).astype(F)


@pytest.mark.parametrize("kind", ["fused", "rooms"])
@pytest.mark.parametrize("world,balance", [(2, True), (2, False), (4, True), (4, False), (8, True), (8, False)])
def test_tiled_queries_equal_single_map(kind, world, balance):
    from taichislam_b200.distributed import run_local_near_occupy, run_local_query_points, run_local_raycast
    tiled = _scene(kind, world, balance)
    ref = _single_map(tiled)
    bound = sum(tiled[0].tiles) - 2
    rng = np.random.default_rng(world * 2 + balance)
    # raycast: 2^16 rays per rank, 4 m (several tiles at world 8), plus the edge cases; then short and empty lengths
    cases = [_ray_cases(t, ref, rng, 1 << 16) for t in tiled]
    got = run_local_raycast(tiled, [(p, d, 4.0) for p, d in cases])
    st = tiled[0].last_query
    assert 1 <= st["rounds"] <= bound and st["rays_forwarded"] > 0, st
    n_cross = 0
    for (p, d), g in zip(cases, got):
        want = ref.raycast(p, d, 4.0)
        _same_rays(g, want)
        n_cross += int((want[2] > 0.5).sum())
    assert n_cross > 200
    for md in (0.0, 0.03, 0.05, 0.26):
        got = run_local_raycast(tiled, [(p[:4096], d[:4096], md) for p, d in cases])
        for (p, d), g in zip(cases, got):
            _same_rays(g, ref.raycast(p[:4096], d[:4096], md))
        assert tiled[0].last_query["rounds"] <= bound
    # is_pos_occupy / is_pos_unobserved
    pts = [np.concatenate([rng.uniform(-H - 0.2, H + 0.2, size=(1 << 16, 3)).astype(F), _seam_points(t, rng, 2000), cases[0][0][: 1 << 12],
                           np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1e30, 0, 0]], F)]) for t in tiled]
    got = run_local_query_points(tiled, pts)
    for p, (occ, un) in zip(pts, got):
        assert np.array_equal(occ, ref.is_pos_occupy(p)) and np.array_equal(un, ref.is_pos_unobserved(p))
        assert (~un).sum() > 100 and (~occ).sum() > 100
    # is_near_pos_occupy next to seams, diagonal tiles included
    near = [np.concatenate([_seam_points(t, rng, 1500), cases[0][0][:2000]]) for t in tiled]
    for voxel in (0, 1, 3, 16):
        got = run_local_near_occupy(tiled, near, voxel)
        for p, g in zip(near, got):
            want = ref.is_near_pos_occupy(p, voxel)
            assert np.array_equal(g, want)
            if voxel == 3:
                assert 0 < want.sum() < len(want)


def test_diagonal_ray_rounds_and_rank_local_gap():
    """World 8, default cuts at 0 on every axis: a ray through the corridor that crosses the z, then y, then x cut
    takes 3 rounds asked from tile (0,0,0) and 4 = tx+ty+tz-2 asked from tile (1,1,1).  The rank-local DenseTSDF.raycast
    on the asking rank reports a wall at the seam instead."""
    from taichislam_b200.distributed import run_local_raycast
    tiled = _rooms(8, False)
    ref = _single_map(tiled)
    assert tiled[0].tiles == (2, 2, 2) and _seams(tiled[0]) == [[-1], [-1], [-1]]
    p = np.array([[-0.3, -0.2, -0.1]], F)
    d = np.array([[1, 1, 1]], F) / F(np.sqrt(3))
    want = ref.raycast(p, d, 0.9)
    assert not want[0][0] and want[2][0] > 0.75
    for asker, rounds in ((0, 3), (7, 4)):
        batches = [(p, d, 0.9) if r == asker else (np.zeros((0, 3), F), np.zeros((0, 3), F), 0.9) for r in range(8)]
        got = run_local_raycast(tiled, batches)
        _same_rays(got[asker], want)
        assert tiled[0].last_query == dict(rounds=rounds, rays_forwarded=rounds)
    # without the hand-over: the rank holding the start reads the next tile (absent or ghost) as TSDF 0 -> a hit there
    local = tiled[0].m.raycast(p, d, 0.9)
    assert local[0][0] and local[2][0] < want[2][0]
    # seam-crossing rays of the uniform set differ in bulk on every rank
    rng = np.random.default_rng(5)
    q, e = _free_cells(ref, 4096, rng), _unit(rng, 4096)
    w = ref.raycast(q, e, 3.0)
    own = np.array([tiled[0].owner_of_block(*c) for c in np.floor(q / VS + 0.5).astype(int) >> 4])
    differ = sum(int(np.count_nonzero(tm.m.raycast(q[own == r], e[own == r], 3.0)[2] != w[2][own == r])) for r, tm in enumerate(tiled))
    assert differ > 200


def test_near_occupancy_voxel_limit_and_halo_refresh():
    from taichislam_b200.distributed import LocalGroupMap, run_local_fusion, run_local_near_occupy
    from test_gpu_dist_esdf import _fused
    tiled, subs = _fused(4, True, keep_submaps=True)
    with pytest.raises(ValueError):
        run_local_near_occupy(tiled, [np.zeros((1, 3), F)] * 4, 17)
    with pytest.raises(ValueError):
        LocalGroupMap(tiled).is_near_pos_occupy(np.zeros(3, F), -1)
    h = tiled[0].m._h
    x = np.zeros(3, np.float32)
    out = np.zeros(1, np.uint8)
    for v in (17, -1):
        assert h.L.tslam_tsdf_query_near_occupy_tiled(h.h, 0, 1, capi.np_ptr(x), v, capi.np_ptr(out), capi.stream_ptr()) == capi.E_INVALID
    tiles = (C.c_int32 * 3)(*tiled[0].tiles)
    assert h.L.tslam_tiling_owner_cells(h.h, tiles, 3, 0, None, None, capi.stream_ptr()) == capi.E_INVALID   # tiling != world
    assert h.L.tslam_tiling_owner_cells(h.h, tiles, 4, -1, None, None, capi.stream_ptr()) == capi.E_INVALID
    assert h.L.tslam_tsdf_raycast_tiled(h.h, tiles, 4, 4, 0, 0, None, None, None, None, None, None, capi.stream_ptr()) == capi.E_INVALID  # rank
    assert h.L.tslam_tsdf_raycast_tiled(h.h, tiles, 0, 4, 0, 1, None, None, None, None, None, None, capi.stream_ptr()) == capi.E_INVALID
    rng = np.random.default_rng(3)
    pts = [_seam_points(t, rng, 1000) for t in tiled]
    assert not any(t._halo_current for t in tiled)
    first = run_local_near_occupy(tiled, pts, 2)             # exchanges the halo the fusion made stale
    assert all(t._halo_current for t in tiled)
    ref = _single_map(tiled)
    assert all(np.array_equal(g, ref.is_near_pos_occupy(p, 2)) for p, g in zip(pts, first))
    # a new fusion rebuilds the tiles without ghosts: the next query exchanges the halo again and is still exact
    run_local_fusion(tiled, subs)
    assert not any(t._halo_current for t in tiled)
    again = run_local_near_occupy(tiled, pts, 2)
    ref2 = _single_map(tiled)
    assert all(np.array_equal(g, ref2.is_near_pos_occupy(p, 2)) for p, g in zip(pts, again))
    assert all(t._halo_current for t in tiled)


def _graph(topo):
    nf, ne = topo.num_facelets[None], topo.edge_num[None]
    nodes = [(n["start"], n["end"], n["master_idx"], np.asarray(n["center"], F).tobytes()) for n in topo.nodes]
    fr = [(k, v["is_valid"], np.asarray(v["projected_center"], F).tobytes()) for k, v in sorted(topo.frontiers.items())]
    arrays = [topo.f_normal.a[:nf], topo.f_center.a[:nf], topo.f_v0.a[:nf], topo.f_edge1.a[:nf], topo.f_edge2.a[:nf],
              topo.f_is_frontier.a[:nf], topo.f_poly.a[:nf], topo.edges.to_numpy()[:ne]]
    return topo.num_nodes[None], nf, topo.num_frontiers[None], nodes, fr, [np.ascontiguousarray(a).tobytes() for a in arrays]


@pytest.mark.parametrize("world", [4, 8])
def test_topo_graph_on_tiled_map_equals_single_map(world):
    from taichi_slam.mapping import TopoGraphGen
    from taichislam_b200.distributed import LocalGroupMap
    tiled = _rooms(world, False)
    ref = _single_map(tiled)
    single = TopoGraphGen(ref, coll_det_num=64, max_raycast_dist=2.5)
    n = single.generate_topo_graph(START_A, max_nodes=12)
    local = LocalGroupMap(tiled, asker=0)
    topo = TopoGraphGen(local, coll_det_num=64, max_raycast_dist=2.5)
    assert topo.generate_topo_graph(START_A, max_nodes=12) == n >= 2
    assert _graph(topo) == _graph(single)
    # the graph reaches room B across the x cut
    assert max(nd["center"][0] for nd in topo.nodes) > 0.45
