"""Incremental fusion of the tiled global map on ONE GPU (TiledGlobalMap.update_fused_submaps' phases driven by
taichislam_b200.distributed.run_local_update_fused_submaps over `world` virtual ranks): after every update the union
of the ranks' tiles equals, bit for bit, the numpy reference of the fusion contract (tests/fuse_update_reference.py)
and a single-map tslam_tsdf_fuse_update of all ranks' submaps, whatever the world size, cuts and history.  Map sizes
and the collector fixture are those of tests/test_gpu_dist_local.py (world 8 takes about 50 GB)."""
import gc

import numpy as np
import pytest

from fuse_update_reference import fuse_reference, same_rows, same_values
from taichislam_b200 import _capi as capi
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu

NSUB = 8  # submap table (max_submap_num) of these maps


@pytest.fixture(autouse=True)
def release_maps():
    gc.collect()
    yield
    gc.collect()


def _poses():
    # spread over a flat volume: every sphere submap straddles the seams of a 2, 4 or 8 rank tiling
    return {s: (rot_xyz(0.05 * s, 0.03 * s, 0.7 * s + 0.1), np.array([2.2 * (s % 3) - 2.0, 2.0 * (s // 3) - 1.5, 0.1 * (s % 2)]))
            for s in range(NSUB)}


K = [syn.FX / 2, 0, syn.CX / 2, 0, syn.FY / 2, syn.CY / 2, 0, 0, 1]
DEPTH = syn.scene_sphere(2.5, 240, 320)


def _maps(tex, max_blocks=0):
    from taichi_slam.mapping import DenseTSDF
    sub = DenseTSDF(map_scale=[6.4, 6.4], voxel_scale=0.05, max_ray_length=3.0, max_submap_num=NSUB, max_disp_particles=1024,
                    max_image_pixels=240 * 320, texture_enabled=tex)
    sub.set_dep_camera_intrinsic(K)
    glo = DenseTSDF(map_scale=[12.8, 12.8], voxel_scale=0.05, is_global_map=True, max_submap_num=NSUB, max_disp_particles=1024,
                    texture_enabled=tex, max_blocks=max_blocks)
    return sub, glo


def _frame(sub, s, tex, T=(0.0, 0.0, 0.0), seed=0):
    img = syn.texture_gradient(4 + seed, 240, 320) if tex else np.array([])
    sub.active_submap_id[None] = s
    sub.set_base_pose_submap(s, np.eye(3), np.zeros(3))
    sub.recast_depth_to_map(np.eye(3), np.asarray(T, np.float64), DEPTH, img)
    sub._flush()


class World:
    """`world` virtual ranks: rank r's submap collection holds the submaps it owns (s % world == r, or `owner`)."""

    def __init__(self, world, tex=False, balance=True, present=range(6), owner=None, max_blocks=None):
        from taichislam_b200.distributed import LocalGroup, TiledGlobalMap
        self.world, self.tex = world, tex
        self.owner = owner or (lambda s: s % world)
        self.poses = _poses()
        grp = LocalGroup(world)
        self.subs, self.glos, self.tiled = [], [], []
        for r in range(world):
            sub, glo = _maps(tex, (max_blocks or {}).get(r, 0))
            self.subs.append(sub)
            self.glos.append(glo)
            self.tiled.append(TiledGlobalMap(glo, grp, r, world, tiles=None if balance else _factor(world), balance=balance))
        self.present = []
        for s in present:
            self.add(s)
        self.set_poses()

    def add(self, s, T=(0.0, 0.0, 0.0), seed=0):
        _frame(self.subs[self.owner(s)], s, self.tex, T, seed)
        if s not in self.present:
            self.present.append(s)

    def set_poses(self):
        for glo in self.glos:
            for s, (R, T) in self.poses.items():
                glo.set_base_pose_submap(s, R, T)

    def update(self, include=None, tolerance=0.0, full=False):
        from taichislam_b200.distributed import run_local_update_fused_submaps
        self.set_poses()
        return run_local_update_fused_submaps(self.tiled, self.subs, include=include, tolerance=tolerance, full=full)

    def union(self):
        """gather() of every rank, concatenated; each rank holds only blocks of its own tile."""
        parts = []
        for r, (t, glo) in enumerate(zip(self.tiled, self.glos)):
            g = glo._h.gather(0, color=self.tex)
            if g[0].shape[0]:
                assert {t.owner_of_block(*b) for b in np.unique(np.floor_divide(g[0], 16), axis=0)} == {r}
            parts.append(g)
        return tuple(np.concatenate([p[c] for p in parts]) for c in range(len(parts[0])))

    def gathered(self, s):
        return self.subs[self.owner(s)]._h.gather(s, color=self.tex)

    def reference(self, include=None):
        parts = []
        for s in self.present:
            if include is not None and not include[s]:
                continue
            g = self.gathered(s)
            R, T = self.poses[s]
            p = dict(idx=g[0], tsdf=g[1], w=g[2], occ=g[3], R=np.float32(R), T=np.float32(T))
            if self.tex:
                p["color"] = g[4]
            parts.append(p)
        N = self.glos[0]._h.N
        return fuse_reference(parts, N, self.glos[0]._h.Nz, np.float32(0.05))

    def single(self, include=None, keep=False):
        """One collection holding every rank's submaps (scattered from their gather) fused into one global map."""
        sub, glo = _maps(self.tex)
        for s in self.present:
            sub._h.scatter(s, *self.gathered(s))
        for s, (R, T) in self.poses.items():
            glo.set_base_pose_submap(s, R, T)
        st = glo._h.fuse_update(sub._h, include=include)
        assert st["full"]
        rows = glo._h.gather(0, color=self.tex)
        return (rows, glo) if keep else rows


def _factor(world):
    from taichislam_b200.distributed import factor_tiles
    return factor_tiles(world)


def same(a, b):
    a, b = as_dict_rows(*a), as_dict_rows(*b)
    return len(a) == len(b) and all(same_values(x, y) for x, y in zip(a, b))


def check(w, include=None):
    u = w.union()
    assert same_rows(u, w.reference(include))
    assert same(u, w.single(include))
    gc.collect()  # (the single map's DenseTSDFs)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world,balance,tex", [(2, True, False), (4, True, False), (8, True, False), (4, False, False), (2, False, False),
                                               (2, True, True)])
def test_first_update_is_the_single_map_bit_for_bit(world, balance, tex):
    w = World(world, tex, balance)
    st = w.update()
    assert st["full"] and st["reason"] == "first call" and st["added"] == 6 and st["voxels_skipped"] == 0
    assert st["foreign_blocks_sent"] > 0 and st["foreign_blocks_received"] == st["foreign_blocks_sent"]
    assert st["bytes_sent"] == st["foreign_blocks_sent"] * 8 * (1 + (6 if tex else 3) * 4096)
    assert (w.tiled[0].cuts is not None) == balance
    ref = w.reference()
    assert st["voxels_splatted"] == ref["splatted"] > 0
    check(w)


def test_history_independence_over_a_seeded_sequence():
    rng = np.random.default_rng(11)
    w = World(4)
    include = np.zeros(NSUB, bool)
    include[w.present] = True
    assert w.update(include)["reason"] == "first call"
    check(w, include)
    jit = lambda s, j: (rot_xyz(0.05 * s + j, 0.03 * s, 0.7 * s + 0.1 - j), _poses()[s][1] + np.array([j, -j, 0.5 * j]))
    for step in ["move1", "move2", "exclude", "include", "new_submap", "content_excluded", "scatter", "content", "full"]:
        expect, kw = "incremental", {}
        if step == "move1":
            s = int(rng.choice(np.flatnonzero(include)))
            w.poses[s] = jit(s, float(rng.uniform(0.01, 0.05)))
        elif step == "move2":  # two submaps of different ranks
            a = int(rng.choice(np.flatnonzero(include)))
            b = int(rng.choice([s for s in np.flatnonzero(include) if w.owner(s) != w.owner(a)]))
            for s in (a, b):
                w.poses[s] = jit(s, float(rng.uniform(0.01, 0.05)))
        elif step == "exclude":
            include[int(rng.choice(np.flatnonzero(include)))] = False
        elif step == "include":
            include[int(rng.choice([s for s in w.present if not include[s]]))] = True
        elif step == "new_submap":
            w.add(6)
            include[6] = True
        elif step == "content_excluded":
            s = int(rng.choice(np.flatnonzero(include)))
            include[s] = False
            st = w.update(include)
            assert st["reason"] == "incremental" and st["removed"] == 1
            w.add(s, T=(0.05, 0.0, 0.0), seed=1)  # not fused now: nothing to subtract
        elif step == "scatter":  # a remote-style load into one rank's collection
            g = w.gathered(0)
            w.subs[w.owner(7)]._h.scatter(7, *g)
            w.present.append(7)
            include[7] = True
        elif step == "content":
            s = int(rng.choice(np.flatnonzero(include)))
            w.add(s, T=(0.0, 0.02, 0.0), seed=2)  # its old content is gone: a full update on every rank
            expect = "content changed"
        elif step == "full":
            kw, expect = dict(full=True), "full requested"
        st = w.update(include, **kw)
        assert st["reason"] == expect, (step, st)
        if step in ("move1", "move2"):
            assert st["moved"] == (1 if step == "move1" else 2) and st["foreign_blocks_sent"] > 0, (step, st)
        check(w, include)


def test_halo_and_tiled_esdf_do_not_force_a_full_update():
    from taichi_slam.mapping import MarchingCubeMesher
    from taichislam_b200.distributed import balanced_tiling, run_local_esdf, run_local_mesh
    w = World(4)
    w.update()
    meshers = [MarchingCubeMesher(g, 400000, tsdf_surface_thres=0.25) for g in w.glos]
    run_local_mesh(w.tiled, meshers)
    run_local_esdf(w.tiled)
    w.poses[1] = (w.poses[1][0], w.poses[1][1] + np.array([0.03, 0.0, 0.0]))
    st = w.update()
    assert st["reason"] == "incremental" and st["moved"] == 1
    check(w)
    # any other write of a rank's global map does force one
    w.glos[2]._h.scatter(0, np.zeros((1, 3), np.int32), np.zeros(1, np.float32), np.ones(1, np.float32), np.zeros(1, np.int8))
    st = w.update()
    assert st["reason"] == "destination written" and st["full"]
    check(w)
    # and so do new cuts
    t0 = w.tiled[0]
    cuts = [list(c) for c in t0.cuts]
    a = int(np.argmax([len(c) for c in cuts]))
    cuts[a][1] += 1
    for t in w.tiled:
        t.set_tiling(t0.tiles, cuts)
    st = w.update()
    assert st["reason"] == "tile cuts changed"
    check(w)
    assert w.update()["reason"] == "incremental"


def test_mesh_and_esdf_after_an_incremental_update_match_the_single_map():
    from taichi_slam.mapping import MarchingCubeMesher
    from taichislam_b200.distributed import run_local_esdf, run_local_mesh
    w = World(4)
    w.update()
    w.poses[4] = (rot_xyz(0.0, 0.0, 0.3) @ w.poses[4][0], w.poses[4][1] + np.array([0.0, 0.2, 0.0]))
    st = w.update()
    assert st["reason"] == "incremental" and st["moved"] == 1
    meshers = [MarchingCubeMesher(g, 400000, tsdf_surface_thres=0.25) for g in w.glos]
    mv, mn, counts = run_local_mesh(w.tiled, meshers)
    rows, glo = w.single(keep=True)
    ref = MarchingCubeMesher(glo, 400000, tsdf_surface_thres=0.25)
    ref.generate_mesh(1)
    n = int(ref.num_facelets[None])
    assert n > 1000 and sum(counts) == n and min(counts) > 0

    def tris(v, nrm):
        t = np.concatenate([np.ascontiguousarray(v, np.float32).reshape(-1, 9), np.ascontiguousarray(nrm, np.float32).reshape(-1, 9)], 1)
        t = t.view(np.int32)
        return t[np.lexsort(t.T[::-1])]

    assert np.array_equal(tris(mv.cpu().numpy(), mn.cpu().numpy()),
                          tris(ref.mesh_vertices.to_numpy()[:3 * n], ref.mesh_normals.to_numpy()[:3 * n]))
    run_local_esdf(w.tiled)
    glo._h.esdf_update2(0, full=True)
    parts = [g._h.esdf_gather(0) for g in w.glos]
    gi, ge = as_dict_rows(np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]))
    si, se = as_dict_rows(*glo._h.esdf_gather(0))
    assert np.array_equal(gi, si) and same_values(ge, se)


def test_refusals():
    import torch
    from taichislam_b200.distributed import merge_fuse_plans
    w = World(2, present=range(4))
    w.update()
    before = w.union()
    # include that differs between ranks: refused, nothing written, the next update is incremental
    inc = np.ones(NSUB, bool)
    rows = [t.update_plan(s, inc if r == 0 else ~inc) for r, (t, s) in enumerate(zip(w.tiled, w.subs))]
    with pytest.raises(ValueError, match="include differs"):
        merge_fuse_plans(np.stack(rows))
    for t, s in zip(w.tiled, w.subs):
        t.update_finish(s, False)
    st = w.update()
    assert st["reason"] == "incremental" and st["added"] == 0 and st["blocks_committed"] == 0
    assert same(w.union(), before)
    # phases out of order
    h, src = w.glos[0]._h, w.subs[0]._h
    rows0 = torch.zeros((0, 1 + 3 * 4096), dtype=torch.int64, device="cuda")
    for call in (lambda: h.fuse_update_tiled_splat(src, 0), lambda: h.fuse_update_tiled_pack(w.tiled[0].tiles, 0, 2),
                 lambda: h.fuse_update_tiled_unpack(rows0), lambda: h.fuse_update_tiled_finish(src, True)):
        with pytest.raises(capi.TslamError) as e:
            call()
        assert e.value.code == capi.E_INVALID
    w.tiled[0].update_plan(w.subs[0])
    for call in (lambda: h.fuse_update_tiled_pack(w.tiled[0].tiles, 0, 2), lambda: h.fuse_update_tiled_unpack(rows0),
                 lambda: h.fuse_update_tiled_splat(w.subs[1]._h, 0)):  # (another src than the plan's)
        with pytest.raises(capi.TslamError) as e:
            call()
        assert e.value.code == capi.E_INVALID
    w.tiled[0].update_finish(w.subs[0], False)
    # the single-map update still refuses a tiled dst
    with pytest.raises(capi.TslamError) as e:
        w.glos[0]._h.fuse_update(src)
    assert e.value.code == capi.E_INVALID and "tiled" in str(e.value)
    # a submap with blocks on two ranks: refused on every rank, nothing written
    _frame(w.subs[1], 0, False)
    with pytest.raises(ValueError, match="several ranks"):
        w.update()
    assert same(w.union(), before)


def test_plan_present_has_the_c_side_submap_table():
    """max_submaps = 0 gives the C side's 1024-entry table: the plan's present array has 1024 entries."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    src = TsdfHandle(128, 128, voxel_scale=0.05, K=K, max_ray_length=3.0, max_submaps=0)
    dst = TsdfHandle(256, 256, voxel_scale=0.05, K=K, max_ray_length=3.0, is_global_map=True, max_submaps=0)
    src.integrate_depth(DEPTH, np.eye(3)[None], np.zeros((1, 3)), submaps=[3])
    plan, present = dst.fuse_update_tiled_plan(src, (1, 1, 1), 0, 1)
    assert present.shape == (1024,) and np.flatnonzero(present).tolist() == [3]
    dst.fuse_update_tiled_finish(src, False)


def test_pool_exhaustion_on_an_owner_fails_every_rank_and_the_next_update_is_full():
    # rank 1 contributes nothing, so its pool fills only with the blocks it receives: size it between what the first
    # and the second update need
    probe = World(2, balance=False, present=range(6), owner=lambda s: 0)
    own = lambda ref: len({tuple(b) for b in np.floor_divide(ref["idx"], 16) if probe.tiled[0].owner_of_block(*b) == 1})
    small = np.zeros(NSUB, bool)
    small[:2] = True
    n_small, n_all = own(probe.reference(small)), own(probe.reference())
    assert n_all > n_small + 8
    del probe
    gc.collect()
    w = World(2, balance=False, present=range(6), owner=lambda s: 0, max_blocks={1: (n_small + n_all) // 2})
    assert w.update(small)["reason"] == "first call"
    check(w, small)
    with pytest.raises(capi.TslamError) as e:
        w.update()
    assert e.value.code == capi.E_POOL_FULL
    st = w.update(small)
    assert st["full"] and st["reason"] == "sums not valid"
    check(w, small)
    assert w.update(small)["reason"] == "incremental"
