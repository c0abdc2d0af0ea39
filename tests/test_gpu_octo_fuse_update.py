"""tslam_octo_fuse_update on the GPU (OctoHandle.fuse_update, Octomap.update_fused_submaps,
SubmapMapping(Octomap, global_fusion="incremental")): bit for bit against fuse_from with everything included and
against the numpy statement of the contract (tests/octo_fuse_update_reference.py) with include masks; history
independence, every full-update reason, tolerance, pool exhaustion, side effects, refusals, and the occupancy ESDF
and frontier trackers after incremental updates that move and remove submaps."""
import numpy as np
import pytest

import octo_esdf_reference as oe
import octo_frontier_reference as fr
import octo_fuse_update_reference as ofr
import octo_logodds_reference as ref
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu

VS = 0.05
N = 256
LO = ref.params()
KH = [syn.FX / 4, 0.0, syn.CX / 4, 0.0, syn.FY / 4, syn.CY / 4, 0.0, 0.0, 1.0]
NSUB = 6
MODELS = [("hits", False), ("hits", True), ("logodds", False), ("logodds", True)]


def handle(model, tex, max_submaps=64, **kw):
    from taichislam_b200.octo_handle import OctoHandle
    kw.setdefault("Kcam", KH)
    kw.setdefault("max_blocks", 1 << 14)
    h = OctoHandle(N, N, K=2, voxel_scale=VS, min_occupy_thres=1, max_ray_length=6.0, max_submaps=max_submaps,
                   texture_enabled=tex, logodds=LO if model == "logodds" else None, **kw)
    if tex:
        h.set_color_intrinsics(KH, color_same_proj=True)
    return h


def refused(fn, *a, code=None, **kw):
    from taichislam_b200 import _capi as capi
    with pytest.raises(capi.TslamError) as e:
        fn(*a, **kw)
    assert e.value.code == (capi.E_INVALID if code is None else code)
    return str(e.value)


class World:
    """Submaps of a few scene_room frames each (local poses), their global poses, and the frames in integrate order
    (so a collection of a subset can be integrated again in the same order: the same colour words win)."""

    def __init__(self, model, tex, seed=0, nsub=NSUB):
        self.model, self.tex = model, tex
        self.rng = np.random.default_rng(seed)
        self.depth = syn.scene_room(h=120, w=160)
        self.frames = []  # (submap, R, T, texture)
        self.src = handle(model, tex)
        self.poses = {}
        for s in range(nsub):
            self.add_submap(s)

    def frame(self, s):
        R = rot_xyz(*self.rng.uniform(-0.3, 0.3, 3))
        T = self.rng.uniform(-0.2, 0.2, 3)
        t = self.rng.integers(0, 256, (120, 160, 3), dtype=np.uint8) if self.tex else None
        self.frames.append((s, R, T, t))
        self.src.integrate_depth(self.depth, R, T, submap=s, texture=t)

    def add_submap(self, s, nframes=2):
        for _ in range(nframes):
            self.frame(s)
        self.poses[s] = (rot_xyz(0.0, 0.0, self.rng.uniform(-np.pi, np.pi)), self.rng.uniform(-1.0, 1.0, 3) * [1, 1, 0.2])

    def move(self, s, scale=0.3):
        R, T = self.poses[s]
        self.poses[s] = (rot_xyz(0.0, 0.0, self.rng.uniform(-scale, scale)) @ R, T + self.rng.uniform(-scale, scale, 3))

    def set_poses(self, h):
        for s, (R, T) in self.poses.items():
            h.set_submap_pose(s, R, T)

    def subset_src(self, keep):
        """a collection holding only the submaps in `keep`, integrated in the same order"""
        h = handle(self.model, self.tex)
        for s, R, T, t in self.frames:
            if s in keep:
                h.integrate_depth(self.depth, R, T, submap=s, texture=t)
        return h

    def rebuild(self, keep=None):
        """fuse_from of the included submaps into a fresh map"""
        src = self.src if keep is None else self.subset_src(keep)
        d = handle(self.model, self.tex)
        self.set_poses(d)
        d.fuse_from(src)
        return d

    def reference(self, include=None):
        rows = {}
        for s in self.poses:
            g = self.src.gather(s)
            rows[s] = (g[0], g[1], None)
        return ofr.fuse(rows, {s: self.poses[s] for s in self.poses}, VS, N, N, model=self.model, thres=1, l_min=LO["l_min"],
                        l_max=LO["l_max"], include=include)


def rows(h):
    """sorted gathered rows (idx, word value[, colour]) of submap 0"""
    return ofr.sorted_rows(*h.gather(0, color=h.texture_enabled))


def assert_same(a, b):
    ra, rb = rows(a), rows(b)
    assert ra[0].shape == rb[0].shape, f"{ra[0].shape[0]} rows, expected {rb[0].shape[0]}"
    for x, y in zip(ra, rb):
        assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x, y.view(np.uint32) if y.dtype == np.float32 else y)


def assert_reference(h, w, include=None):
    ri, rv, _ = w.reference(include)
    g = rows(h)
    assert g[0].shape[0] == ri.shape[0] and ri.shape[0] > 0
    assert np.array_equal(g[0], ri) and np.array_equal(g[1], rv)


@pytest.mark.parametrize("model,tex", MODELS)
def test_everything_included_matches_fuse_from(model, tex):
    w = World(model, tex)
    d = handle(model, tex)
    w.set_poses(d)
    st = d.fuse_update(w.src)
    assert st["full"] and st["reason"] == "first call" and st["added"] == NSUB and st["voxels_splatted"] > 0
    assert_same(d, w.rebuild())
    assert_reference(d, w)
    st = d.fuse_update(w.src)
    assert not st["full"] and st["added"] == st["moved"] == st["removed"] == 0 and st["blocks_committed"] == 0
    assert_same(d, w.rebuild())


@pytest.mark.parametrize("model,tex", MODELS)
def test_include_masks_match_the_reference(model, tex):
    w = World(model, tex, seed=1)
    d = handle(model, tex)
    w.set_poses(d)
    d.fuse_update(w.src)
    for keep in ({0, 2, 4, 5}, {0, 1, 2, 4, 5}, {3}, set(range(NSUB))):
        inc = np.array([s in keep for s in range(NSUB)])
        st = d.fuse_update(w.src, include=inc)
        assert_reference(d, w, include=keep)
        if tex:
            assert_same(d, w.rebuild(keep))
        if not st["full"] and tex and st["removed"]:
            assert st["voxels_skipped"] > 0  # recoloured voxels


@pytest.mark.parametrize("model,tex", MODELS)
def test_history_independence(model, tex):
    w = World(model, tex, seed=2)
    d = handle(model, tex)
    w.set_poses(d)
    keep = set(range(NSUB))
    d.fuse_update(w.src)
    rng = np.random.default_rng(7)
    reasons = set()
    for step in range(10):
        op = ["move", "move_all", "exclude", "include", "new", "content"][step % 6]
        if op == "move":
            w.move(int(rng.integers(0, len(w.poses))))
        elif op == "move_all":  # subtracting and re-adding every submap costs more than a rebuild: the cost rule
            for s in range(len(w.poses)):
                w.move(s, 0.05)
        elif op == "exclude":
            keep.discard(int(rng.integers(0, len(w.poses))))
        elif op == "include":
            keep |= set(range(len(w.poses)))
        elif op == "new":
            s = len(w.poses)
            w.add_submap(s, 1)
            keep.add(s)
        else:
            w.frame(int(rng.integers(0, len(w.poses))))
        w.set_poses(d)
        inc = np.array([s in keep for s in range(len(w.poses))])
        st = d.fuse_update(w.src, include=inc)
        reasons.add(st["reason"])
        fresh = handle(model, tex)
        w.set_poses(fresh)
        sf = fresh.fuse_update(w.src, include=inc)
        assert sf["full"]
        assert_same(d, fresh)
        if keep == set(w.poses):
            assert_same(d, w.rebuild())
    assert {"incremental", "content changed", "cheaper than subtract and re-add"} <= reasons


def test_full_update_reasons_and_tolerance():
    w = World("logodds", False, seed=3)
    d = handle("logodds", False)
    w.set_poses(d)
    assert d.fuse_update(w.src)["reason"] == "first call"
    assert d.fuse_update(w.src, full=True)["reason"] == "full requested"
    other = World("logodds", False, seed=3)
    assert d.fuse_update(other.src)["reason"] == "other source"
    assert d.fuse_update(w.src)["reason"] == "other source"
    d.integrate_points(np.array([[0.5, 0.0, 0.0]], np.float32), np.eye(3), np.zeros(3), submap=3)
    assert d.fuse_update(w.src)["reason"] == "destination written"
    d.reset()
    assert d.fuse_update(w.src)["reason"] == "destination written"
    d.fuse_from(w.src)
    assert d.fuse_update(w.src)["reason"] == "destination written"
    w.frame(2)
    assert d.fuse_update(w.src)["reason"] == "content changed"
    for s in range(NSUB):
        w.move(s)
    w.set_poses(d)
    assert d.fuse_update(w.src)["reason"] == "cheaper than subtract and re-add"
    assert_same(d, w.rebuild())
    # tolerance: a 1 mm move stays at the fused pose, a larger one is placed again
    before = rows(d)
    R, T = w.poses[1]
    d.set_submap_pose(1, R, T + [0.001, 0.0, 0.0])
    st = d.fuse_update(w.src, tolerance=0.01)
    assert st["reason"] == "incremental" and st["within_tolerance"] == 1 and st["moved"] == 0
    assert all(np.array_equal(x, y) for x, y in zip(rows(d), before))
    st = d.fuse_update(w.src, tolerance=0.0)
    assert st["moved"] == 1 and st["within_tolerance"] == 0
    w.poses[1] = (R, T + [0.001, 0.0, 0.0])
    assert_same(d, w.rebuild())


@pytest.mark.parametrize("model", ["hits", "logodds"])
def test_pool_exhaustion_changes_nothing_and_the_next_call_is_full(model):
    from taichislam_b200 import _capi as capi
    w = World(model, False, seed=4)
    big = handle(model, False)
    w.set_poses(big)
    big.fuse_update(w.src)
    nb_all = big.gather(0)[0]
    one = handle(model, False)
    w.set_poses(one)
    one.fuse_update(w.src, include=[1])
    need1 = len({tuple(c) for c in (one.gather(0)[0] >> 3)})
    need_all = len({tuple(c) for c in (nb_all >> 3)})
    assert need_all > need1 + 8
    d = handle(model, False, max_blocks=need1 + 4)
    w.set_poses(d)
    d.fuse_update(w.src, include=[1])
    before = rows(d)
    refused(d.fuse_update, w.src, code=capi.E_POOL_FULL)
    assert all(np.array_equal(x, y) for x, y in zip(rows(d), before))
    st = d.fuse_update(w.src, include=[1])
    assert st["full"]
    assert_same(d, one)
    # a full update resets dst before it runs out: nothing is added, dst comes back empty, the next call is full
    refused(d.fuse_update, w.src, full=True, code=capi.E_POOL_FULL)
    assert rows(d)[0].shape[0] == 0
    st = d.fuse_update(w.src, include=[1])
    assert st["full"] and st["reason"] == "first call"
    assert_same(d, one)


def test_no_side_effects_on_src():
    w = World("logodds", True, seed=5)
    src = w.src
    src.esdf_update(2, max_dist=0.5)
    src.frontier_update(2)
    before = ofr.sorted_rows(*src.gather(2, color=True))
    e_before = as_dict_rows(*src.esdf_gather(2))
    d = handle("logodds", True)
    w.set_poses(d)
    d.fuse_update(src)
    w.move(2)
    w.set_poses(d)
    d.fuse_update(src, include=[1, 1, 0, 1, 1, 1])
    after = ofr.sorted_rows(*src.gather(2, color=True))
    assert all(np.array_equal(x, y) for x, y in zip(after, before))
    assert all(np.array_equal(x, y) for x, y in zip(as_dict_rows(*src.esdf_gather(2)), e_before))
    assert src.esdf_update(2, max_dist=0.5)["raise_sweeps"] != -1  # still incremental
    assert not src.frontier_update(2)["full"]


def test_refusals():
    w = World("logodds", False, seed=6, nsub=2)
    d = handle("logodds", False)
    w.set_poses(d)
    d.fuse_update(w.src)
    before = rows(d)
    for other, what in ((handle("hits", False), "hit-counter"), (handle("logodds", True), "texture"),
                        (handle("logodds", False, max_submaps=32), "max_submaps")):
        refused(d.fuse_update, other)
    from taichislam_b200.octo_handle import OctoHandle
    refused(d.fuse_update, OctoHandle(N, N, K=2, voxel_scale=0.1, logodds=LO, max_submaps=64))
    big = dict(LO, l_max=1 << 20, l_occ=0)
    msg = refused(d.fuse_update, OctoHandle(N, N, K=2, voxel_scale=VS, logodds=big, max_submaps=64))
    assert "2^30" in msg
    refused(d.fuse_update, w.src, tolerance=-1.0)
    refused(d.fuse_update, w.src, tolerance=float("nan"))
    refused(d.fuse_update, d)
    assert all(np.array_equal(x, y) for x, y in zip(rows(d), before))
    assert d.fuse_update(w.src)["reason"] == "incremental"  # a refusal wrote nothing


def test_trackers_stay_incremental_and_exact_after_moves_and_removals():
    w = World("logodds", False, seed=8)
    d = handle("logodds", False)
    w.set_poses(d)
    d.fuse_update(w.src)
    D = 0.5
    d.esdf_update(0, max_dist=D)
    d.frontier_update(0)
    keep = set(range(NSUB))
    rng = np.random.default_rng(9)
    for step in range(6):
        if step % 3 == 0:
            w.move(int(rng.integers(0, NSUB)))
        elif step % 3 == 1:
            keep.discard(int(rng.integers(0, NSUB)))
        else:
            keep.add(int(rng.integers(0, NSUB)))
            w.move(int(rng.integers(0, NSUB)), 0.1)
        w.set_poses(d)
        st = d.fuse_update(w.src, include=np.array([s in keep for s in range(NSUB)]))
        assert st["reason"] == "incremental"
        as_dict_rows(*d.esdf_gather(0))          # readable as of the last update
        d.frontier_gather(0)
        e0 = d.esdf_update(0, max_dist=D)
        assert e0["raise_sweeps"] != -1          # incremental
        g0 = as_dict_rows(*d.esdf_gather(0))
        d.esdf_update(0, max_dist=D, full=True)
        g1 = as_dict_rows(*d.esdf_gather(0))
        idx, L = d.gather(0)
        gr = as_dict_rows(idx, oe.esdf(idx, L, LO["l_occ"], VS, D))
        for a, b, c in zip(g0, g1, gr):
            assert np.array_equal(a.view(np.int32) if a.dtype == np.float32 else a, b.view(np.int32) if b.dtype == np.float32 else b)
            assert np.array_equal(a.view(np.int32) if a.dtype == np.float32 else a, c.view(np.int32) if c.dtype == np.float32 else c)
        f0 = d.frontier_update(0)
        assert not f0["full"]
        i0, c0 = as_dict_rows(*d.frontier_gather(0))
        r0 = d.frontier_clusters(0)
        d.frontier_update(0, full=True)
        i1, c1 = as_dict_rows(*d.frontier_gather(0))
        r1 = d.frontier_clusters(0)
        ri, rc, rr = fr.frontiers(idx, L, LO["l_occ"], N, N)
        assert np.array_equal(i0, i1) and np.array_equal(c0, c1) and np.array_equal(r0, r1)
        assert np.array_equal(i0, ri) and np.array_equal(c0, rc) and np.array_equal(r0, rr)
    d.fuse_update(w.src, full=True)
    refused(d.esdf_gather, 0)
    refused(d.frontier_gather, 0)


def rebuild(sm, opts):
    """fuse_submaps of the collection at the global map's poses, the active submap left out (placed outside the volume,
    as the incremental mode leaves it out)"""
    from taichislam_b200.mapping.taichi_octomap import Octomap
    g = sm.global_map
    reb = Octomap(**dict(opts, max_submap_num=16))
    active = sm.submap_collection.get_active_submap_id()
    for s in range(16):
        T = g.submaps_base_T_np[s] + (np.array([1e4, 0.0, 0.0]) if s == active else 0.0)
        reb._h.set_submap_pose(s, g.submaps_base_R_np[s], T)
    reb.fuse_submaps(sm.submap_collection)
    return reb._h


@pytest.mark.parametrize("model", ["hits", "logodds"])
def test_submap_mapping_incremental_octomap(model):
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    from taichislam_b200.mapping.taichi_octomap import Octomap
    opts = dict(map_scale=[12.8, 12.8], voxel_scale=VS, max_ray_length=6.0, occupancy_model=model, min_occupy_thres=1)
    sm = SubmapMapping(Octomap, keyframe_step=2, sub_opts=dict(opts, max_submap_num=16), global_opts=dict(opts),
                       global_fusion="incremental")
    sm.set_dep_camera_intrinsic(KH)
    d = syn.scene_room(h=120, w=160)
    rng = np.random.default_rng(11)
    frames = {}
    g = sm.global_map
    for q in range(8):
        R, T = rot_xyz(0.0, 0.0, 0.2 * q), np.array([0.1 * q, 0.0, 0.0])
        frames[q] = (R, T)
        sm.recast_depth_to_map_by_frame(q, True, (R, T), (np.eye(3), np.zeros(3)), d, None)
        if q % 2 == 1 and q > 1:
            # move an old submap: the correction reaches the global map at once
            fid = sorted(sm.submaps)[0]
            R0, T0 = frames[fid]
            sm.set_frame_poses({fid: (rot_xyz(0.0, 0.0, rng.uniform(-0.1, 0.1)) @ R0, T0 + rng.uniform(-0.05, 0.05, 3))})
            st = sm.last_fusion_stats  # (with few fused submaps the cost rule may pick the rebuild)
            assert (st["reason"], st["moved"]) in (("incremental", 1), ("cheaper than subtract and re-add", 0))
        if q > 1:
            assert_same(g._h, rebuild(sm, opts))
    assert len(sm.submaps) == 4
    with pytest.raises(ValueError):
        SubmapMapping(Octomap, global_fusion="incremental", reclaim_empty=True)


@pytest.mark.parametrize("model", ["hits", "logodds"])
def test_volumes_may_differ(model):
    """placement tests only dst's bounds, as fuse_from does: a large global map of small submaps, and a small one"""
    w = World(model, False, seed=12)
    for n_dst in (4 * N, N // 2):
        from taichislam_b200.octo_handle import OctoHandle
        kw = dict(K=2, voxel_scale=VS, min_occupy_thres=1, max_ray_length=6.0, Kcam=KH, max_submaps=64, max_blocks=1 << 15,
                  logodds=LO if model == "logodds" else None)
        d, reb = OctoHandle(n_dst, n_dst, **kw), OctoHandle(n_dst, n_dst, **kw)
        for s, (R, T) in w.poses.items():  # far from the origin: beyond the submaps' own half-extent when the map is large
            T = np.asarray(T) + [0.6 * n_dst * VS / 2, 0.0, 0.0]
            d.set_submap_pose(s, R, T)
            reb.set_submap_pose(s, R, T)
        assert d.fuse_update(w.src)["full"]
        w.move(1)
        R, T = w.poses[1]
        T = np.asarray(T) + [0.6 * n_dst * VS / 2, 0.0, 0.0]
        d.set_submap_pose(1, R, T)
        reb.set_submap_pose(1, R, T)
        assert d.fuse_update(w.src)["moved"] == 1
        reb.fuse_from(w.src)
        assert_same(d, reb)
        idx = rows(d)[0]
        assert idx.shape[0] > 0 and (idx.max() < n_dst // 2) and (idx.min() >= -(n_dst // 2))
        if n_dst > N:
            assert (idx[:, 0] >= N // 2).any()  # cells outside the submaps' own volume are kept


@pytest.mark.parametrize("model", ["hits", "logodds"])
def test_submap_mapping_incremental_octomap_default_options(model):
    """SubmapMapping's defaults: 10 m submaps, a 100 m global map; the incremental mode keeps the global volume"""
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    from taichislam_b200.mapping.taichi_octomap import Octomap
    gopts = dict(occupancy_model=model)
    sm = SubmapMapping(Octomap, keyframe_step=2, sub_opts=dict(occupancy_model=model), global_opts=gopts,
                       global_fusion="incremental")
    g = sm.global_map
    assert g.N == 2048 and sm.submap_collection.N == 256
    sm.set_dep_camera_intrinsic(KH)
    d = syn.scene_sphere(2.0, h=120, w=160)
    for q in range(6):
        R, T = rot_xyz(0.0, 0.0, 0.3 * q), np.array([9.0 + 0.2 * q, 0.0, 0.0])  # 9 m out: beyond a 10 m map's 6.4 m
        sm.recast_depth_to_map_by_frame(q, True, (R, T), (np.eye(3), np.zeros(3)), d, None)
        if q == 3:
            fid = sorted(sm.submaps)[0]
            sm.set_frame_poses({fid: (R, T + [0.03, -0.02, 0.01])})
        if q > 1:
            reb = sm.create_globalmap(gopts)
            active = sm.submap_collection.get_active_submap_id()
            for s in range(g.max_submap_num):
                Ts = g.submaps_base_T_np[s] + (np.array([1e5, 0.0, 0.0]) if s == active else 0.0)
                reb._h.set_submap_pose(s, g.submaps_base_R_np[s], Ts)
            reb.fuse_submaps(sm.submap_collection)
            assert_same(g._h, reb._h)
            idx = rows(g._h)[0]
            assert idx.shape[0] > 0 and (idx[:, 0] * VS > 6.4).any()
