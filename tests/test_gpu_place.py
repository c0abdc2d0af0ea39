"""GPU: loop detection between TSDF submaps (tslam_tsdf_place_describe, tslam_place_match) against
tests/place_reference.py: descriptors and match outputs bit for bit, batching and determinism, no side effects, every
refusal, and the loop world (tests/loop_world.py) through DenseTSDF.detect_loops and SubmapMapping.detect_loops."""
import numpy as np
import pytest

import loop_world as lw
import place_reference as ref
import track_world as tw
from taichislam_b200 import _capi as capi
from taichislam_b200 import place
from taichislam_b200 import synthetic as syn
from util import as_dict_rows

pytestmark = pytest.mark.gpu
F = np.float32
VS = 0.05
BAND = 4 * VS
R_MAX, H_MIN = 8.0, 0.3


def handle(N=256, Nz=256, **kw):
    from taichislam_b200.tsdf_handle import TsdfHandle
    return TsdfHandle(N, Nz, K=syn.K_DEPTH, max_ray_length=kw.pop("max_ray_length", 6.0), max_submaps=kw.pop("max_submaps", 16), **kw)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def levelled_f32(Rs, up=(0.0, 0.0, 1.0)):
    L = place.level(up)
    return np.stack([L @ R for R in Rs])


def check_describe(m, submaps, Rs, up=(0.0, 0.0, 1.0), r_max=R_MAX, h_min=H_MIN, band=BAND, min_weight=0.0, vs=VS):
    M = levelled_f32(Rs, up)
    got = m.place_describe(submaps, M, r_max, h_min, band, min_weight)
    for i, s in enumerate(submaps):
        idx, t, w, _ = m.gather(s)
        want = ref.describe_rows(idx, t, w, M[i].astype(F), vs, r_max, h_min, band, min_weight)
        assert got["n_points"][i] == want["n_points"], (s, got["n_points"][i], want["n_points"])
        assert np.array_equal(bits(got["sc"][i].cpu().numpy()), bits(want["sc"])), s
        assert np.array_equal(bits(got["ring"][i].cpu().numpy()), bits(want["ring"])), s
        assert np.array_equal(got["bev"][i].cpu().numpy().view(np.uint32), want["bev"]), s
    return got


def box_rows(lo, hi, fn, vs=VS):
    r = [np.arange(a, b) for a, b in zip(lo, hi)]
    I, J, K = np.meshgrid(*r, indexing="ij")
    idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
    return idx, np.asarray(fn(idx.astype(np.float64) * vs), F), np.ones(len(idx), F)


def pillars(x):
    """A floor at z = -0.6 and two pillars: vertical structure at negative coordinates."""
    d = x[:, 2] + 0.6
    for cx, cy in ((-1.1, -0.7), (0.9, -1.4)):
        d = np.minimum(d, np.hypot(x[:, 0] - cx, x[:, 1] - cy) - 0.25)
    return d


@pytest.fixture(scope="module")
def scenes():
    out = {}
    for name, depth in (("S1", syn.scene_plane()), ("S2", syn.scene_sphere(4.0)), ("room", syn.scene_room()),
                        ("box", tw.render(*tw.pose(0)))):
        m = handle()
        m.integrate_depth(depth, np.eye(3)[None], np.zeros((1, 3)), submaps=[0])
        m.integrate_depth(depth, tw.rot([0, 1, 0], 5.0)[None], np.array([[0.1, 0.0, 0.05]]), submaps=[1])
        out[name] = m
    return out


@pytest.mark.parametrize("name", ["S1", "S2", "room", "box"])
def test_descriptors_match_reference_on_integrated_scenes(scenes, name):
    m = scenes[name]
    Rs = [np.eye(3), tw.rot([0, 1, 0], 33.0) @ tw.rot([1, 0, 0], -4.0)]
    check_describe(m, [0, 1], Rs, up=(0.0, -1.0, 0.0))
    check_describe(m, [1, 0, 1], [Rs[0], Rs[1], np.eye(3)], up=(0.2, -1.0, 0.1), r_max=3.3, h_min=0.11)  # a repeated submap


def test_descriptors_negative_blocks_odd_volume_and_extreme_submaps():
    m = handle(200, 72, max_submaps=1024)
    for s in (0, 1023):
        idx, t, w = box_rows((-60, -60, -20), (40, 20, 30), pillars)
        m.scatter(s, idx, t, w, np.zeros(len(idx), np.int8))
    got = check_describe(m, [0, 1023, 5], [np.eye(3), tw.rot([0, 0, 1], 17.0), np.eye(3)], r_max=4.0, h_min=0.2)
    assert got["n_points"][0] > 0 and got["n_points"][2] == 0
    assert np.array_equal(got["sc"][2].cpu().numpy(), np.zeros((20, 60), F))
    bev0 = ref.unpack(got["bev"][0].cpu().numpy().view(np.uint32))
    assert bev0.any() and not bev0.all()
    # every point of submap 1023 at once: rings, sectors and cells agree with the reference for the same rotation
    check_describe(m, [1023], [tw.rot([1, 1, 0], 3.0)], r_max=2.0, h_min=0.05, band=0.1, min_weight=0.5)


def test_descriptors_textured_map():
    m = handle(texture_enabled=True)
    d = syn.scene_room()
    m.integrate_depth(d[None], np.eye(3)[None], np.zeros((1, 3)), submaps=[0], texture=syn.texture_gradient(1)[None])
    check_describe(m, [0], [np.eye(3)], up=(0.0, -1.0, 0.0))


def test_descriptors_ten_voxel_blocks():
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    dm = DenseTSDF(map_scale=[12.8, 6.4], voxel_scale=VS, num_voxel_per_blk_axis=10, max_ray_length=6.0, max_submap_num=4,
                   max_disp_particles=1 << 16)
    dm.set_dep_camera_intrinsic(syn.K_DEPTH)
    R, t = tw.pose(5)
    dm.set_base_pose_submap(0, R, t)
    dm.recast_depth_to_map(R, t, tw.render(R, t), np.array([]))
    got = dm.describe_places([0], up=lw.UP, r_max=R_MAX, h_min=H_MIN)
    idx, ts, w, _ = dm._h.gather(0)
    want = ref.describe_rows(idx, ts, w, got["M"][0].astype(F), VS, R_MAX, H_MIN, BAND)
    assert got["n_points"][0] == want["n_points"] > 0
    assert np.array_equal(bits(got["sc"][0].cpu().numpy()), bits(want["sc"]))
    assert np.array_equal(got["bev"][0].cpu().numpy().view(np.uint32), want["bev"])


# ---- the loop world ---------------------------------------------------------------------------------------------------
def build_loop_world(num_voxel_per_blk_axis=16):
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    dm = DenseTSDF(map_scale=[12.8, 12.8], voxel_scale=VS, num_voxel_per_blk_axis=num_voxel_per_blk_axis, max_ray_length=6.0,
                   max_submap_num=16, max_disp_particles=1 << 16)
    dm.set_dep_camera_intrinsic(syn.K_DEPTH)
    for s in range(lw.n_submaps()):
        if s:
            dm.switch_to_next_submap()
        dm.set_base_pose_submap(s, *lw.odometry_pose(s, 0))
        for f in range(lw.FRAMES):
            dm.recast_depth_to_map(*lw.odometry_pose(s, f), lw.render(s, f), np.array([]))
    dm.finalization_current_submap()
    return dm


@pytest.fixture(scope="module")
def loop_map():
    return build_loop_world()


def test_match_outputs_match_reference(loop_map):
    dm = loop_map
    S = list(range(lw.n_submaps()))
    desc = dm.describe_places(S, up=lw.UP, r_max=R_MAX, h_min=H_MIN)
    rdesc = []
    for s in S:
        idx, t, w, _ = dm._h.gather(s)
        r = ref.describe_rows(idx, t, w, desc["M"][s].astype(F), VS, R_MAX, H_MIN, BAND)
        assert np.array_equal(r["bev"], desc["bev"][s].cpu().numpy().view(np.uint32)) and r["n_points"] == desc["n_points"][s]
        rdesc.append(r)
    ids = np.array(S, np.int64) * 3
    queries = [lw.N_LOOP - 1, 0, lw.N_LOOP]
    got = place.match(desc["sc"], desc["ring"], desc["bev"], desc["n_points"], ids, queries, top_k=4, min_gap=5, min_points=200)
    info, dist = ref.match(rdesc, ids, queries, 4, 5, 200)
    assert np.array_equal(got["info6"].reshape(-1, 6), info)
    assert np.array_equal(bits(got["dist3"].reshape(-1, 3)), bits(dist))
    # a query's rows do not depend on the other queries; two identical calls give the same bits
    for qi, q in enumerate(queries):
        one = place.match(desc["sc"], desc["ring"], desc["bev"], desc["n_points"], ids, [q], top_k=4, min_gap=5, min_points=200)
        assert np.array_equal(one["info6"][0], got["info6"][qi]) and np.array_equal(bits(one["dist3"][0]), bits(got["dist3"][qi]))
    again = place.match(desc["sc"], desc["ring"], desc["bev"], desc["n_points"], ids, queries, top_k=4, min_gap=5, min_points=200)
    assert np.array_equal(again["info6"], got["info6"]) and np.array_equal(bits(again["dist3"]), bits(got["dist3"]))
    # the coarse pose of the loop pair is the reference's
    k = int(np.nonzero(got["match"][0] == 0)[0][0])
    R0, T0 = place.coarse_pose(desc["M"][queries[0]], desc["M"][0], got["yaw_deg"][0, k], got["dx"][0, k], got["dy"][0, k], R_MAX)
    Rr, Tr = ref.coarse_pose(desc["M"][queries[0]], desc["M"][0], got["shift"][0, k], got["yaw_idx"][0, k], got["dx"][0, k],
                             got["dy"][0, k], R_MAX)
    assert np.allclose(R0, Rr, atol=1e-14) and np.allclose(T0, Tr, atol=1e-14)


def pose_error(R, T, Rg, Tg):
    dR = R @ Rg.T
    ang = np.degrees(np.arccos(np.clip((np.trace(dR) - 1.0) / 2.0, -1.0, 1.0)))
    return float(np.linalg.norm(T - Tg)), float(ang)


def check_constraints(found):
    """The loop pair is accepted, every accepted constraint is within 0.5 voxel and 0.5 degree of the truth, and none joins
    the two rooms."""
    acc = [c for c in found if c["accepted"]]
    assert any(c["query"] == lw.N_LOOP - 1 and c["match"] == 0 for c in acc), [(c["query"], c["match"], c["accepted"]) for c in found]
    for c in acc:
        assert (c["query"] < lw.N_LOOP) == (c["match"] < lw.N_LOOP), (c["query"], c["match"])
        et, er = pose_error(c["R"], c["T"], *lw.relative(c["query"], c["match"]))
        assert et <= 0.5 * VS and er <= 0.5, (c["query"], c["match"], et, er)
    return acc


def test_detect_loops_finds_the_loop_and_rejects_the_other_room(loop_map):
    found = loop_map.detect_loops([lw.N_LOOP - 1], up=lw.UP, min_gap=2)
    check_constraints(found)
    # every submap as a query: all accepted constraints are true ones, none between the rooms
    found = loop_map.detect_loops(list(range(lw.n_submaps())), up=lw.UP, min_gap=2)
    check_constraints(found)


def test_no_side_effects(loop_map):
    from util import tri_multiset
    h = loop_map._h
    S = list(range(lw.n_submaps()))
    rows = [as_dict_rows(*h.gather(s)) for s in S]
    n0, v0, _ = h.marching_cubes()
    before = h.stats()
    loop_map.describe_places(S, up=lw.UP)
    after = h.stats()
    assert after["launches"] > before["launches"]
    for k in before:
        if k != "launches":
            assert before[k] == after[k], k
    for s in S:
        for x, y in zip(rows[s], as_dict_rows(*h.gather(s))):
            assert np.array_equal(bits(x), bits(y))
    n1, v1, _ = h.marching_cubes()
    assert n0 == n1 and np.array_equal(tri_multiset(v0), tri_multiset(v1))


def test_refusals(loop_map):
    h = loop_map._h
    I = np.eye(3)[None]

    def refused(fn, *a, **kw):
        with pytest.raises(capi.TslamError) as e:
            fn(*a, **kw)
        assert e.value.code == capi.E_INVALID

    refused(h.place_describe, [], np.zeros((0, 3, 3)), R_MAX, H_MIN, BAND)
    refused(h.place_describe, [0] * 1025, np.stack([np.eye(3)] * 1025), R_MAX, H_MIN, BAND)
    refused(h.place_describe, [16], I, R_MAX, H_MIN, BAND)
    refused(h.place_describe, [-1], I, R_MAX, H_MIN, BAND)
    for r_max, h_min, band, mw in ((0.0, H_MIN, BAND, 0.0), (R_MAX, np.nan, BAND, 0.0), (R_MAX, H_MIN, -1.0, 0.0),
                                   (R_MAX, H_MIN, BAND, np.inf)):
        refused(h.place_describe, [0], I, r_max, h_min, band, mw)
    refused(h.place_describe, [0], np.full((1, 3, 3), np.nan), R_MAX, H_MIN, BAND)
    with pytest.raises(ValueError):
        loop_map.describe_places([0], up=(0.0, 0.0, 0.0))
    d = loop_map.describe_places([0, 1, 2], up=lw.UP)
    args = (d["sc"], d["ring"], d["bev"], d["n_points"], [0, 1, 2])
    for kw in (dict(queries=[3]), dict(queries=[-1]), dict(queries=[0], top_k=0), dict(queries=[0], top_k=33),
               dict(queries=[0], min_gap=-1), dict(queries=[])):
        refused(place.match, *args, **kw)


def test_submap_mapping_detect_loops_ten_voxel_blocks():
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    sub = dict(map_scale=[12.8, 12.8], voxel_scale=VS, num_voxel_per_blk_axis=10, max_ray_length=6.0, max_submap_num=16,
               max_disp_particles=1 << 16)
    glo = dict(map_scale=[25.6, 12.8], voxel_scale=VS, num_voxel_per_blk_axis=10, max_ray_length=6.0, max_submap_num=16,
               max_disp_particles=1 << 16)
    sm = SubmapMapping(DenseTSDF, sub_opts=sub, global_opts=glo, keyframe_step=lw.FRAMES)
    sm.set_dep_camera_intrinsic(syn.K_DEPTH)
    ext = (np.eye(3), np.zeros(3))
    fid = 0
    for s in range(lw.N_LOOP):
        for f in range(lw.FRAMES):
            sm.recast_depth_to_map_by_frame(fid, True, lw.odometry_pose(s, f), ext, lw.render(s, f), np.array([]))
            fid += 1
    sm.submap_collection.finalization_current_submap()
    assert sm.submaps == {lw.FRAMES * s: s for s in range(lw.N_LOOP)}
    last = lw.FRAMES * (lw.N_LOOP - 1)
    base_before = sm.global_map.submaps_base_R_np[lw.N_LOOP - 1].copy()
    out = sm.detect_loops(min_gap=2)
    assert (last, 0) in out, list(out)
    for (fq, fd), c in out.items():
        assert fq == last and c["accepted"]
        et, er = pose_error(c["R"], c["T"], *lw.relative(fq // lw.FRAMES, fd // lw.FRAMES))
        assert et <= 0.5 * VS and er <= 0.5, (fq, fd, et, er)
    c = out[(last, 0)]
    # the implied world pose of the newest submap is its true pose (submap 0 is drift-free)
    et, er = pose_error(c["world_R"], c["world_T"], *lw.true_pose(lw.N_LOOP - 1, 0))
    assert et <= 0.5 * VS and er <= 0.5, (et, er)
    assert np.array_equal(sm.global_map.submaps_base_R_np[lw.N_LOOP - 1], base_before)  # nothing applied
