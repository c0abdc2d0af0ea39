"""GPU: SDF-to-SDF registration of TSDF submap pairs (tslam_tsdf_register) against tests/submap_register_reference.py:
the normal equations at the initial pose, full solves, known-answer recovery, batching and determinism, cross-handle
pairs, no side effects, every refusal and status, and the Python flows (DenseTSDF.register_submaps,
SubmapMapping.align_submap)."""
import numpy as np
import pytest

import submap_register_reference as ref
from taichislam_b200 import _capi as capi
from taichislam_b200 import synthetic as syn
from util import as_dict_rows

pytestmark = pytest.mark.gpu
F = np.float32
VS = 0.05
BAND = 4 * VS


def handle(N=256, Nz=256, **kw):
    from taichislam_b200.tsdf_handle import TsdfHandle
    return TsdfHandle(N, Nz, K=syn.K_DEPTH, max_ray_length=kw.pop("max_ray_length", 6.0), max_submaps=kw.pop("max_submaps", 16), **kw)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def box_rows(lo, hi, fn):
    r = [np.arange(a, b) for a, b in zip(lo, hi)]
    I, J, K = np.meshgrid(*r, indexing="ij")
    idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
    return idx, np.asarray(fn(idx.astype(np.float64) * VS), F), np.ones(len(idx), F)


def corner(R=np.eye(3), t=np.zeros(3)):
    def f(x):
        y = x @ R.T + t
        return np.minimum(np.minimum(y[:, 0] - 0.1, y[:, 1] + 0.05), y[:, 2] - 0.2)
    return f


def ref_pair(A, sa, B, sb, band=BAND, min_weight=0.0):
    ia, ta, wa, _ = A.gather(sa)
    ib, tb, wb, _ = B.gather(sb)
    return ref.Reading(ib, tb, wb, B.N, B.Nz, VS), ref.select_points(ia, ta, wa, VS, band, min_weight)


def check_normal_equations(A, sa, B, sb, R0, T0, band=BAND, min_weight=0.0, huber=VS):
    got = A.register(B, [sa], [sb], R0[None], T0[None], band, min_weight, huber, max_iters=0, min_points=0)
    rd, (p, d) = ref_pair(A, sa, B, sb, band, min_weight)
    S = ref.normal_equations(rd, p, d, R0, T0, huber)
    Aabs, q = ref.abs_sums(rd, p, d, R0, T0, huber)
    assert got["n_points"][0] == len(p)
    assert got["n_valid"][0] == S[28]
    H = got["H"][0]
    k = 0
    for i in range(6):
        for j in range(i, 6):
            assert H[i, j] == H[j, i] and abs(H[i, j] - S[k]) <= 1e-9 * Aabs[k], (i, j, H[i, j], S[k])
            k += 1
    assert np.all(np.abs(got["b"][0] - S[21:27]) <= 1e-9 * Aabs[21:27])
    assert abs(got["cost"][0] - S[27]) <= 1e-9 * Aabs[27] and got["cost_init"][0] == got["cost"][0]
    assert np.array_equal(got["R"][0], R0) and np.array_equal(got["T"][0], T0) and got["iterations"][0] == 0
    return q


@pytest.fixture(scope="module")
def analytic():
    """Submap 0: the corner field; submap 1: the same field seen through a known pose; submap 2: a plane at the +x edge of
    the volume (N = 128)."""
    m = handle(128, 64)
    dR, dt = ref.rot([1, 2, 3], 2.5), np.array([0.01, 0.01, 0.04])
    for s, f in ((0, corner()), (1, corner(dR, dt))):
        m.scatter(s, *box_rows((-24, -24, -16), (24, 24, 24), f), np.zeros(48 * 48 * 40, np.int8))
    idx, t, w = box_rows((56, -8, -8), (64, 8, 8), lambda x: x[:, 0] - 3.05)
    m.scatter(2, idx, t, w, np.zeros(len(idx), np.int8))
    return m, dR, dt


def test_normal_equations_analytic_fields_block_spans_and_volume_edge(analytic):
    m, dR, dt = analytic
    for R0, T0 in ((np.eye(3), np.zeros(3)), (dR, dt), (ref.rot([0, 0, 1], 4.0), np.array([0.013, -0.021, 0.007]))):
        q = check_normal_equations(m, 1, m, 0, R0, T0)
        i0 = np.floor(q["x"][q["valid"]] / F(VS)).astype(np.int64)
        spans = ((i0 & 15) == 15).sum(1)
        assert all((spans == k).any() for k in (1, 2, 3))        # corner cubes over 2, 4 and 8 blocks
    q = check_normal_equations(m, 2, m, 2, np.eye(3), np.array([0.02, 0.0, 0.0]))
    assert q["valid"].any() and not q["valid"].all()              # some corner cubes leave the volume


@pytest.fixture(scope="module")
def scenes():
    """S1, S2 and scene_room, each integrated into submap 0 (camera at the origin) and submap 1 (camera moved)."""
    out = {}
    for name, depth in (("S1", syn.scene_plane()), ("S2", syn.scene_sphere(4.0)), ("room", syn.scene_room())):
        m = handle()
        m.integrate_depth(depth, np.eye(3)[None], np.zeros((1, 3)), submaps=[0])
        m.integrate_depth(depth, ref.rot([0, 1, 0], 5.0)[None], np.array([[0.1, 0.0, 0.05]]), submaps=[1])
        out[name] = m
    return out


@pytest.mark.parametrize("name", ["S1", "S2", "room"])
def test_normal_equations_integrated_scenes(scenes, name):
    m = scenes[name]
    for k, (R0, T0) in enumerate(((np.eye(3), np.zeros(3)), (ref.rot([0, 1, 0], -5.0), np.array([-0.1, 0.0, -0.05])),
                                  (ref.rot([1, 1, 0], 2.0), np.array([0.03, -0.04, 0.02])))):
        check_normal_equations(m, 0, m, 1, R0, T0)


def test_full_solves_match_reference(analytic, scenes):
    m, dR, dt = analytic
    for A, sa, sb, R0, T0 in ((m, 1, 0, np.eye(3), np.zeros(3)), (scenes["room"], 0, 1, np.eye(3), np.zeros(3))):
        got = A.register(A, [sa], [sb], R0[None], T0[None], BAND, 0.0, VS, max_iters=20, min_points=100)
        rd, (p, d) = ref_pair(A, sa, A, sb)
        want = ref.register(rd, p, d, R0, T0, VS, max_iters=20, min_points=100)
        et, er = ref.pose_error(got["R"][0], got["T"][0], want["R"], want["T"])
        assert et < 1e-6 and np.radians(er) < 1e-6, (et, er)
        assert got["iterations"][0] == want["iterations"] and got["converged"][0] == want["converged"]


@pytest.fixture(scope="module")
def room_pair():
    m = handle()
    for s, base, seeds in ((0, ref.ROOM_BASE_A, ref.ROOM_SEEDS_A), (1, ref.ROOM_BASE_B, ref.ROOM_SEEDS_B)):
        R, T = ref.local_pose(base)
        for sd in seeds:
            m.integrate_depth(syn.scene_room(seed=sd), R[None], T[None], submaps=[s])
    return m


@pytest.mark.parametrize("k", range(3))
def test_room_recovery(room_pair, k):
    Rt, tt = ref.true_relative(ref.ROOM_BASE_A, ref.ROOM_BASE_B)
    R0, T0 = ref.perturbed(Rt, tt, k)
    got = room_pair.register(room_pair, [0], [1], R0[None], T0[None], BAND)
    et, er = ref.pose_error(got["R"][0], got["T"][0], Rt, tt)
    assert et < 0.25 * VS and er < 0.25, (et, er)
    assert got["status"][0] == 0 and got["cost"][0] < got["cost_init"][0]


def test_s1_plane_recovers_depth_and_leaves_unobservable_components():
    m = handle()
    m.integrate_depth(syn.scene_plane(), np.eye(3)[None], np.zeros((1, 3)), submaps=[0])
    m.integrate_depth(syn.scene_plane(), np.eye(3)[None], np.array([[0.0, 0.0, 0.03]]), submaps=[1])
    # submap 1's plane lies 3 cm further along z in its local frame: the truth is t = (0, 0, 0.03)
    T0 = np.array([0.04, -0.03, 0.0])                          # in-plane offset, which the plane does not constrain
    got = m.register(m, [0], [1], np.eye(3)[None], T0[None], BAND)
    R, t = got["R"][0], got["T"][0]
    # the solve is the reference's on the same fields, step for step
    rd, (p, d) = ref_pair(m, 0, m, 1)
    want = ref.register(rd, p, d, np.eye(3), T0, VS)
    et, er = ref.pose_error(R, t, want["R"], want["T"])
    assert et < 1e-6 and np.radians(er) < 1e-6 and got["iterations"][0] == want["iterations"], (et, er)
    assert abs(t[2] - 0.03) < 0.25 * VS
    # An integrated plane is a frustum-limited patch with projective TSDF values, so the in-plane translation and the
    # rotation about the normal are constrained only weakly, through the patch's edges (the same solve on the CPU
    # oracle's S1 map moves them by 2.4 mm and 0.076 degrees); they must stay well inside the recovery bound.
    assert np.linalg.norm(t[:2] - T0[:2]) < 0.1 * VS, t
    assert abs(np.degrees(np.arctan2(R[1, 0], R[0, 0]))) < 0.1
    assert np.degrees(np.arccos(np.clip(R[2, 2], -1.0, 1.0))) < 0.25   # tilt of the normal


def test_batches_are_bit_identical_to_single_pairs_and_repeatable():
    m = handle()
    rng = np.random.default_rng(7)
    for s in range(4):
        R = ref.rot([0, 1, 0], 6.0 * s)
        m.integrate_depth(syn.scene_room(seed=3 + s), R[None], np.array([[0.05 * s, 0.0, 0.02 * s]]), submaps=[s])
    for P in (1, 7, 64):
        a = rng.integers(0, 4, P)
        b = rng.integers(0, 4, P)
        R0 = np.stack([ref.rot(rng.normal(size=3), rng.uniform(-3, 3)) for _ in range(P)])
        T0 = rng.uniform(-0.05, 0.05, (P, 3))
        batch = m.register(m, a, b, R0, T0, BAND, max_iters=8)
        again = m.register(m, a, b, R0, T0, BAND, max_iters=8)
        for key in batch:
            assert np.array_equal(bits(batch[key]), bits(again[key])), key
        for p in range(P):
            one = m.register(m, a[p:p + 1], b[p:p + 1], R0[p:p + 1], T0[p:p + 1], BAND, max_iters=8)
            for key in batch:
                assert np.array_equal(bits(batch[key][p:p + 1]), bits(one[key])), (P, p, key)


def test_cross_handle_submap_against_fused_global_map():
    from taichislam_b200.tsdf_handle import TsdfHandle
    col = handle(max_submaps=4)
    glob = TsdfHandle(256, 256, K=syn.K_DEPTH, max_ray_length=6.0, is_global_map=True)
    base = (ref.rot([0, 1, 0], 20.0), np.array([0.3, 0.0, 0.2]))
    R, T = ref.local_pose(base)
    col.integrate_depth(syn.scene_room(), R[None], T[None], submaps=[1])
    glob.set_submap_pose(1, *base)                             # fusion places submap 1 by the global map's pose table
    glob.fuse_from(col)
    R0, T0 = ref.perturbed(base[0], base[1], 0)
    check_normal_equations(col, 1, glob, 0, R0, T0)
    got = col.register(glob, [1], [0], R0[None], T0[None], BAND)
    et, er = ref.pose_error(got["R"][0], got["T"][0], base[0], base[1])
    assert got["status"][0] == 0 and et < 0.25 * VS and er < 0.25, (et, er)


def test_no_side_effects(room_pair):
    """Voxel rows (in key order), mesh and statistics of the map are the same bits before and after registering."""
    from util import tri_multiset
    rows = [as_dict_rows(*room_pair.gather(s)) for s in (0, 1)]
    n0, v0, _ = room_pair.marching_cubes()
    before = room_pair.stats()
    room_pair.register(room_pair, [0, 1], [1, 0], np.stack([np.eye(3)] * 2), np.zeros((2, 3)), BAND)
    after = room_pair.stats()
    # every statistic but the kernel-launch counter, which counts the call's own launches like every other call's
    assert after["launches"] > before["launches"]
    for k in before:
        if k != "launches":
            assert before[k] == after[k], k
    for s in (0, 1):
        for x, y in zip(rows[s], as_dict_rows(*room_pair.gather(s))):
            assert np.array_equal(bits(x), bits(y))
    n1, v1, _ = room_pair.marching_cubes()
    assert n0 == n1 and np.array_equal(tri_multiset(v0), tri_multiset(v1))


def test_refusals_and_status(room_pair):
    m = room_pair
    I, Z = np.eye(3)[None], np.zeros((1, 3))

    def refused(*args, **kw):
        with pytest.raises(capi.TslamError) as e:
            m.register(*args, **kw)
        assert e.value.code == capi.E_INVALID

    refused(m, [], [], np.zeros((0, 3, 3)), np.zeros((0, 3)), BAND)
    n = capi.REG_MAX_PAIRS + 1
    refused(m, [0] * n, [1] * n, np.stack([np.eye(3)] * n), np.zeros((n, 3)), BAND)
    refused(m, [16], [1], I, Z, BAND)
    refused(m, [0], [-1], I, Z, BAND)
    refused(m, [0], [1], I, np.array([[np.nan, 0, 0]]), BAND)
    refused(m, [0], [1], np.array([np.diag([np.inf, 1, 1])]), Z, BAND)
    refused(m, [0], [1], I, Z, 0.0)
    refused(m, [0], [1], I, Z, BAND, huber=0.0)
    refused(m, [0], [1], I, Z, BAND, max_iters=-1)
    refused(m, [0], [1], I, Z, BAND, min_weight=np.nan)
    refused(handle(128, 128, voxel_scale=0.04), [0], [1], I, Z, BAND)
    got = m.register(m, [0, 0], [1, 5], np.concatenate([I, I]), np.concatenate([Z, Z]), BAND, min_points=10 ** 9)
    assert np.array_equal(got["status"], [1, 1]) and np.array_equal(got["iterations"], [0, 0])
    got = m.register(m, [0, 0], [1, 5], np.concatenate([I, I]), np.concatenate([Z, Z]), BAND)
    assert np.array_equal(got["status"], [0, 1]) and got["n_valid"][1] == 0      # submap 5 is empty


def test_dense_tsdf_register_submaps_default_poses():
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    m = DenseTSDF(map_scale=[12.8, 12.8], voxel_scale=VS, num_voxel_per_blk_axis=16, max_ray_length=6.0, max_submap_num=4,
                  max_disp_particles=1 << 16)
    m.set_dep_camera_intrinsic(syn.K_DEPTH)
    for s, base, seeds in ((0, ref.ROOM_BASE_A, ref.ROOM_SEEDS_A), (1, ref.ROOM_BASE_B, ref.ROOM_SEEDS_B)):
        if s:
            m.switch_to_next_submap()
        m.set_base_pose_submap(s, *base)
        for sd in seeds:
            m.set_pose(np.eye(3), np.zeros(3))
            m.recast_depth_to_map(np.eye(3), np.zeros(3), syn.scene_room(seed=sd), None)
    Rt, tt = ref.true_relative(ref.ROOM_BASE_A, ref.ROOM_BASE_B)
    # drift: the stored base pose of submap 1 is off by a few centimetres and degrees after integration
    Rd, Td = ref.perturbed(ref.ROOM_BASE_B[0], ref.ROOM_BASE_B[1], 1)
    m.submaps_base_R_np[1], m.submaps_base_T_np[1] = Rd, Td
    (res,) = m.register_submaps([0], [1])
    et, er = ref.pose_error(res["R"], res["T"], Rt, tt)
    assert et < 0.25 * VS and er < 0.25 and res["status"] == 0, (et, er)
    R0, T0 = Rd.T @ ref.ROOM_BASE_A[0], Rd.T @ (ref.ROOM_BASE_A[1] - Td)
    direct = m._h.register(m._h, [0], [1], R0[None], T0[None], BAND)
    assert np.array_equal(direct["R"][0], res["R"]) and np.array_equal(direct["T"][0], res["T"])


def test_submap_mapping_align_submap_apply_moves_the_global_base_pose():
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    sub = dict(map_scale=[12.8, 12.8], voxel_scale=VS, num_voxel_per_blk_axis=16, max_ray_length=6.0, max_submap_num=8,
               max_disp_particles=1 << 16)
    glo = dict(map_scale=[25.6, 25.6], voxel_scale=VS, num_voxel_per_blk_axis=16, max_ray_length=6.0, max_submap_num=8,
               max_disp_particles=1 << 16)
    sm = SubmapMapping(DenseTSDF, sub_opts=sub, global_opts=glo, keyframe_step=2)
    sm.set_dep_camera_intrinsic(syn.K_DEPTH)
    ext = (np.eye(3), np.zeros(3))
    # the camera never moves; odometry reports a drifted pose from frame 2 on, so submap 1 is stored off by the drift
    drift = ref.perturbed(np.eye(3), np.zeros(3), 2)
    for fid in range(4):
        pose = (np.eye(3), np.zeros(3)) if fid < 2 else drift
        sm.recast_depth_to_map_by_frame(fid, True, pose, ext, syn.scene_room(seed=3 + fid), np.array([]))
    sm.submap_collection.finalization_current_submap()
    assert sm.submaps == {0: 0, 2: 1}
    res = sm.align_submap(2, apply=True)
    et, er = ref.pose_error(res["world_R"], res["world_T"], np.eye(3), np.zeros(3))
    assert et < 0.25 * VS and er < 0.25, (et, er)
    assert np.array_equal(sm.global_map.submaps_base_R_np[1], res["world_R"])
    assert np.array_equal(sm.global_map.submaps_base_T_np[1], res["world_T"])
