"""GPU: frame tracking against the TSDF (tslam_tsdf_track_depth / tslam_tsdf_track_points) against
tests/frame_track_reference.py: selected point counts, the normal equations at the initial pose, full solves,
known-answer recovery, batching and determinism, host and device input, point clouds, no side effects, the flush of
queued frames, every refusal and status, DenseTSDF.track_depth on a submap with a base pose, and drift along a
40-frame trajectory with noisy odometry."""
import numpy as np
import pytest

import frame_track_reference as ref
import submap_register_reference as reg
import track_world as tw
from taichislam_b200 import _capi as capi
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, compare_voxels

pytestmark = pytest.mark.gpu
F = np.float32
VS = 0.05
MIN_RAY, MAX_RAY = 0.3, 6.0


def handle(N=256, Nz=256, **kw):
    from taichislam_b200.tsdf_handle import TsdfHandle
    return TsdfHandle(N, Nz, K=syn.K_DEPTH, max_ray_length=MAX_RAY, min_ray_length=MIN_RAY, max_submaps=kw.pop("max_submaps", 16), **kw)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def reading(m, s=0):
    return ref.reading(m.gather(s), m.N, m.Nz, VS)


def check_normal_equations(m, depth, s, R0, T0, step):
    got = m.track_depth(depth, R0[None], T0[None], submaps=[s], step=step, max_iters=0, min_points=0)
    p = ref.select_depth(depth, syn.K_DEPTH, step, MIN_RAY, MAX_RAY)
    assert got["n_points"][0] == len(p)
    rd = reading(m, s)
    S = ref.normal_equations(rd, p, R0, T0, VS)
    A, _ = ref.abs_sums(rd, p, R0, T0, VS)
    assert got["n_valid"][0] == S[28]
    H = got["H"][0]
    k = 0
    for i in range(6):
        for j in range(i, 6):
            assert H[i, j] == H[j, i] and abs(H[i, j] - S[k]) <= 1e-9 * A[k], (i, j, H[i, j], S[k])
            k += 1
    assert np.all(np.abs(got["b"][0] - S[21:27]) <= 1e-9 * A[21:27])
    assert abs(got["cost"][0] - S[27]) <= 1e-9 * A[27] and got["cost_init"][0] == got["cost"][0]
    assert np.array_equal(got["R"][0], R0) and np.array_equal(got["T"][0], T0) and got["iterations"][0] == 0


@pytest.fixture(scope="module")
def scenes():
    """S1, S2, S4 and scene_room, each integrated into submap 0 at the identity."""
    out = {}
    for name, depth in (("S1", syn.scene_plane()), ("S2", syn.scene_sphere(4.0)), ("S4", syn.scene_noise()), ("room", syn.scene_room())):
        m = handle()
        m.integrate_depth(depth, np.eye(3)[None], np.zeros((1, 3)), submaps=[0])
        out[name] = (m, depth)
    return out


@pytest.fixture(scope="module")
def box_room():
    """Every fifth frame of the box-room trajectory integrated at its true pose into submap 0 (the CPU test's map)."""
    m = handle()
    for k in range(0, tw.N_FRAMES, 5):
        R, t = tw.pose(k)
        m.integrate_depth(tw.render(R, t, seed=k), R[None], t[None], submaps=[0])
    return m


def box_frame(k):
    Rt, tt = tw.pose(k)
    return tw.render(Rt, tt, seed=100 + k), Rt, tt


@pytest.mark.parametrize("step", [1, 2, 3])
def test_selected_counts_equal_the_reference(scenes, box_room, step):
    cases = [(m, d) for m, d in scenes.values()] + [(box_room, box_frame(21)[0])]
    cases.append((box_room, np.ascontiguousarray(box_frame(27)[0][:, 3:616])))     # width 613: not a multiple of 32
    for m, d in cases:
        got = m.track_depth(d, np.eye(3)[None], np.zeros((1, 3)), step=step, max_iters=0, min_points=0)
        assert got["n_points"][0] == len(ref.select_depth(d, syn.K_DEPTH, step, MIN_RAY, MAX_RAY)), (d.shape, step)


def test_normal_equations_at_t0(scenes, box_room):
    for name in ("S1", "S2", "room"):
        m, d = scenes[name]
        check_normal_equations(m, d, 0, reg.rot([1, 1, 0], 2.0), np.array([0.03, -0.04, 0.02]), 2)
    d, Rt, tt = box_frame(21)
    for step in (2, 3):
        check_normal_equations(box_room, d, 0, *tw.perturb(Rt, tt, np.random.default_rng(step)), step)


def test_full_solves_match_reference(scenes, box_room):
    d, Rt, tt = box_frame(27)
    m_room, d_room = scenes["room"]
    for m, dd, R0, T0, step in ((box_room, d, *tw.perturb(Rt, tt, np.random.default_rng(2)), 4),
                                (m_room, d_room, reg.rot([0, 1, 0], 2.0), np.array([0.02, 0.0, -0.03]), 2)):
        got = m.track_depth(dd, R0[None], T0[None], step=step)
        want = ref.track(reading(m), ref.select_depth(dd, syn.K_DEPTH, step, MIN_RAY, MAX_RAY), R0, T0, VS)
        et, er = reg.pose_error(got["R"][0], got["T"][0], want["R"], want["T"])
        assert et < 1e-6 and np.radians(er) < 1e-6, (et, er)
        assert got["iterations"][0] == want["iterations"] and got["converged"][0] == want["converged"]


# the CPU test's cases and bound (tests/test_frame_track_reference_cpu.py), on the GPU-integrated map
@pytest.mark.parametrize("case", range(4))
def test_box_room_recovery(box_room, case):
    import test_frame_track_reference_cpu as cpu
    k, s = cpu.RECOVERY[case]
    d, Rt, tt = box_frame(k)
    R0, T0 = tw.perturb(Rt, tt, np.random.default_rng(s))
    got = box_room.track_depth(d, R0[None], T0[None], step=cpu.ROOM_STEP)
    et, er = reg.pose_error(got["R"][0], got["T"][0], Rt, tt)
    assert got["status"][0] == 0 and got["cost"][0] < got["cost_init"][0]
    assert et < cpu.BOUND_T and er < cpu.BOUND_DEG, (et, er)


def test_batches_are_bit_identical_to_single_frames_and_repeatable(box_room):
    rng = np.random.default_rng(5)
    for n in (1, 7, 64):
        ks = rng.integers(0, tw.N_FRAMES, n)
        depth = np.stack([box_frame(int(k))[0] for k in ks])
        starts = [tw.perturb(*tw.pose(int(k)), rng, dt=0.03, deg=2.0) for k in ks]
        R0, T0 = np.stack([s[0] for s in starts]), np.stack([s[1] for s in starts])
        batch = box_room.track_depth(depth, R0, T0, max_iters=8)
        again = box_room.track_depth(depth, R0, T0, max_iters=8)
        for key in batch:
            assert np.array_equal(bits(batch[key]), bits(again[key])), key
        for f in range(n):
            one = box_room.track_depth(depth[f], R0[f:f + 1], T0[f:f + 1], max_iters=8)
            for key in batch:
                assert np.array_equal(bits(batch[key][f:f + 1]), bits(one[key])), (n, f, key)


def test_device_input_is_bit_identical_to_host_input(box_room):
    import torch
    d = np.stack([box_frame(k)[0] for k in (21, 27)])
    R0 = np.stack([tw.pose(k)[0] for k in (21, 27)])
    T0 = np.stack([tw.pose(k)[1] + 0.02 for k in (21, 27)])
    host = box_room.track_depth(d, R0, T0)
    dev = box_room.track_depth(torch.from_numpy(d.view(np.int16)).cuda(), R0, T0)
    for key in host:
        assert np.array_equal(bits(host[key]), bits(dev[key])), key
    Rt, tt = tw.pose(21)
    xyz = tw.cloud(Rt, tt)
    host = box_room.track_points(xyz, Rt, tt + 0.02)
    dev = box_room.track_points(torch.from_numpy(xyz).cuda(), Rt, tt + 0.02)
    for key in host:
        assert np.array_equal(bits(host[key]), bits(dev[key])), key


def test_track_points_matches_reference_and_ignores_zero_points(box_room):
    Rt, tt = tw.pose(27)
    xyz = tw.cloud(Rt, tt, seed=3)
    p = ref.select_points(xyz, MIN_RAY, MAX_RAY)
    zero = (xyz == 0).all(1)
    assert zero.sum() == 300 and not (p == 0).all(1).any()
    R0, T0 = tw.perturb(Rt, tt, np.random.default_rng(9))
    got = box_room.track_points(xyz, R0, T0)
    assert got["n_points"][0] == len(p)
    want = ref.track(reading(box_room), p, R0, T0, VS)
    et, er = reg.pose_error(got["R"][0], got["T"][0], want["R"], want["T"])
    assert et < 1e-6 and np.radians(er) < 1e-6 and got["iterations"][0] == want["iterations"], (et, er)
    # the same cloud without its zero points gives the same bits
    alone = box_room.track_points(xyz[~zero], R0, T0)
    for key in got:
        assert np.array_equal(bits(got[key]), bits(alone[key])), key


def test_no_side_effects(box_room):
    """Voxel rows, mesh and statistics of the map are the same bits before and after tracking."""
    from util import tri_multiset
    rows = as_dict_rows(*box_room.gather(0))
    n0, v0, _ = box_room.marching_cubes()
    before = box_room.stats()
    d, Rt, tt = box_frame(21)
    box_room.track_depth(d, Rt[None], tt[None])
    box_room.track_points(tw.cloud(Rt, tt), Rt, tt)
    after = box_room.stats()
    assert after["launches"] > before["launches"]
    for k in before:
        if k != "launches":
            assert before[k] == after[k], k
    for x, y in zip(rows, as_dict_rows(*box_room.gather(0))):
        assert np.array_equal(bits(x), bits(y))
    n1, v1, _ = box_room.marching_cubes()
    assert n0 == n1 and np.array_equal(tri_multiset(v0), tri_multiset(v1))


def test_queued_frames_are_flushed_first():
    import ctypes as C
    d, Rt, tt = box_frame(27)
    res = []
    for flush in (False, True):
        m = handle()
        for k in (20, 25, 30):
            R, t = tw.pose(k)
            dk = tw.render(R, t, seed=k)
            capi.check(m.L.tslam_tsdf_queue_depth(m.h, dk.ctypes.data_as(C.c_void_p), dk.shape[0], dk.shape[1],
                                                  capi.np_ptr(capi.f32c(R).reshape(9)), capi.np_ptr(capi.f32c(t)), 0, capi.stream_ptr()))
        if flush:
            capi.check(m.L.tslam_tsdf_flush(m.h, capi.stream_ptr()))
        res.append(m.track_depth(d, Rt[None], (tt + 0.02)[None]))
    assert res[0]["status"][0] == 0 and res[0]["n_valid"][0] > 1000
    for key in res[0]:
        assert np.array_equal(bits(res[0][key]), bits(res[1][key])), key


def test_refusals_and_status(box_room):
    m = box_room
    d = box_frame(21)[0]
    I, Z = np.eye(3)[None], np.zeros((1, 3))

    def refused(fn, *args, **kw):
        with pytest.raises(capi.TslamError) as e:
            fn(*args, **kw)
        assert e.value.code == capi.E_INVALID

    n = capi.REG_MAX_PAIRS + 1
    refused(m.track_depth, np.zeros((n, 4, 4), np.uint16), np.stack([np.eye(3)] * n), np.zeros((n, 3)))
    refused(m.track_depth, d, I, Z, step=0)
    refused(m.track_depth, np.zeros((0, 8), np.uint16), I, Z)
    refused(m.track_depth, d, I, Z, huber=0.0)
    refused(m.track_depth, d, I, Z, huber=np.nan)
    refused(m.track_depth, d, I, Z, max_iters=-1)
    refused(m.track_depth, d, I, Z, min_points=-1)
    refused(m.track_depth, d, I, Z, submaps=[16])
    refused(m.track_depth, d, I, Z, submaps=[-1])
    refused(m.track_depth, d, I, np.array([[np.nan, 0, 0]]))
    refused(m.track_depth, d, np.array([np.diag([np.inf, 1, 1])]), Z)
    refused(m.track_points, tw.cloud(*tw.pose(21)), np.eye(3), np.zeros(3), submap=16)
    refused(m.track_points, tw.cloud(*tw.pose(21)), np.eye(3), np.array([0, np.inf, 0]))
    refused(m.track_points, tw.cloud(*tw.pose(21)), np.eye(3), np.zeros(3), huber=-1.0)
    Rt, tt = tw.pose(21)
    got = m.track_depth(np.stack([d, d]), np.stack([Rt, Rt]), np.stack([tt, tt]), submaps=[0, 5])
    assert np.array_equal(got["status"], [0, 1]) and got["n_valid"][1] == 0 and got["iterations"][1] == 0   # submap 5 is empty
    assert np.array_equal(got["R"][1], Rt) and np.array_equal(got["T"][1], tt)
    got = m.track_points(np.zeros((10, 3), F), Rt, tt)                                   # nothing to track
    assert got["n_points"][0] == 0 and got["status"][0] == 1


def test_dense_tsdf_track_depth_on_a_submap_with_a_base_pose():
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF

    def dense():
        m = DenseTSDF(map_scale=[12.8, 12.8], voxel_scale=VS, num_voxel_per_blk_axis=16, max_ray_length=MAX_RAY, max_submap_num=4,
                      max_disp_particles=1 << 16)
        m.set_dep_camera_intrinsic(syn.K_DEPTH)
        m.switch_to_next_submap()
        m.set_base_pose_submap(1, *base)
        return m

    base = (reg.rot([0, 1, 0], 25.0) @ reg.rot([1, 0, 0], 4.0), np.array([0.4, -0.1, 0.3]))
    m = dense()
    for k in range(0, tw.N_FRAMES, 5):
        R, t = tw.pose(k)                                             # world poses: the map converts them by the base
        m.recast_depth_to_map(R, t, tw.render(R, t, seed=k), None)
    d, Rt, tt = box_frame(27)
    R0, T0 = tw.perturb(Rt, tt, np.random.default_rng(2))
    res = m.track_depth(R0, T0, d)
    assert res["status"] == 0 and res["iterations"] > 0
    Rb, Tb = base
    # the tracked pose is the local one carried back through the base pose, and it is the handle's answer
    assert np.array_equal(res["R"], Rb @ res["R_local"]) and np.array_equal(res["T"], Rb @ res["T_local"] + Tb)
    R0l, T0l = m.convert_by_base(R0, T0)
    direct = m._h.track_depth(d, R0l[None], T0l[None], submaps=[1])
    assert np.array_equal(direct["R"][0], res["R_local"]) and np.array_equal(direct["T"][0], res["T_local"])
    et, er = reg.pose_error(res["R"], res["T"], Rt, tt)
    assert et < 0.25 * VS and er < 0.25, (et, er)                    # achieved 6.0 mm, 0.12 degrees: the map's voxels sit
                                                                      # otherwise than in the box_room fixture's map
    # integrating at the returned pose through DenseTSDF integrates at T_local: the pose recast_depth_to_map hands to the
    # frame queue is f32(T_local), bit for bit, and the map matches a second one whose frame is handed over at T_local
    # through the handle.  The maps are compared as the oracle tests compare (index sets exact, values within 1e-4):
    # two handles fed the same frames through the queue differ in the last bits of some voxels (about 5 % of them,
    # |dTSDF| up to 1e-6), with or without a tracking call in between.
    m.set_pose(res["R"], res["T"])
    assert np.array_equal(m.input_R_np, res["R_local"].astype(F)) and np.array_equal(m.input_T_np, res["T_local"].astype(F))
    m.recast_depth_to_map(res["R"], res["T"], d, None)
    m._flush()
    m2 = dense()                                                      # m's calls, with the frame handed over at T_local
    for k in range(0, tw.N_FRAMES, 5):
        R, t = tw.pose(k)
        m2.recast_depth_to_map(R, t, tw.render(R, t, seed=k), None)
    m2.track_depth(R0, T0, d)
    Rl, Tl = capi.f32c(res["R_local"]).reshape(9), capi.f32c(res["T_local"])
    st = capi.stream_ptr()                                            # recast_depth_to_map's hand-over, pose T_local
    capi.check(m2._h.L.tslam_tsdf_queue_depth_begin(m2._h.h, capi.np_ptr(d), d.shape[0], d.shape[1], st))
    capi.check(m2._h.L.tslam_tsdf_queue_depth_end(m2._h.h, capi.np_ptr(Rl), capi.np_ptr(Tl), 1, st))
    m2._flush()
    compare_voxels(m._h.gather(1), m2._h.gather(1))
    # status 1 (an empty submap) returns the input bits
    m.switch_to_next_submap()
    m.set_base_pose_submap(2, *base)
    R0 = np.asarray(R0, np.float32)                                   # any dtype: the caller's values come back
    res = m.track_depth(R0, T0, d)
    assert res["status"] == 1 and np.array_equal(res["R"], R0) and np.array_equal(bits(res["T"]), bits(np.asarray(T0, np.float64)))


# Drift along the 40-frame trajectory: frame 0 integrated at its true pose, then every frame tracked at step 2 from the
# last tracked pose composed with a noisy odometry delta (tests/track_world.py odometry: ~5 mm and 0.2 degrees per step)
# and integrated at the tracked pose.  Huber threshold 1 cm (a fifth of a voxel): a young map's TSDF is carved into
# free space along the silhouettes of the boxes (rays that pass an edge cross the voxels of the box's side faces), so
# the residuals of a frame's points there are heavy-tailed (up to 12 cm on the boxes against the frame-0 map, 1 cm on the
# walls); with the default threshold of one voxel the pull of those points exceeds the odometry error.
# The CPU reference run of the same stream (oracle integration, tests/frame_track_reference.py solves) gives, in m and
# degrees, over frames 1-39:  tracked  mean 0.0147 / 0.264, max 0.0181 / 0.332, frame 39 0.0164 / 0.319;
#                             dead reckoning mean 0.0263 / 0.731, max 0.0432 / 1.385, frame 39 0.0199 / 0.961.
DRIFT_HUBER = 0.01
DRIFT_DEAD_MEAN = (0.02632663, 0.73131686)


def test_drift_along_the_trajectory_with_noisy_odometry():
    m = handle()
    odo = tw.odometry()
    R, t = tw.pose(0)
    m.integrate_depth(tw.render(R, t, seed=0), R[None], t[None])
    Rd, td = R, t
    err, dead = [], []
    for k in range(1, tw.N_FRAMES):
        dR, dt = odo[k - 1]
        R0, T0 = tw.compose(R, t, dR, dt)
        Rd, td = tw.compose(Rd, td, dR, dt)
        Rt, tt = tw.pose(k)
        d = tw.render(Rt, tt, seed=k)
        out = m.track_depth(d, R0[None], T0[None], step=2, huber=DRIFT_HUBER)
        assert out["status"][0] == 0, k
        R, t = out["R"][0], out["T"][0]
        m.integrate_depth(d, R[None], t[None])
        err.append(reg.pose_error(R, t, Rt, tt))
        dead.append(reg.pose_error(Rd, td, Rt, tt))
    err, dead = np.array(err), np.array(dead)
    assert np.allclose(dead.mean(0), DRIFT_DEAD_MEAN, rtol=1e-6)
    assert err.max(0)[0] < 0.025 and err.max(0)[1] < 0.5, err.max(0)          # CPU: 0.0181 m, 0.332 deg
    assert np.all(err.mean(0) < 0.7 * dead.mean(0)), (err.mean(0), dead.mean(0))  # CPU: 0.56, 0.36 of dead reckoning
    assert err[-1][1] < 0.5 * dead[-1][1], (err[-1], dead[-1])                  # CPU: 0.33 of it at frame 39
