"""The submap registration reference (tests/submap_register_reference.py) pinned on hand-worked answers before any GPU
run is held to it: a plane recovered in one step with its unobservable components left alone, a three-plane corner
recovered in 6 DoF, each point filter and validity rule at its bound, and recovery of a known relative pose between two
submaps the CPU oracle integrated from scene_room frames."""
import numpy as np
import pytest

import submap_register_reference as ref

F = np.float32
VS = 0.05
N, NZ = 128, 64


def box_rows(lo, hi, fn):
    r = [np.arange(a, b) for a, b in zip(lo, hi)]
    I, J, K = np.meshgrid(*r, indexing="ij")
    idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
    return idx, np.asarray(fn(idx.astype(np.float64) * VS), F), np.ones(len(idx), F)


def plane(z0):
    return lambda x: x[:, 2] - z0


def corner(R=np.eye(3), t=np.zeros(3)):
    """min of three axis planes through (0.1, -0.05, 0.2), seen through the pose (R, t)."""
    def f(x):
        y = x @ R.T + t
        return np.minimum(np.minimum(y[:, 0] - 0.1, y[:, 1] + 0.05), y[:, 2] - 0.2)
    return f


LO, HI = (-24, -24, -16), (24, 24, 24)


def test_plane_one_step_and_unobservable_components_stay():
    ib, tb, wb = box_rows(LO, HI, plane(0.3))
    rd = ref.Reading(ib, tb, wb, N, NZ, VS)
    ia, ta, wa = box_rows(LO, HI, plane(0.3 + 0.02))           # the reference plane lies 2 cm higher: T moves it down
    p, d = ref.select_points(ia, ta, wa, VS, 4 * VS)
    S = ref.normal_equations(rd, p, d, np.eye(3), np.zeros(3), VS)
    H = ref.sym(S)
    assert np.linalg.matrix_rank(H, tol=1e-9 * np.abs(H).max()) == 3
    assert np.all(H[[0, 1, 5]] == 0) and np.all(S[[21, 22, 26]] == 0)   # rho_x, rho_y, phi_z unobservable
    out = ref.register(rd, p, d, np.eye(3), np.zeros(3), VS, max_iters=1, min_points=1)
    assert out["iterations"] == 1
    assert abs(out["T"][2] + 0.02) < 1e-5                        # one (damped) Gauss-Newton step on a linear field
    assert np.all(np.abs(out["T"][:2]) < 1e-7)                    # only through the exponential of a ~1e-7 rad tilt
    assert abs(out["R"][0, 1]) < 1e-9 and abs(out["R"][1, 0]) < 1e-9


@pytest.mark.parametrize("k", range(3))
def test_corner_recovers_six_dof_offsets(k):
    dt = [(0.03, -0.02, 0.01), (-0.02, 0.04, -0.03), (0.01, 0.01, 0.04)][k]
    dR = ref.rot([(1, 0, 0), (0, 1, 1), (1, 2, 3)][k], [3.0, -2.0, 2.5][k])
    # the reference voxels sample the corner field seen through the truth (dR, dt): f_A(p) = f_B(dR p + dt)
    ib, tb, wb = box_rows(LO, HI, corner())
    ia, ta, wa = box_rows(LO, HI, corner(dR, np.asarray(dt)))
    rd = ref.Reading(ib, tb, wb, N, NZ, VS)
    p, d = ref.select_points(ia, ta, wa, VS, 4 * VS)
    out = ref.register(rd, p, d, np.eye(3), np.zeros(3), VS, max_iters=30)
    et, er = ref.pose_error(out["R"], out["T"], dR, np.asarray(dt))
    assert et < 0.1 * VS and er < 0.1, (et, er, out["iterations"])


def test_huber_weight_and_cost_on_both_sides_of_delta():
    ib, tb, wb = box_rows((-4, -4, -4), (4, 4, 4), plane(0.0))
    rd = ref.Reading(ib, tb, wb, N, NZ, VS)
    p = np.array([[0.0, 0.0, 0.0]] * 3, F)
    d = np.array([-0.03, -0.05, -0.2], F)                     # r = 0.03 < delta, r = delta, r = 0.2 > delta
    q = ref.point_terms(rd, p, d, np.eye(3), np.zeros(3), VS)
    r = q["rv"]
    delta = float(F(VS))
    assert np.array_equal(q["w"][:2], [1.0, 1.0]) and q["w"][2] == delta / r[2]
    assert np.array_equal(q["rho"][:2], 0.5 * r[:2] * r[:2]) and q["rho"][2] == delta * (r[2] - 0.5 * delta)


def test_band_and_min_weight_bounds_are_inclusive():
    idx = np.array([[0, 0, k] for k in range(6)], np.int32)
    band = F(0.2)
    t = np.array([band, -band, np.nextafter(band, F(1)), 0.0, 0.0, 0.0], F)
    w = np.array([1.0, 1.0, 1.0, 2.0, np.nextafter(F(2), F(0)), 0.0], F)
    p, d = ref.select_points(idx, t, w, VS, band, min_weight=0.0)
    assert len(p) == 4                                         # the voxel just outside the band and W = 0 fail
    p, d = ref.select_points(idx, t, w, VS, band, min_weight=2.0)
    assert len(p) == 1 and p[0, 2] == F(3) * F(VS)             # W == min_weight is kept, W just below is not


def test_invalid_corners_unobserved_zero_weight_absent_block_and_volume_edge():
    ib, tb, wb = box_rows((-8, -8, -8), (24, 8, 8), plane(0.0))
    x = np.array([[0.12, 0.01, 0.01]], F)                     # low corner (2, 0, 0)
    d = np.zeros(1, F)

    def valid(idx, t, w, xx=x):
        return ref.point_terms(ref.Reading(idx, t, w, N, NZ, VS), xx, d, np.eye(3), np.zeros(3), VS)["valid"][0]

    assert valid(ib, tb, wb)
    corner_row = np.nonzero((ib == [3, 1, 1]).all(1))[0][0]
    keep = np.ones(len(ib), bool)
    keep[corner_row] = False
    assert not valid(ib[keep], tb[keep], wb[keep])             # unobserved corner
    w0 = wb.copy()
    w0[corner_row] = 0.0
    assert not valid(ib, tb, w0)                               # W = 0
    blk = (ib >> 4 == [1, 0, 0]).all(1)                        # every voxel of the block of the corners at i = 16
    xe = np.array([[0.77, 0.01, 0.01]], F)                     # low corner (15, 0, 0): the cube spans blocks 0 and 1
    assert valid(ib, tb, wb, xe) and not valid(ib[~blk], tb[~blk], wb[~blk], xe)
    # the volume edge: i0 + 1 must lie below N - N/2
    ie, te, we = box_rows((N // 2 - 4, -2, -2), (N // 2, 2, 2), plane(0.0))
    assert valid(ie, te, we, np.array([[(N // 2 - 2) * VS, 0.01, 0.01]], F))
    assert not valid(ie, te, we, np.array([[(N // 2 - 1) * VS + 0.01, 0.01, 0.01]], F))


def test_min_points_status():
    ib, tb, wb = box_rows(LO, HI, plane(0.3))
    rd = ref.Reading(ib, tb, wb, N, NZ, VS)
    p, d = ref.select_points(ib, tb, wb, VS, 4 * VS)
    n = ref.normal_equations(rd, p, d, np.eye(3), np.zeros(3), VS)[28]
    assert ref.register(rd, p, d, np.eye(3), np.zeros(3), VS, min_points=int(n))["status"] == 0
    out = ref.register(rd, p, d, np.eye(3), np.zeros(3), VS, min_points=int(n) + 1)
    assert out["status"] == 1 and out["iterations"] == 0 and np.array_equal(out["R"], np.eye(3))


@pytest.fixture(scope="module")
def room(oracle_lib):
    from oracle.oracle import OracleTSDF
    from taichislam_b200 import synthetic as syn
    o = OracleTSDF(map_scale=[12.8, 12.8], K=syn.K_DEPTH, max_ray_length=6.0)
    for s, base, seeds in ((0, ref.ROOM_BASE_A, ref.ROOM_SEEDS_A), (1, ref.ROOM_BASE_B, ref.ROOM_SEEDS_B)):
        R, T = ref.local_pose(base)
        for sd in seeds:
            o.integrate_depth(R, T, syn.scene_room(seed=sd), submap=s)
    ia, ta, wa, _ = o.gather(0)
    ib, tb, wb, _ = o.gather(1)
    return ref.Reading(ib, tb, wb, o.N, o.Nz, VS), ref.select_points(ia, ta, wa, VS, 4 * VS)


@pytest.mark.parametrize("k", range(3))
def test_room_submaps_recover_known_relative_pose(room, k):
    rd, (p, d) = room
    Rt, tt = ref.true_relative(ref.ROOM_BASE_A, ref.ROOM_BASE_B)
    R0, T0 = ref.perturbed(Rt, tt, k)
    out = ref.register(rd, p, d, R0, T0, VS)
    et, er = ref.pose_error(out["R"], out["T"], Rt, tt)
    assert et < 0.25 * VS and er < 0.25, (et, er)
    assert out["S"][27] < out["cost_init"]
