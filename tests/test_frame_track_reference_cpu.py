"""The frame-tracking reference (tests/frame_track_reference.py) pinned on hand-worked answers before any GPU run is held
to it: both selection rules at their bounds with exact f32 values, a fronto-parallel plane recovered in one step with
its in-plane components left alone, and recovery of box-room camera poses on a map the CPU oracle integrated."""
import numpy as np
import pytest

import frame_track_reference as ref
import submap_register_reference as reg
import track_world as tw

F = np.float32
VS = 0.05
K_SMALL = [500.0, 0.0, 4.5, 0.0, 250.0, 3.25, 0.0, 0.0, 1.0]


def small_depth():
    d = np.full((7, 10), 2000, np.uint16)
    d[0, 2] = 0                  # dropout
    d[2, 4] = 150                # nearer than min_ray (0.3 m)
    d[4, 6] = 20000              # farther than max_ray (6 m)
    d[2, 2] = 300                # exactly min_ray: kept
    d[4, 4] = 6000               # exactly max_ray: kept
    d[6, 6] = 6001               # just beyond: dropped
    d[3, 3] = 1500
    return d


# step 1: 70 pixels, four dropped (the dropout, too near, too far, just beyond); step 2: rows 0 2 4 x columns 0 2 4 6 8,
# three of them dropped; step 3: rows 0 3 x columns 0 3 6 (7 // 3 = 2 rows, 10 // 3 = 3 columns), none dropped
@pytest.mark.parametrize("step,kept", [(1, 70 - 4), (2, 3 * 5 - 3), (3, 2 * 3)])
def test_depth_selection_steps_and_filter(step, kept):
    p = ref.select_depth(small_depth(), K_SMALL, step, 0.3, 6.0)
    assert p.shape == (kept, 3) and p.dtype == F


def test_depth_selection_exact_values_and_order():
    p = ref.select_depth(small_depth(), K_SMALL, 1, 0.3, 6.0)
    # pixel (0, 0): dep = 2, x = ((0 - 4.5) 2) / 500 = -0.018, y = ((0 - 3.25) 2) / 250 = -0.026, each correctly rounded
    assert np.array_equal(p[0], [F(-0.018), F(-0.026), F(2.0)])
    # the second record is pixel (1, 0) (row-major), the third (3, 0): (2, 0) is the dropout
    assert p[1][0] == F(-0.014) and p[2][0] == F(-0.006)
    # pixel (3, 3), 1500 mm: x = ((3 - 4.5) 1.5) / 500 = -0.0045, y = (-0.25 1.5) / 250 = -0.0015; record 31, after the
    # 33 pixels of rows 0-2 and row 3's first three, less the two dropped before it ((2, 0) and (4, 2))
    assert np.array_equal(p[31], [F(-0.0045), F(-0.0015), F(1.5)])
    assert (p[:, 2] == F(0.3)).sum() == 1 and (p[:, 2] == F(6.0)).sum() == 1
    assert not np.any(p[:, 2] == F(0.15)) and not np.any(p[:, 2] > F(6.0))


def test_cloud_selection_bounds_and_nonfinite():
    x = np.array([[0, 0, 0], [0, 0, 0.3], [0, 0, np.nextafter(F(0.3), F(0))], [0, 0, 6.0], [0, 0, np.nextafter(F(6), F(0))],
                  [np.nan, 0, 1], [np.inf, 0, 1], [1e30, 0, 0], [3, 4, 0]], F)
    p = ref.select_points(x, 0.3, 6.0)
    # kept: r = 0.3 (the lower bound is inclusive), r just below 6, and (3, 4, 0) with r = 5, in input order
    assert np.array_equal(p, x[[1, 4, 8]])


def plane_rows(z0, lo=(-12, -12, 14), hi=(12, 12, 27)):
    r = [np.arange(a, b) for a, b in zip(lo, hi)]
    I, J, K = np.meshgrid(*r, indexing="ij")
    idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
    return idx, (idx[:, 2].astype(np.float64) * VS - z0).astype(F), np.ones(len(idx), F)


def test_plane_frame_depth_in_one_step_in_plane_components_stay():
    rd = reg.Reading(*plane_rows(1.0), 128, 128, VS)
    depth = np.full((24, 32), 1020, np.uint16)                  # the frame sees the plane 2 cm further away
    p = ref.select_depth(depth, [40.0, 0, 16.0, 0, 40.0, 12.0, 0, 0, 1], 1, 0.3, 6.0)
    assert len(p) == 24 * 32
    T0 = np.array([0.03, -0.02, 0.0])
    S = ref.normal_equations(rd, p, np.eye(3), T0, VS)
    H = reg.sym(S)
    assert np.linalg.matrix_rank(H, tol=1e-9 * np.abs(H).max()) == 3   # rho_x, rho_y, phi_z unobservable
    out = ref.track(rd, p, np.eye(3), T0, VS, max_iters=1, min_points=1)
    assert out["iterations"] == 1
    assert abs(out["T"][2] + 0.02) < 1e-5                       # one (damped) Gauss-Newton step on a linear field
    assert np.all(np.abs(out["T"][:2] - T0[:2]) < 1e-7)
    assert abs(out["R"][0, 1]) < 1e-9 and abs(out["R"][1, 0]) < 1e-9


# Recovery in the box room: the CPU oracle integrates every fifth frame of the trajectory at its true pose; frames
# 21, 27 and 33 (not integrated, other dropout seeds) are tracked at step 4 from starts perturbed by 5 cm and 3 degrees.
# Achieved (translation mm, rotation deg): 4.25 / 0.122 and 4.25 / 0.122 (frame 21), 3.16 / 0.056 (27), 4.13 / 0.065
# (33).  The solver lands where it lands from the true pose too (within 0.03 mm): what is left is the integrated map's
# bias - its zero level is a projective TSDF of eight views - not a shortfall of the solve.  Some views are weaker still:
# frame 12, which sees mostly the far wall and the floor, settles 1.9 cm / 0.35 degrees from the truth.
ROOM_STEP = 4
RECOVERY = [(21, 0), (21, 1), (27, 2), (33, 3)]
BOUND_T, BOUND_DEG = 0.12 * VS, 0.15


@pytest.fixture(scope="module")
def room(oracle_lib):
    from oracle.oracle import OracleTSDF
    from taichislam_b200 import synthetic as syn
    o = OracleTSDF(map_scale=[12.8, 12.8], K=syn.K_DEPTH, max_ray_length=6.0, is_global_map=True)
    for k in range(0, tw.N_FRAMES, 5):
        R, t = tw.pose(k)
        o.integrate_depth(R, t, tw.render(R, t, seed=k))
    return ref.reading(o.gather(0), o.N, o.Nz, VS)


@pytest.mark.parametrize("case", range(len(RECOVERY)))
def test_box_room_recovery(room, case):
    from taichislam_b200 import synthetic as syn
    k, s = RECOVERY[case]
    Rt, tt = tw.pose(k)
    p = ref.select_depth(tw.render(Rt, tt, seed=100 + k), syn.K_DEPTH, ROOM_STEP, 0.3, 6.0)
    R0, T0 = tw.perturb(Rt, tt, np.random.default_rng(s))
    out = ref.track(room, p, R0, T0, VS)
    et, er = reg.pose_error(out["R"], out["T"], Rt, tt)
    e0 = reg.pose_error(R0, T0, Rt, tt)
    assert e0[0] > 0.02 and e0[1] > 2.9                           # dt of 5 cm applied on the left, after the 3-degree turn
    assert out["status"] == 0 and out["S"][27] < out["cost_init"]
    assert et < BOUND_T and er < BOUND_DEG, (et, er, out["iterations"])
