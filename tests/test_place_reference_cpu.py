"""CPU checks of tests/place_reference.py, the numpy statement of loop detection's descriptors and matching: hand-worked
rings, sectors and cells (boundaries, rho^2 = 0, just inside and outside r_max), exact sector rotations and bitmap shifts
recovered, invariance to a vertical offset, every tie-break, eligibility, and a loop found on submaps the CPU oracle
integrated (tests/loop_world.py)."""
import math

import numpy as np
import pytest

import loop_world as lw
import place_reference as ref

F = np.float32
VS = 0.05


def pts(*rows):
    return np.array(rows, F).reshape(-1, 3)


def test_tables():
    B = ref.ring_bounds(8.0)
    assert B.dtype == F and B[0] == F(0.16) and B[-1] == F(64.0) and np.all(np.diff(B) > 0)
    c, s = ref.sector_table()
    assert c[0] == 1 and s[0] == 0 and c[60] == c[0] and s[60] == s[0] and 0 < c[15] < 1e-15 and s[15] == 1
    yc, ys = ref.yaw_table()
    assert yc.shape == (120,) and yc[0] == 1 and ys[30] == 1
    assert ref.cell_size(8.0) == F(0.125)


def test_hand_worked_rings_sectors_and_cells():
    # r_max = 2: rings 0.1 wide, B_0 = 0.01; cell 1/32
    x = pts([0.0, 0.0, 0.5],         # rho^2 = 0: ring 0, sector 0, cell (64, 64)
            [0.05, 0.0, 0.0],        # on the +x axis: f_0 = 0 >= 0, f_1 < 0 -> sector 0
            [0.0, 0.15, 0.0],        # on the +y axis (90 deg = the start of sector 15): ring 1, sector 15
            [-0.25, -1e-3, 0.0],     # just below the -x axis: sector 30 (f_30 = 1e-3 >= 0, f_31 < 0)
            [-0.25, 1e-3, 0.0],      # just above it: sector 29
            [1.99, 0.0, 0.0],        # just inside r_max: ring 19
            [2.0, 0.0, 0.0],         # on r_max: left out of the polar grid, cell (128 -> out)
            [-2.0, -2.0, 0.0],       # corner: outside the polar grid, cell (0, 0)
            [-1e-9, 0.0, 0.0])       # floor(-tiny / c) = -1: cell 63
    assert list(ref.rings_of(x, 2.0)) == [0, 0, 1, 2, 2, 19, -1, -1, 0]
    assert list(ref.sectors_of(x)) == [0, 0, 15, 30, 29, 0, 0, 37, 30]
    u, v = ref.cells_of(x, 2.0)
    assert list(u) == [64, 65, 64, 56, 56, 127, -1, 0, 63]
    assert list(v) == [64, 64, 68, 63, 64, 64, -1, 0, 64]


def test_descriptor_spans_ring_key_and_bitmap():
    x = pts([1.0, 0.0, 0.2], [1.0, 0.01, 1.4], [1.0, 0.02, 0.9],   # one bin, one cell: span 1.2
            [0.0, -1.0, 0.3])                                       # another bin: span 0
    d = ref.describe_points(x, 4.0, 0.5)
    r, s = ref.rings_of(x, 4.0), ref.sectors_of(x)
    assert d["sc"][r[0], s[0]] == F(F(1.4) - F(0.2)) and d["sc"][r[3], s[3]] == 0
    assert np.count_nonzero(d["sc"]) == 1
    assert r[0] == r[3] == 5  # rho^2 = 1 = B_4 exactly: not below it, so ring 5
    assert d["ring"][5] == F(2) / F(60) and np.count_nonzero(d["ring"]) == 1
    u, v = ref.cells_of(x, 4.0)
    assert d["bits"][u[0], v[0]] and d["bits"].sum() == 1                  # the span-0 cell marks floor, not structure
    w = 4 * u[0] + v[0] // 32
    assert d["bev"][w] == np.uint32(1 << (v[0] % 32)) and np.array_equal(ref.unpack(d["bev"]), d["bits"])


def scene(seed=0, n=4000):
    """Random vertical structure: posts of random heights around the origin."""
    rng = np.random.default_rng(seed)
    posts = rng.uniform(-5, 5, (40, 2))
    h = rng.uniform(0.2, 2.5, 40)
    k = rng.integers(0, 40, n)
    return np.concatenate([posts[k] + rng.normal(0, 0.02, (n, 2)), (rng.random(n) * h[k])[:, None]], 1).astype(F)


@pytest.mark.parametrize("k", [0, 1, 7, 30, 59])
def test_rotation_by_whole_sectors_gives_the_shift(k):
    x = scene(k)
    d0 = ref.describe_points(x, 8.0, 0.3)
    # the sector rule rotated by exactly k sectors is a roll of the polar grid's columns
    m, D = ref.best_shift(d0["sc"], np.roll(d0["sc"], k, axis=1))
    assert m == k and D == 0.0 or (m == k and abs(float(D)) < 1e-6)


def test_rotated_points_recover_the_yaw():
    x = scene(3)
    a = np.deg2rad(42.0)
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    y = (x.astype(np.float64) @ Rz.T).astype(F)
    m, D = ref.best_shift(ref.describe_points(x, 8.0, 0.3)["sc"], ref.describe_points(y, 8.0, 0.3)["sc"])
    assert m == 7 and D < 0.2


@pytest.mark.parametrize("dx,dy", [(0, 0), (5, 3), (-7, 2), (32, -32), (-1, -20)])
def test_bitmap_shift_is_recovered(dx, dy):
    b = ref.describe_points(scene(1), 8.0, 0.3)["bits"]
    c = np.zeros_like(b)
    c[max(dx, 0):128 + min(dx, 0), max(dy, 0):128 + min(dy, 0)] = b[max(-dx, 0):128 - max(dx, 0), max(-dy, 0):128 - max(dy, 0)]
    y, gx, gy, score, ov = ref.best_offset(b, c, 0)  # shift m = 0: yaws -3, 0, +3 degrees; the 0 yaw is exact
    assert (y, gx, gy) == (1, dx, dy) and score == c.sum() and ov == 1.0


def test_vertical_offset_changes_neither_ring_key_nor_spans():
    x = scene(2)
    y = x + np.array([0.0, 0.0, 0.75], F)
    a, b = ref.describe_points(x, 8.0, 0.3), ref.describe_points(y, 8.0, 0.3)
    assert np.array_equal(a["ring"], b["ring"]) and np.array_equal(a["bits"], b["bits"])
    assert np.allclose(a["sc"], b["sc"], atol=2e-6)  # the same spans up to the f32 rounding of the shifted heights


def test_tie_breaks():
    # shift: D equal at two shifts -> the smaller m; an all-zero descriptor gives D = 1 everywhere -> m = 0
    sc = np.zeros((20, 60), F)
    sc[3, 10] = sc[3, 40] = 1.0
    m, D = ref.best_shift(sc, sc)
    assert (m, D) == (0, 0.0)
    D_all = ref.shift_distances(sc, sc)
    assert D_all[30] == 0.0 and D_all[0] == 0.0  # the tie at m = 30 goes to m = 0
    assert ref.best_shift(np.zeros((20, 60), F), sc) == (0, 1.0)
    # offset: a symmetric pair of cells gives equal scores at +-d -> the smaller |dx| + |dy|, then dy, then dx
    b = np.zeros((128, 128), bool)
    b[64, 64] = True
    c = np.zeros_like(b)
    c[64, 66] = c[64, 62] = c[66, 64] = c[62, 64] = True
    y, dx, dy, score, ov = ref.best_offset(b, c, 0)
    assert (dx, dy, score) == (0, -2, 1) and y == 0  # equal |dx| + |dy| = 2: dy = -2 first; yaw index 0 before 1 and 2
    # empty bitmaps: score 0 everywhere -> (0, 0) at yaw index 0, overlap 0
    assert ref.best_offset(np.zeros_like(b), np.zeros_like(b), 5) == (0, 0, 0, 0, 0.0)
    # shortlist: equal ring distances -> the smaller index
    ring = np.zeros((4, 20), F)
    ring[0, 0] = 0.5
    assert [d for d, _ in ref.shortlist(0, ring, np.arange(4), np.full(4, 500), 3, 0, 200)] == [1, 2, 3]


def test_eligibility_and_min_gap():
    ring = np.zeros((5, 20), F)
    ids = np.array([10, 11, 12, 20, 30])
    npts = np.array([500, 500, 100, 500, 500])
    got = [d for d, _ in ref.shortlist(0, ring, ids, npts, 8, 2, 200)]
    assert got == [3, 4]                      # 1: |10 - 11| < 2; 2: too few points; never the query itself
    assert [d for d, _ in ref.shortlist(0, ring, ids, npts, 8, 0, 200)] == [1, 3, 4]
    assert ref.shortlist(2, ring, ids, npts, 8, 0, 200) == []  # a query with too few points matches nothing
    assert ref.eligible(0, 4, ids, npts, 20, 200) and not ref.eligible(0, 4, ids, npts, 21, 200)


@pytest.fixture(scope="module")
def oracle_loop(oracle_lib):
    """Submaps 0, 2 and N_LOOP - 1 of room A and the first of room B, each integrated by the CPU oracle in its local frame
    (camera at P_s^-1 P_f), described at the drifted base poses."""
    from oracle.oracle import OracleTSDF
    from taichislam_b200 import synthetic as syn
    S = [0, 2, lw.N_LOOP - 1, lw.N_LOOP]
    L = ref.level(lw.UP)
    desc, M = [], []
    for s in S:
        o = OracleTSDF(map_scale=[12.8, 12.8], K=syn.K_DEPTH, max_ray_length=6.0, is_global_map=True)
        Rb, tb = lw.true_pose(s, 0)
        for f in range(lw.FRAMES):
            R, t = lw.true_pose(s, f)
            o.integrate_depth(Rb.T @ R, Rb.T @ (t - tb), lw.render(s, f))
        idx, t, w, _ = o.gather(0)
        M.append(L @ lw.odometry_pose(s, 0)[0])
        desc.append(ref.describe_rows(idx, t, w, ref.levelled(L, lw.odometry_pose(s, 0)[0]), VS, 8.0, 0.3, 4 * VS))
    return S, desc, M


def test_oracle_loop_is_shortlisted_with_a_coarse_pose_near_the_truth(oracle_loop):
    S, desc, M = oracle_loop
    q = S.index(lw.N_LOOP - 1)
    info, dist = ref.match(desc, np.array(S), [q], 3, 2, 200)
    assert info[0, 0] == S.index(0), info          # the loop pair first by ring distance
    d, m, y, dx, dy, score = info[0]
    assert dist[0, 1] <= 0.35 and dist[0, 2] >= 0.3, dist[0]
    R0, T0 = ref.coarse_pose(M[q], M[d], m, y, dx, dy, 8.0)
    Rg, Tg = lw.relative(lw.N_LOOP - 1, 0)
    ang = np.degrees(np.arccos(np.clip((np.trace(R0 @ Rg.T) - 1) / 2, -1, 1)))
    assert ang <= 4.5 and np.linalg.norm(T0 - Tg) <= 3 * float(ref.cell_size(8.0)), (ang, T0, Tg)
