"""The viewpoint-gain reference (octo_view_gain_reference.py) on hand-worked answers.  Volume 32^3 (cells in [-16, 16)),
voxels of 0.5 m, views at cell centres with R = I (camera z along +k)."""
import numpy as np

import octo_view_gain_reference as vg

N = NZ = 32
VS = 0.5
FREE_L, OCC_L, L_OCC = -415, 868, 0
EYE = np.eye(3, dtype=np.float32)[None]
# a 1x1 image with cx = cy = 0: one ray, along +z
RAY = dict(fx=1.0, fy=1.0, cx=0.0, cy=0.0, width=1, height=1, step=1, max_range=4.0)


def rows(free=(), occ=()):
    free = np.asarray(free, np.int64).reshape(-1, 3)
    occ = np.asarray(occ, np.int64).reshape(-1, 3)
    idx = np.concatenate([free, occ]).astype(np.int32)
    L = np.concatenate([np.full(len(free), FREE_L), np.full(len(occ), OCC_L)]).astype(np.int32)
    return idx, L


def unknown(idx, L, pos, R=EYE, cam=RAY):
    return vg.unknown_gain(idx, L, L_OCC, N, NZ, VS, np.asarray(pos, np.float32).reshape(-1, 3), R, cam)


def test_one_ray_through_unknown_space_gains_max_range_over_vs():
    idx, L = rows(free=[(0, 0, 0)])
    valid, gain = unknown(idx, L, [0.0, 0.0, 0.0])
    assert valid.tolist() == [True] and gain.tolist() == [8]      # cells (0,0,1..8): 4 m / 0.5 m, end cell included


def test_occupied_cell_on_the_ray_stops_the_gain():
    idx, L = rows(free=[(0, 0, 0)], occ=[(0, 0, 5)])
    assert unknown(idx, L, [0.0, 0.0, 0.0])[1].tolist() == [4]    # (0,0,1..4)
    idx, L = rows(free=[(0, 0, 0), (0, 0, 1), (0, 0, 2)], occ=[(0, 0, 6)])
    assert unknown(idx, L, [0.0, 0.0, 0.0])[1].tolist() == [3]    # known FREE cells see through, gain nothing: (0,0,3..5)


def test_two_rays_sharing_cells_count_them_once():
    idx, L = rows(free=[(0, 0, 0)])
    cam = dict(RAY, width=2, fx=16.0)          # pixel 1: x = 4 / 16 = 0.25 m -> end cell (1,0,8), its x step comes last
    valid, gain = unknown(idx, L, [0.0, 0.0, 0.0], cam=cam)
    assert gain.tolist() == [9]                 # (0,0,1..8) shared, plus (1,0,8)


def test_view_at_the_volume_edge_counts_only_in_volume_cells():
    idx, L = rows(free=[(0, 0, 12)])
    assert unknown(idx, L, [0.0, 0.0, 6.0])[1].tolist() == [3]   # (0,0,13..15); 16..20 are outside


def test_invalid_views():
    idx, L = rows(free=[(0, 0, 0)], occ=[(1, 0, 0)])
    R = np.repeat(EYE, 5, 0)
    R[4, 1, 1] = np.nan
    pos = [[0.5, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 100.0], [np.nan, 0.0, 0.0], [0.0, 0.0, 0.0]]
    valid, gain = unknown(idx, L, pos, R)
    assert valid.tolist() == [False] * 5 and gain.tolist() == [0] * 5   # OCC, UNKNOWN, outside, NaN position, NaN in R


# -- frontier gain ---------------------------------------------------------------------------------------------------
SLAB = np.stack(np.meshgrid(np.arange(-4, 5), np.arange(-1, 2), np.arange(-4, 9), indexing="ij"), -1).reshape(-1, 3)
CAM = dict(fx=1.0, fy=1.0, cx=0.0, cy=0.0, width=3, height=1, step=1, max_range=3.0)


def frontier(fidx, fcl, nc, free=SLAB, occ=(), pos=(0.0, 0.0, 0.0), cam=CAM):
    free = [c for c in np.asarray(free).tolist() if c not in np.asarray(occ).reshape(-1, 3).tolist()]
    idx, L = rows(free, occ)
    return vg.frontier_gain(idx, L, L_OCC, N, NZ, VS, np.asarray(pos, np.float32).reshape(1, 3), EYE, cam,
                            np.asarray(fidx).reshape(-1, 3), np.asarray(fcl), nc)


def test_frontier_voxel_in_view_is_counted():
    valid, total, per = frontier([(0, 0, 4)], [0], 1)
    assert valid.tolist() == [True] and total.tolist() == [1] and per.tolist() == [[1]]


def test_frontier_voxel_behind_occ_or_unknown_is_not_visible():
    assert frontier([(0, 0, 4)], [0], 1, occ=[(0, 0, 2)])[1].tolist() == [0]
    free = [c for c in SLAB.tolist() if c != [0, 0, 2]]
    assert frontier([(0, 0, 4)], [0], 1, free=free)[1].tolist() == [0]   # (0,0,2) UNKNOWN: FUEL's conservative rule
    assert frontier([(0, 0, 4)], [0], 1, occ=[(0, 0, 4)])[1].tolist() == [1]  # only the cells before the voxel matter


def test_frustum_limits():
    # u = q_x fx / q_z + cx: (2,0,1) projects to u = 2 = width - 1 (counted), (3,0,1) to 3 and (-1,0,2) to -0.5 (outside);
    # (0,0,7) lies beyond max_range (3.5 m > 3 m) and (0,0,-2) behind the camera
    cases = [((2, 0, 1), 1), ((3, 0, 1), 0), ((-1, 0, 2), 0), ((0, 0, 7), 0), ((0, 0, -2), 0), ((0, 0, 6), 1)]
    for c, want in cases:
        assert frontier([c], [0], 1)[1].tolist() == [want], c


def test_counts_split_between_clusters():
    valid, total, per = frontier([(0, 0, 4), (2, 0, 1), (0, 0, 3), (3, 0, 1)], [0, 1, 0, 1], 2)
    assert total.tolist() == [3] and per.tolist() == [[2, 1]]


def test_invalid_view_gets_zero_frontier_gain():
    valid, total, per = frontier([(0, 0, 4)], [0], 1, pos=(0.0, 0.0, 20.0))
    assert valid.tolist() == [False] and total.tolist() == [0] and per.tolist() == [[0]]
