"""The frontier reference (octo_frontier_reference.py) on hand-worked answers.  Volume 16^3: cells in [-8, 8)."""
import numpy as np

import octo_frontier_reference as fr

N = NZ = 16
FREE_L, OCC_L, L_OCC = -415, 868, 0


def run(free=(), occ=()):
    free = np.asarray(free, np.int64).reshape(-1, 3)
    occ = np.asarray(occ, np.int64).reshape(-1, 3)
    idx = np.concatenate([free, occ]).astype(np.int32)
    L = np.concatenate([np.full(len(free), FREE_L), np.full(len(occ), OCC_L)]).astype(np.int32)
    return fr.frontiers(idx, L, L_OCC, N, NZ)


def k(i, j, k_):
    return ((i + 8) * N + (j + 8)) * NZ + (k_ + 8)


def test_lone_free_cell():
    fidx, cl, rec = run(free=[(0, 0, 0)])
    assert fidx.tolist() == [[0, 0, 0]] and cl.tolist() == [0]
    assert rec.tolist() == [[k(0, 0, 0), 1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 6, 0, 0, 0, 0]]


def test_free_slab_points_into_unknown():
    g = np.stack(np.meshgrid(np.arange(-8, 1), np.arange(-8, 8), np.arange(-8, 8), indexing="ij"), -1).reshape(-1, 3)
    fidx, cl, rec = run(free=g)                      # i <= 0 known FREE, i >= 1 UNKNOWN; every other face leaves the volume
    assert fidx.shape == (256, 3) and (fidx[:, 0] == 0).all() and (cl == 0).all()
    assert rec.shape == (1, 16)
    r = rec[0]
    assert r[0] == k(0, -8, -8) and r[1] == 256
    assert r[2:5].tolist() == [0, -128, -128]
    assert r[5:8].tolist() == [0, -8, -8] and r[8:11].tolist() == [0, 7, 7]
    assert r[11] == 256 and r[12:15].tolist() == [256, 0, 0] and r[15] == 0


def test_occupied_cell_is_never_a_frontier():
    fidx, cl, rec = run(occ=[(0, 0, 0)])
    assert fidx.shape == (0, 3) and rec.shape == (0, 16)
    fidx, cl, rec = run(free=[(1, 0, 0)], occ=[(0, 0, 0)])   # the OCC neighbour is known: 5 UNKNOWN faces
    assert fidx.tolist() == [[1, 0, 0]] and rec[0, 11] == 5 and rec[0, 12:15].tolist() == [1, 0, 0]


def test_fully_known_neighbourhood_is_not_a_frontier():
    g = np.stack(np.meshgrid(*[np.arange(-1, 2)] * 3, indexing="ij"), -1).reshape(-1, 3)
    fidx, cl, rec = run(free=g)
    assert fidx.shape == (26, 3) and not (fidx == 0).all(1).any()
    assert rec.shape == (1, 16) and rec[0, 1] == 26 and rec[0, 11] == 54 and rec[0, 12:15].tolist() == [0, 0, 0]


def test_volume_boundary_faces_do_not_count():
    fidx, cl, rec = run(free=[(-8, -8, -8)])
    assert rec[0, 11] == 3 and rec[0, 12:15].tolist() == [1, 1, 1]
    fidx, cl, rec = run(free=[(7, 0, 7)])
    assert rec[0, 11] == 4 and rec[0, 12:15].tolist() == [-1, 0, -1]
    assert rec[0, 0] == k(7, 0, 7) == (15 * N + 8) * NZ + 15


def test_corner_contact_joins_and_a_gap_separates():
    fidx, cl, rec = run(free=[(0, 0, 0), (1, 1, 1)])
    assert rec.shape == (1, 16) and rec[0, 1] == 2 and rec[0, 11] == 12
    fidx, cl, rec = run(free=[(0, 0, 0), (2, 0, 0)])
    assert rec.shape == (2, 16) and rec[:, 1].tolist() == [1, 1]
    assert rec[:, 0].tolist() == [k(0, 0, 0), k(2, 0, 0)]


def test_label_is_the_smallest_key_and_orders_the_list():
    # an L-shaped cluster whose first voxel in key order is not its first in any other order, and two singletons
    cl_a = [(3, 5, 0), (3, 4, 1), (2, 4, 2), (4, 4, 0)]
    fidx, cl, rec = run(free=cl_a + [(-5, 0, 0), (6, -7, 3)])
    labels = rec[:, 0]
    assert labels.tolist() == sorted(labels.tolist())
    assert labels.tolist() == [k(-5, 0, 0), k(2, 4, 2), k(6, -7, 3)]
    assert rec[:, 1].tolist() == [1, 4, 1]
    keys = fr.key(fidx, N, NZ)
    for c in range(3):
        assert keys[cl == c].min() == labels[c]
    assert rec[1, 2:5].tolist() == [12, 17, 3]
    assert rec[1, 5:11].tolist() == [2, 4, 0, 4, 5, 2]
