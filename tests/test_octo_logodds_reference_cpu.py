"""The numpy reference of the log-odds Octomap (octo_logodds_reference.py) on answers worked out by hand."""
import numpy as np
import pytest

import octo_logodds_reference as ref

VS = 0.05


def path(c0, c1, clipped=False):
    """Cells of the walk from cell c0 to cell c1 (points at the cell centres)."""
    o = np.asarray(c0, np.float32) * np.float32(VS)
    e = (np.asarray(c1, np.float32) * np.float32(VS)).reshape(1, 3)
    _, cells = ref.walk(o, e, np.array([True]), VS)  # clipped: every cell of the path is emitted
    return [tuple(int(v) for v in c) for c in cells]


def check_path(p, c0, c1):
    assert p[0] == tuple(c0) and p[-1] == tuple(c1)
    assert len(p) == int(np.abs(np.subtract(c1, c0)).sum()) + 1
    assert all(np.abs(np.subtract(a, b)).sum() == 1 for a, b in zip(p, p[1:]))  # 6-connected


def test_q10_defaults():
    assert ref.params() == dict(l_hit=868, l_miss=-415, l_min=-2048, l_max=3595, l_occ=0)


def test_tie_rule_diagonal():
    p = path((0, 0, 0), (3, 3, 0))
    assert p == [(0, 0, 0), (1, 0, 0), (1, 1, 0), (2, 1, 0), (2, 2, 0), (3, 2, 0), (3, 3, 0)]


@pytest.mark.parametrize("c1", [(5, 0, 0), (0, -4, 0), (0, 0, 7), (-3, 0, 0), (-2, -5, 3), (4, -1, -6), (-7, 7, -7)])
def test_paths_axis_negative_and_3d(c1):
    p = path((0, 0, 0), c1)
    check_path(p, (0, 0, 0), c1)
    if sum(v != 0 for v in c1) == 1:  # axis-aligned: a straight line
        ax = int(np.flatnonzero(c1)[0])
        assert [c[ax] for c in p] == list(range(0, c1[ax] + (1 if c1[ax] > 0 else -1), 1 if c1[ax] > 0 else -1))


def test_3d_diagonal_through_a_corner():
    # (0,0,0) -> (2,2,2) passes through the corners (0.5,0.5,0.5), (1.5,1.5,1.5): all three axes tie, x then y then z
    p = path((0, 0, 0), (2, 2, 2))
    assert p == [(0, 0, 0), (1, 0, 0), (1, 1, 0), (1, 1, 1), (2, 1, 1), (2, 2, 1), (2, 2, 2)]


def test_off_centre_endpoints_keep_the_cell_count():
    rng = np.random.default_rng(0)
    o = np.array([0.013, -0.021, 0.007], np.float32)
    e = rng.uniform(-1.5, 1.5, (500, 3)).astype(np.float32)
    rays, cells = ref.walk(o, e, np.ones(500, bool), VS)
    c0 = ref.cells(o, VS).reshape(3)
    c1 = ref.cells(e, VS)
    for r in range(500):
        p = [tuple(c) for c in cells[rays == r]]
        check_path(p, tuple(c0), tuple(c1[r]))


def m_points(**kw):
    return ref.LogoddsMap(256, 256, VS, min_ray_length=0.0, max_ray_length=kw.pop("max_ray_length", 3.0), **kw)


def L_of(m, c):
    known, val = m._lookup(np.asarray([c]), 0)
    return int(val[0]) if known[0] else None


def test_zero_length_ray_gives_a_hit_only():
    m = m_points()
    m.integrate_points(np.array([[0.01, 0.0, 0.0]], np.float32), np.eye(3), np.zeros(3))
    idx, L = m.gather()
    assert idx.tolist() == [[0, 0, 0]] and L.tolist() == [868]
    assert m.stats.tolist() == [1, 0, 1, 1]


def test_hit_wins_over_miss_in_one_frame():
    m = m_points()
    # ray A ends in cell (2,0,0); ray B runs on to (5,0,0) through it
    pts = np.array([[2 * VS, 0, 0], [5 * VS, 0, 0]], np.float32)
    m.integrate_points(pts, np.eye(3), np.zeros(3))
    assert L_of(m, (2, 0, 0)) == 868 and L_of(m, (5, 0, 0)) == 868
    assert [L_of(m, (i, 0, 0)) for i in (0, 1, 3, 4)] == [-415] * 4
    assert m.stats.tolist() == [2, 2 + 5, 2, 6]   # visits: A (0,1), B (0..4)


def test_clamp_sequence_defaults():
    m = m_points(max_ray_length=5.0)
    hit = np.array([[2.0, 0.0, 0.0]], np.float32)    # cell (40, 0, 0)
    far = np.array([[4.0, 0.0, 0.0]], np.float32)
    for f in range(5):
        m.integrate_points(hit, np.eye(3), np.zeros(3))
    assert L_of(m, (40, 0, 0)) == 3595 and L_of(m, (20, 0, 0)) == -2048   # crossed 5 times: exactly l_min
    for f in range(1, 10):
        m.integrate_points(far, np.eye(3), np.zeros(3))
        occ = m.occupied_cells(np.array([[40, 0, 0]]))[0][0]
        assert L_of(m, (40, 0, 0)) == 3595 - 415 * f
        assert occ == (f <= 8), f


def test_clipped_point_gives_misses_only():
    m = m_points(max_ray_length=1.0)
    m.integrate_points(np.array([[2.0, 0.0, 0.0]], np.float32), np.eye(3), np.zeros(3))
    idx, L = m.gather()
    assert sorted(idx[:, 0].tolist()) == list(range(0, 21)) and (L == -415).all()   # cut at 1 m = cell 20, which is a miss
    assert m.stats.tolist() == [1, 21, 0, 21]


def test_depth_clip_and_range_filter():
    m = ref.LogoddsMap(128, 128, VS, min_ray_length=0.3, max_ray_length=2.0, recast_step=1, K=[100, 0, 2, 0, 100, 2, 0, 0, 1])
    d = np.array([[0, 200, 1500, 5000]] * 4, np.uint16)
    e, cl = ref.depth_endpoints(d, np.eye(3), np.zeros(3), m.K, m.min_ray, m.max_ray, 1)
    assert e.shape[0] == 8 and cl.tolist() == [False, True] * 4
    assert np.allclose(e[1::2, 2], 2.0)   # cut at depth max_ray_length along the pixel ray


def test_fusion_sums_then_one_clamp():
    src = m_points()
    dst = ref.LogoddsMap(64, 64, VS)
    src.maps = {0: (ref.pack([[1, 0, 0], [2, 0, 0]]), np.array([3000, -2000], np.int32)),
                1: (ref.pack([[1, 0, 0], [2, 0, 0], [3, 0, 0]]), np.array([3000, -2000, 5], np.int32))}
    ref.fuse(dst, src, {0: (np.eye(3), np.zeros(3)), 1: (np.eye(3), np.zeros(3))})
    idx, L = dst.gather()
    assert idx[:, 0].tolist() == [1, 2, 3] and L.tolist() == [3595, -2048, 5]
    # a shifted base pose moves the contribution to another cell, where it is summed alone
    ref.fuse(dst, src, {0: (np.eye(3), np.zeros(3)), 1: (np.eye(3), np.array([VS, 0, 0]))})
    idx, L = dst.gather()
    assert idx[:, 0].tolist() == [1, 2, 3, 4] and L.tolist() == [3000, 1000, -2000, 5]


def test_queries_and_lod():
    m = m_points()
    m.maps = {0: (ref.pack([[0, 0, 0], [2, 0, 0], [3, 0, 0]]), np.array([10, 0, -5], np.int32))}
    occ, unk = m.query_points(np.array([[0, 0, 0], [2 * VS, 0, 0], [3 * VS, 0, 0], [VS, 0, 0]], np.float32))
    assert occ.tolist() == [True, False, False, False] and unk.tolist() == [False, False, False, True]
    assert m.query_near(np.array([[VS, 0, 0], [2 * VS, 0, 0]], np.float32), 1).tolist() == [True, False]
    hit, x, ln = m.raycast(np.array([[-5 * VS, 0, 0]], np.float32), np.array([[1, 0, 0]], np.float32), 1.0)
    assert hit[0] and abs(ln[0] - 5 * VS) < 1e-6
    assert m.export(1).shape == (1, 3) and m.export(2).shape == (1, 3) and m.export(3).shape == (1, 3)
