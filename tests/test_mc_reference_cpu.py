"""tests/mc_reference.py, the numpy statement of the marching-cubes mesher, pinned without a GPU: hand-worked single
cells with their expected bits written out, table-independent invariants on every mesh it makes, a closed and
consistently wound sphere, and bit equality with the CPU oracle's marching_cubes on the golden crop and a sphere."""
import os

import numpy as np
import pytest

import mc_reference as mcr

F = np.float32
HERE = os.path.dirname(os.path.abspath(__file__))
VS = 0.5


def bits(*x):
    return np.array(x, np.uint32).view(F)


def box(lo, hi, f):
    """Every voxel of the box [lo, hi] (inclusive) with T = f(i, j, k) in f32."""
    r = [np.arange(a, b + 1) for a, b in zip(lo, hi)]
    I, J, K = np.meshgrid(*r, indexing="ij")
    idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
    return idx, np.asarray(f(idx[:, 0], idx[:, 1], idx[:, 2]), np.float64).astype(F)


def with_values(idx, t, set_=None, drop=()):
    """Rows (idx, t, w, occ) with T overridden at the voxels of set_ ({(i, j, k): value}) and the voxels of drop removed."""
    t = t.copy()
    keep = np.ones(len(t), bool)
    pos = {tuple(v): n for n, v in enumerate(idx.tolist())}
    for v, x in (set_ or {}).items():
        t[pos[v]] = x
    for v in drop:
        keep[pos[v]] = False
    return idx[keep], t[keep], np.ones(int(keep.sum()), F), np.zeros(int(keep.sum()), np.int8)


def linear(set_=None, drop=()):
    """T = i + 2j + 4k - 0.5 on [-1, 2]^3: in cell (0, 0, 0) only corner 0 (-0.5) is negative, case 1, edges 0, 8, 3."""
    return with_values(*box((-1, -1, -1), (2, 2, 2), lambda i, j, k: i + 2 * j + 4 * k - 0.5), set_, drop)


def cell(rows, c=(0, 0, 0), step=1, thres=0.1, s=0):
    m = mcr.mesh({s: rows}, 64, 64, VS, step, thres)
    sel = np.all(m["tag"][:, :4] == np.array((s,) + tuple(c)), 1)
    d = {k: (x[sel] if isinstance(x, np.ndarray) else x) for k, x in m.items()}  # the cell's triangles
    return d["verts"], d["normals"], d


def u32(a):
    return np.ascontiguousarray(a, F).view(np.uint32)


# -- hand-worked cells -----------------------------------------------------------------------------------------------
def test_one_negative_corner():
    v, n, _ = cell(linear())
    assert v.shape == (1, 3, 3)
    # E0: mu = 0.5 / 1 -> x = 0.5; E8: mu = 0.5 / 4 -> z = 0.125; E3 (corner 3 -> 0): mu = -1.5 / -2 = 0.75 -> y = 1 - 0.75
    assert np.array_equal(u32(v[0]), u32([[0.25, 0, 0], [0, 0, 0.0625], [0, 0.125, 0]]))
    # gradient (2, 4, 8) at (1, 0, 0) (roundf(0.5) = 1) and at (0, 0, 0): / sqrt(84) in f32
    g = bits(0x3E5F7482, 0x3EDF7482, 0x3F5F7482)
    assert np.array_equal(u32(n[0]), u32(np.stack([g, g, g])))


def test_snap_branches():
    below, eps = bits(0x358637BC)[0], bits(0x358637BD)[0]  # nextafter(1e-6f, 0), 1e-6f
    assert eps == F(1e-6)
    v, _, m = cell(linear({(1, 0, 0): below}))       # |v2| < 1e-6f: E0's vertex is p2
    assert np.array_equal(u32(v[0, 0]), u32([0.5, 0, 0])) and m["snap"][0, 0] == 2
    v, _, m = cell(linear({(1, 0, 0): -below}))      # same, and -below is negative: corners 0 and 1 (case 3, two triangles)
    assert v.shape[0] == 2
    v, _, m = cell(linear({(1, 0, 0): eps}))         # |v2| == 1e-6f is not below: interpolated, mu = 0.5 / 0.500001
    assert np.array_equal(u32(v[0, 0]), np.array([0x3EFFFFDE, 0, 0], np.uint32)) and m["snap"][0, 0] == 0
    v, _, m = cell(linear({(0, 0, 0): F(-5e-7)}))    # |v1| < 1e-6f on all three edges of corner 0: every vertex is (0,0,0)
    assert v.shape[0] == 1 and np.array_equal(u32(v[0]), np.zeros((3, 3), np.uint32))
    assert m["snap"][0].tolist() == [1, 1, 2]        # (E3 runs from corner 3 to corner 0: p2)


def test_negative_zero_and_nan():
    v, _, _ = cell(linear({(1, 0, 0): F(-0.0)}))     # -0.0 is not negative: still case 1; |0 - -0| = 0 snaps to p2
    assert v.shape[0] == 1 and np.array_equal(u32(v[0, 0]), u32([0.5, 0, 0]))
    v, _, m = cell(linear({(0, 0, 0): F(-0.0)}))     # corner 0 = -0.0 passes the filter (< 0.1) but no corner is negative
    assert v.shape[0] == 0 and m["cand"] > 0
    v, _, _ = cell(linear({(0, 0, 0): F(np.nan)}))   # NaN fails T < thres: the cell is not meshed
    assert v.shape[0] == 0
    v, n, _ = cell(linear({(1, 0, 0): F(np.nan)}))   # NaN corner 1: not negative (case 1); E0: mu = NaN
    assert v.shape[0] == 1 and np.isnan(v[0, 0]).all() and np.isnan(n[0, 0]).all()
    assert np.array_equal(u32(v[0, 1]), u32([0, 0, 0.0625]))
    assert np.isnan(n[0, 1]).all()                   # its normal at (0, 0, 0) reads T(1, 0, 0) = NaN


def test_threshold_is_strict():
    rows = linear({(0, 0, 0): F(0.1), (1, 0, 0): F(-0.5)})   # case 2 if the cell is meshed
    assert cell(rows, thres=F(0.1))[0].shape[0] == 0
    assert cell(rows, thres=bits(0x3DCCCCCE)[0])[0].shape[0] == 1  # nextafter(0.1f, 1)


def test_half_tie_on_negative_coordinates_rounds_away_from_zero():
    """Cell (-3, 0, 0) with T(-3, ...) = -1, T(-2, ...) = 1 (+ j): E0's vertex is x = -2.5.  roundf gives -3, where the
    gradient is (3, 0, 0); rounding half to even (-2) would read (6, 2, 0)."""
    f = {-4: -2.0, -3: -1.0, -2: 1.0, -1: 5.0}
    rows = with_values(*box((-4, -1, -1), (-1, 2, 2), lambda i, j, k: np.vectorize(f.get)(i) + np.where(i == -2, j, 0)))
    v, n, m = cell(rows, c=(-3, 0, 0))
    at = np.all(u32(v) == u32([-1.25, 0, 0]), 2)
    assert at.sum() >= 1
    assert np.array_equal(u32(n[at]), np.tile(np.array([0x3F800000, 0, 0], np.uint32), (int(at.sum()), 1)))
    assert np.array_equal(m["at"][at], np.tile([-3, 0, 0], (int(at.sum()), 1)))


def test_normal_next_to_a_hole():
    v, n, m = cell(linear(drop=[(2, 0, 0)]))   # T(2, 0, 0) reads 0: nx = 0 - (-0.5) at (1, 0, 0)
    assert np.array_equal(u32(n[0, 0]), np.array([0x3D649DCE, 0x3EE49DCE, 0x3F649DCE], np.uint32))
    assert m["hole"][0].tolist() == [True, False, False]


def test_zero_gradient_gives_nan_normal():
    rows = with_values(*box((-1, -1, -1), (2, 2, 2), lambda i, j, k: np.where((i == 0) & (j == 0) & (k == 0), -1.0, 3.0)))
    v, n, _ = cell(rows)
    assert np.array_equal(u32(v[0]), u32([[0.125, 0, 0], [0, 0, 0.125], [0, 0.125, 0]]))  # mu = 1/4, 1/4, 3/4
    assert np.isnan(n).all()  # every vertex rounds to (0, 0, 0), whose six neighbours all read 3


def test_case_table_matches_edge_masks():
    """The parsed table against the edge masks of Bourke's edgeTable, restated from the corner signs: an edge is used by
    a case iff its corners differ in sign."""
    for c in range(256):
        neg = [(c >> q) & 1 for q in range(8)]
        want = {e for e, (a, b) in enumerate(mcr.EDGES) if neg[a] != neg[b]}
        got = set(mcr.TRI[c][mcr.TRI[c] >= 0].tolist())
        assert got == want, c


# -- invariants on every mesh --------------------------------------------------------------------------------------
def lookup(submaps):
    keys, t = [], []
    for s, g in submaps.items():
        i = np.asarray(g[0], np.int64)
        keys.append(((s * 4096 + i[:, 0] + 2048) * 4096 + i[:, 1] + 2048) * 4096 + i[:, 2] + 2048)
        t.append(np.asarray(g[1], F))
    keys, t = np.concatenate(keys), np.concatenate(t)
    o = np.argsort(keys)
    keys, t = keys[o], t[o]

    def read(s, ijk):
        k = ((s * 4096 + ijk[..., 0] + 2048) * 4096 + ijk[..., 1] + 2048) * 4096 + ijk[..., 2] + 2048
        p = np.minimum(np.searchsorted(keys, k), len(keys) - 1)
        return np.where(keys[p] == k, t[p], F(0))
    return read


def check_invariants(submaps, m, step, vs):
    """Edges used by each cell = its sign-change edges; every vertex on its edge between the corner positions."""
    n = m["tag"].shape[0]
    if n == 0:
        return
    read = lookup(submaps)
    tag = m["tag"]
    cp = tag[:, None, 1:4] + step * mcr.CORNERS[None]
    with np.errstate(invalid="ignore"):
        neg = read(tag[:, :1], cp) < 0
    e = m["edge"].astype(np.int64)
    a, b = mcr.EDGES[e, 0], mcr.EDGES[e, 1]
    r = np.arange(n)[:, None]
    assert np.all(neg[r, a] != neg[r, b]), "a vertex on an edge without a sign change"
    used = np.bitwise_or.reduce(np.left_shift(1, e), 1)
    first = np.r_[True, np.any(tag[1:, :4] != tag[:-1, :4], 1)]
    starts = np.nonzero(first)[0]
    cell_used = np.bitwise_or.reduceat(used, starts)
    ng = neg[starts]
    want = np.zeros(len(starts), np.int64)
    for q, (x, y) in enumerate(mcr.EDGES):
        want |= (ng[:, x] != ng[:, y]).astype(np.int64) << q
    assert np.array_equal(cell_used, want), "a cell's triangles miss a sign-change edge"
    # every vertex lies on its edge: off-axis coordinates are the corner's, the edge axis is between its two corners
    p1 = (cp[r, a].astype(F) * F(vs)).astype(F)
    p2 = (cp[r, b].astype(F) * F(vs)).astype(F)
    v = m["verts"]
    fin = np.isfinite(v).all(2)
    axis = (mcr.CORNERS[a] != mcr.CORNERS[b])
    lo, hi = np.minimum(p1, p2), np.maximum(p1, p2)
    ok = np.where(axis, (v >= lo) & (v <= hi), u32(v) == u32(p1))
    assert np.all(ok[fin])


def noise_map(seed, n=24):
    rng = np.random.default_rng(seed)
    idx, _ = box((-n // 2,) * 3, (n // 2 - 1,) * 3, lambda i, j, k: i * 0.0)
    t = rng.normal(0.3, 1.0, len(idx)).astype(F)
    t[rng.random(len(t)) < 0.03] = F(0)
    keep = rng.random(len(t)) > 0.05
    return idx[keep], t[keep], np.ones(int(keep.sum()), F), np.zeros(int(keep.sum()), np.int8)


@pytest.mark.parametrize("seed,step", [(0, 1), (1, 1), (2, 2), (3, 3)])
def test_invariants_on_noise(seed, step):
    rows = noise_map(seed)
    m = mcr.mesh({0: rows}, 64, 64, VS, step, 0.5)
    assert m["tag"].shape[0] > 500 and (m["snap"] > 0).any() and m["hole"].any()
    check_invariants({0: rows}, m, step, VS)


def sphere(c, r, half):
    """T = |p - c| - r (voxel units) on the cube of half-width `half` around round(c)."""
    c0 = np.round(c).astype(int)
    return box(c0 - half, c0 + half, lambda i, j, k: np.sqrt((i - c[0]) ** 2 + (j - c[1]) ** 2 + (k - c[2]) ** 2) - r)


@pytest.mark.parametrize("step", [1, 2])
def test_sphere_closed_and_oriented(step):
    idx, t = sphere(np.array([-3.3, 2.71, -0.45]), 7.13, 11)
    rows = (idx, t, np.ones_like(t), np.zeros(len(t), np.int8))
    m = mcr.mesh({0: rows}, 64, 64, VS, step, 100.0)  # (every cell: a threshold below the field's range opens the mesh)
    n = m["tag"].shape[0]
    assert n > 200 and not (m["snap"] > 0).any() and not m["hole"].any()
    check_invariants({0: rows}, m, step, VS)
    # no face of a meshed cell has the ambiguous (checkerboard) sign pattern
    read = lookup({0: rows})
    cp = m["tag"][:, None, 1:4] + step * mcr.CORNERS[None]
    neg = read(m["tag"][:, :1], cp) < 0
    for face in ([0, 1, 2, 3], [4, 5, 6, 7], [0, 1, 5, 4], [3, 2, 6, 7], [0, 3, 7, 4], [1, 2, 6, 5]):
        f = neg[:, face]
        assert not np.any((f[:, 0] == f[:, 2]) & (f[:, 1] == f[:, 3]) & (f[:, 0] != f[:, 1]))
    # closed: the vertex on a physical edge is named by the edge's two voxels; every side is shared by two triangles
    e = m["edge"].astype(np.int64)
    ends = np.stack([cp[np.arange(n)[:, None], mcr.EDGES[e, 0]], cp[np.arange(n)[:, None], mcr.EDGES[e, 1]]], 2)  # [n,3,2,3]
    ends = np.sort((ends + 64) @ np.array([1 << 16, 1 << 8, 1]), 2)                                           # [n,3,2]
    vid = ends[..., 0] * (1 << 24) + ends[..., 1]                                                           # [n,3]
    sides = np.sort(np.stack([vid[:, [0, 1]], vid[:, [1, 2]], vid[:, [2, 0]]], 1), 2).reshape(-1, 2)
    _, cnt = np.unique(sides, axis=0, return_counts=True)
    assert np.all(cnt == 2)
    # winding and vertex normals agree on every triangle: Bourke's table winds clockwise seen from where T grows, so the
    # right-handed face normal points against the vertex normals (the gradient of T)
    v = m["verts"].astype(np.float64)
    fn = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
    d = np.einsum("ij,ij->i", fn, m["normals"].astype(np.float64).sum(1))
    assert np.all(d < 0)


# -- the CPU oracle --------------------------------------------------------------------------------------------------
def test_oracle_golden_crop_bit_exact(oracle_lib):
    from oracle.oracle import OracleTSDF
    z = np.load(os.path.join(HERE, "golden", "ri_new_crop.npz"))
    vs = float(z["voxel_size"])
    o = OracleTSDF(map_scale=list(z["map_scale"]), voxel_scale=vs, is_global_map=True)
    rows = (z["indices"].astype(np.int32), z["TSDF"].astype(F), z["W_TSDF"].astype(F), z["occupy"])
    o.scatter(0, *rows)
    n, ov, on = o.marching_cubes(1, 5 * vs)
    m = mcr.mesh({0: o.gather(0)}, o.N, o.Nz, vs, 1, 5 * vs)
    assert m["tag"].shape[0] == n > 10000
    assert np.isnan(m["verts"]).any()  # the crop has NaN TSDF corners
    assert np.array_equal(mcr.sorted_rows(m["verts"], m["normals"]), mcr.sorted_rows(ov, on))
    check_invariants({0: o.gather(0)}, m, 1, vs)


@pytest.mark.parametrize("step", [1, 2, 3])
def test_oracle_sphere_bit_exact(oracle_lib, step):
    from oracle.oracle import OracleTSDF
    vs = 0.05
    o = OracleTSDF(map_scale=[6.4, 6.4], voxel_scale=vs, is_global_map=True)
    r = np.arange(-15, 15)
    I, J, K = np.meshgrid(r, r, r, indexing="ij")
    idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
    p = idx.astype(F) * F(vs)
    t = np.sqrt((p * p).sum(1)).astype(F) - F(3 * vs)
    o.scatter(0, idx, t, np.ones_like(t), np.zeros(len(t), np.int8))
    n, ov, on = o.marching_cubes(step, 0.1)
    m = mcr.mesh({0: o.gather(0)}, o.N, o.Nz, vs, step, 0.1)
    assert m["tag"].shape[0] == n > 10
    assert np.array_equal(mcr.sorted_rows(m["verts"], m["normals"]), mcr.sorted_rows(ov, on))
