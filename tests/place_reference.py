"""numpy statement of loop detection's place descriptors and matching (tslam_tsdf_place_describe, tslam_place_match;
csrc/tslam_place.cu; DESIGN.md section 7, "Loop detection").

Every f32 value below is one correctly rounded operation in the kernels' order (the library builds with -fmad=false), and
min, max and integer counts do not depend on order, so the GPU's outputs are these bits exactly.  The f64 tables are made
with the C library's cos and sin (math.cos / math.sin here), as the host code makes them.

Inputs are voxel rows as gather() returns them (idx int32[m,3] centred indices, tsdf, w f32[m] of the observed voxels of
one submap) and the levelled rotation M f32[3,3] of the submap.
"""
import math

import numpy as np

F = np.float32
NR, NS, G = 20, 60, 128
WORDS = G * G // 32
OFF = 32


# ---- frames ----------------------------------------------------------------------------------------------------------
def level(up=(0.0, 0.0, 1.0)):
    """L f64[3,3]: the minimal rotation taking the unit vector along `up` to +z (identity for +z; a half turn about x
    for -z)."""
    u = np.asarray(up, np.float64).reshape(3)
    if not np.all(np.isfinite(u)) or not np.linalg.norm(u) > 0.0:
        raise ValueError(f"up must be finite and non-zero, not {tuple(u)}")
    u = u / np.linalg.norm(u)
    z = np.array([0.0, 0.0, 1.0])
    v = np.cross(u, z)
    s2, c = float(v @ v), float(u @ z)
    if s2 == 0.0:
        return np.eye(3) if c > 0.0 else np.diag([1.0, -1.0, -1.0])
    K = np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])
    return np.eye(3) + K + K @ K * ((1.0 - c) / s2)


def levelled(L, R):
    """M_s = L R_s in f64, rounded to f32 once."""
    return (np.asarray(L, np.float64) @ np.asarray(R, np.float64)).astype(F)


def select(idx, tsdf, w, vs, band, min_weight=0.0):
    """p f32[n,3] of the registration points (tslam_tsdf_register's selection)."""
    idx, tsdf, w = np.asarray(idx, np.int32).reshape(-1, 3), np.asarray(tsdf, F), np.asarray(w, F)
    with np.errstate(invalid="ignore"):
        keep = (w > 0) & (w >= F(min_weight)) & (np.abs(tsdf) <= F(band))
    return idx[keep].astype(F) * F(vs)


def apply(M, p):
    """x = M p in f32, pose_apply's order with a zero translation: ((M0 px + M1 py) + M2 pz) + 0 per row."""
    M, p = np.asarray(M, F).reshape(3, 3), np.asarray(p, F).reshape(-1, 3)
    return np.stack([((M[i, 0] * p[:, 0] + M[i, 1] * p[:, 1]) + M[i, 2] * p[:, 2]) + F(0.0) for i in range(3)], 1).astype(F)


# ---- tables -----------------------------------------------------------------------------------------------------------
def ring_bounds(r_max):
    """B f32[20]: (f64(r_max) (i + 1) / 20)^2."""
    out = []
    for i in range(NR):
        r = float(F(r_max)) * float(i + 1) / 20.0
        out.append(r * r)
    return np.array(out).astype(F)


def sector_table():
    """(c, s) f32[61]: cos, sin(2 pi k / 60), k = 0 .. 60 (entry 60 = entry 0)."""
    a = [2.0 * math.pi * float(k % NS) / float(NS) for k in range(NS + 1)]
    return np.array([math.cos(x) for x in a]).astype(F), np.array([math.sin(x) for x in a]).astype(F)


def yaw_table():
    """(c, s) f32[120]: cos, sin(2 pi h / 120), the yaw h x 3 degrees."""
    a = [2.0 * math.pi * float(h) / float(2 * NS) for h in range(2 * NS)]
    return np.array([math.cos(x) for x in a]).astype(F), np.array([math.sin(x) for x in a]).astype(F)


def cell_size(r_max):
    return F(r_max) / F(64.0)


# ---- binning ----------------------------------------------------------------------------------------------------------
def rings_of(x, r_max):
    """ring int64[n] of levelled points x (-1: rho^2 >= B_19, left out)."""
    B = ring_bounds(r_max)
    r2 = (x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]).astype(F)
    ring = (r2[:, None] >= B[None, :]).sum(1)
    return np.where(r2 < B[-1], ring, -1)


def sectors_of(x):
    """sector int64[n]: the first k with f_k >= 0 and f_{k+1} < 0, f_k = c_k x1 - s_k x0 (f32); 0 when there is none."""
    c, s = sector_table()
    f = (c[None, :] * x[:, 1:2] - s[None, :] * x[:, 0:1]).astype(F)
    cond = (f[:, :NS] >= 0) & (f[:, 1:] < 0)
    return np.where(cond.any(1), np.argmax(cond, 1), 0)


def cells_of(x, r_max):
    """(u, v) int64[n] bird's-eye cells, -1 for points outside the grid."""
    c = cell_size(r_max)
    fu, fv = np.floor((x[:, 0] / c).astype(F)), np.floor((x[:, 1] / c).astype(F))
    ok = (fu >= -64) & (fu < 64) & (fv >= -64) & (fv < 64)
    return np.where(ok, fu.astype(np.int64) + 64, -1), np.where(ok, fv.astype(np.int64) + 64, -1)


def _span(index, z, size):
    zmin = np.full(size, np.inf, F)
    zmax = np.full(size, -np.inf, F)
    np.minimum.at(zmin, index, z)
    np.maximum.at(zmax, index, z)
    any_ = np.isfinite(zmin)
    return np.where(any_, (zmax - zmin).astype(F), F(0.0)).astype(F), any_


def describe_points(x, r_max, h_min):
    """Descriptor of levelled points x f32[n,3]: dict(sc f32[20,60], ring f32[20], bev uint32[512], bits bool[128,128])."""
    x = np.asarray(x, F).reshape(-1, 3)
    r, s = rings_of(x, r_max), sectors_of(x)
    k = r >= 0
    span, any_ = _span(r[k] * NS + s[k], x[k, 2], NR * NS)
    sc = span.reshape(NR, NS)
    ring = (any_.reshape(NR, NS).sum(1).astype(F) / F(60.0)).astype(F)
    u, v = cells_of(x, r_max)
    k = u >= 0
    bspan, bany = _span(u[k] * G + v[k], x[k, 2], G * G)
    bits = (bany & (bspan >= F(h_min))).reshape(G, G)
    return dict(sc=sc, ring=ring, bev=pack(bits), bits=bits)


def describe_rows(idx, tsdf, w, M, vs, r_max, h_min, band, min_weight=0.0):
    """Descriptor of one submap's gathered rows, levelled by M: describe_points plus n_points."""
    p = select(idx, tsdf, w, vs, band, min_weight)
    out = describe_points(apply(M, p), r_max, h_min)
    out["n_points"] = len(p)
    return out


def pack(bits):
    """bool[128,128] -> uint32[512]: bit v % 32 of word 4 u + v // 32."""
    b = np.asarray(bits, bool).reshape(G, G // 32, 32).astype(np.uint64)
    return (b << np.arange(32, dtype=np.uint64)).sum(2).astype(np.uint32).reshape(-1)


def unpack(words):
    w = np.asarray(words, np.uint32).reshape(G, G // 32, 1)
    return ((w >> np.arange(32, dtype=np.uint32)) & 1).astype(bool).reshape(G, G)


# ---- matching ---------------------------------------------------------------------------------------------------------
def eligible(q, d, ids, n_points, min_gap, min_points):
    return d != q and abs(int(ids[q]) - int(ids[d])) >= min_gap and n_points[q] >= min_points and n_points[d] >= min_points


def ring_distance(kq, kd):
    acc = F(0.0)
    for i in range(NR):
        t = F(kq[i] - kd[i])
        acc = F(acc + F(t * t))
    return acc


def shortlist(q, ring, ids, n_points, top_k, min_gap, min_points):
    """[(d, ring distance)] of the top_k eligible entries by (distance, index)."""
    c = [(ring_distance(ring[q], ring[d]), d) for d in range(len(ring)) if eligible(q, d, ids, n_points, min_gap, min_points)]
    c.sort()
    return [(d, dist) for dist, d in c[:top_k]]


def _col_norms(A):
    acc = np.zeros(NS, F)
    for i in range(NR):
        acc = (acc + (A[i] * A[i]).astype(F)).astype(F)
    return np.sqrt(acc).astype(F)


def shift_distances(scq, scd):
    """D f32[60]: D(m) for every shift m (x_d ~ Rz(6 m deg) x_q)."""
    A, B = np.asarray(scq, F).reshape(NR, NS), np.asarray(scd, F).reshape(NR, NS)
    na, nb = _col_norms(A), _col_norms(B)
    D = np.ones(NS, F)
    for m in range(NS):
        jb = (np.arange(NS) + m) % NS
        acc, nj = F(0.0), 0
        for j in range(NS):
            if not (na[j] != 0 and nb[jb[j]] != 0):
                continue
            dot = F(0.0)
            for i in range(NR):
                dot = F(dot + F(A[i, j] * B[i, jb[j]]))
            acc = F(acc + F(dot / F(na[j] * nb[jb[j]])))
            nj += 1
        D[m] = F(F(1.0) - F(acc / F(nj))) if nj else F(1.0)
    return D


def best_shift(scq, scd):
    """(m*, D(m*)): the argmin, ties to the smaller m."""
    D = shift_distances(scq, scd)
    m = int(np.argmin(D))  # np.argmin returns the first minimum
    return m, D[m]


def rotate_bits(bits, h):
    """q's bitmap rotated by the yaw h x 3 degrees (inverse mapping of cell centres by Rz(-psi) in f32)."""
    c, s = yaw_table()
    c, s = c[h], s[h]
    u, v = np.meshgrid(np.arange(G), np.arange(G), indexing="ij")
    a, b = ((u - 64).astype(F) + F(0.5)).astype(F), ((v - 64).astype(F) + F(0.5)).astype(F)
    xs = ((c * a).astype(F) + (s * b).astype(F)).astype(F)
    ys = ((c * b).astype(F) - (s * a).astype(F)).astype(F)
    fu, fv = np.floor(xs), np.floor(ys)
    ok = (fu >= -64) & (fu < 64) & (fv >= -64) & (fv < 64)
    su = np.where(ok, fu + 64, 0).astype(np.int64)
    sv = np.where(ok, fv + 64, 0).astype(np.int64)
    return ok & np.asarray(bits, bool)[su, sv]


def correlate(rq, bd):
    """score int64[65,65] indexed [dx + 32, dy + 32]: popc(rq shifted by (dx, dy) AND bd)."""
    from scipy.signal import fftconvolve
    full = fftconvolve(np.asarray(bd, np.float64), np.asarray(rq, np.float64)[::-1, ::-1], mode="full")
    out = full[G - 1 - OFF:G + OFF, G - 1 - OFF:G + OFF]
    r = np.rint(out)
    assert np.all(np.abs(out - r) < 0.25)
    return r.astype(np.int64)


def best_offset(bits_q, bits_d, m):
    """(y, dx, dy, score, overlap) over the yaws (2 m + y - 1) x 3 deg: the largest score, ties to the smaller |dx| + |dy|,
    then y, then dy, then dx."""
    rows = []
    pd = int(np.asarray(bits_d, bool).sum())
    for y in range(3):
        rq = rotate_bits(bits_q, (2 * m + y - 1) % (2 * NS))
        S = correlate(rq, bits_d)
        pq = int(rq.sum())
        dx, dy = np.meshgrid(np.arange(-OFF, OFF + 1), np.arange(-OFF, OFF + 1), indexing="ij")
        for a, b, sc in zip(dx.ravel(), dy.ravel(), S.ravel()):
            rows.append((-int(sc), abs(a) + abs(b), y, int(b), int(a), pq))
    rows.sort()
    neg, _, y, dy, dx, pq = rows[0]
    score, den = -neg, min(pq, pd)
    return y, dx, dy, score, (F(score) / F(den)) if den > 0 else F(0.0)


def match(desc, ids, queries, top_k, min_gap, min_points):
    """desc: list of dicts from describe_rows.  -> info6 int32[n_q top_k, 6], dist3 f32[n_q top_k, 3] as tslam_place_match."""
    ring = np.stack([d["ring"] for d in desc])
    npts = np.array([d["n_points"] for d in desc])
    info = np.zeros((len(queries) * top_k, 6), np.int32)
    dist = np.zeros((len(queries) * top_k, 3), F)
    info[:, 0] = -1
    dist[:, 1] = 1.0
    for qi, q in enumerate(queries):
        for k, (d, rd) in enumerate(shortlist(q, ring, ids, npts, top_k, min_gap, min_points)):
            m, D = best_shift(desc[q]["sc"], desc[d]["sc"])
            y, dx, dy, score, ov = best_offset(desc[q]["bits"], desc[d]["bits"], m)
            info[qi * top_k + k] = (d, m, y, dx, dy, score)
            dist[qi * top_k + k] = (rd, D, ov)
    return info, dist


# ---- coarse pose ------------------------------------------------------------------------------------------------------
def rz(deg):
    a = np.deg2rad(deg)
    return np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])


def coarse_pose(Mq, Md, m, y, dx, dy, r_max):
    """T0 = (Md^T Rz(psi) Mq, Md^T (dx c, dy c, 0)) in f64 from the f64 levelled rotations: the q-local -> d-local pose."""
    psi = 6.0 * m + 3.0 * (y - 1)
    c = float(cell_size(r_max))
    Mq, Md = np.asarray(Mq, np.float64), np.asarray(Md, np.float64)
    return Md.T @ rz(psi) @ Mq, Md.T @ np.array([dx * c, dy * c, 0.0])
