"""numpy reference of the incremental global fusion (tslam_tsdf_fuse_update, DESIGN.md section 7).

Every observed source voxel (i, j, k) of a submap placed at pose (R, T) lands at g = pose_apply(i vs, j vs, k vs) / vs
(f32, the expression order of k_fuse) and splats into the 7 upper corners lo + (c >> 2 & 1, c >> 1 & 1, c & 1),
c = 1 .. 7, of lo = floor(g), with weight wt = (1 - |ci - gx|)(1 - |cj - gy|)(1 - |ck - gz|).  Its terms w = W wt, w T
and (textured) w c are f32; each is quantised to q = rint(f * 2^24) and summed exactly in int64, together with a
contribution count and the sum of occ.  A voxel with a term (of an in-volume corner) that is not finite or has
|f| >= 2^23 adds nothing.  The readout is T = f32(S_wT / S_w), W = f32(S_w 2^-24), occ = clip(S_occ), colour =
f32(S_c / S_w) in f64, for every voxel with count > 0.
"""
import numpy as np

Q = 2.0 ** 24
FMAX = np.float32(2.0 ** 23)


def place(idx, R, T, vs):
    """g = pose_apply(idx * vs) / vs in f32 (the build's -fmad=false order), and lo = floor(g)."""
    vs = np.float32(vs)
    R = np.asarray(R, np.float32).reshape(3, 3)
    T = np.asarray(T, np.float32).reshape(3)
    lx, ly, lz = (np.asarray(idx, np.int64)[:, a].astype(np.float32) * vs for a in range(3))
    g = []
    for r in range(3):
        x = ((R[r, 0] * lx + R[r, 1] * ly) + R[r, 2] * lz) + T[r]
        g.append((x / vs).astype(np.float32))
    g = np.stack(g, 1)
    return g, np.floor(g).astype(np.int64)


def corners(g, lo):
    """[7, n, 3] corner cells and [7, n] f32 weights."""
    cells, wts = [], []
    one = np.float32(1.0)
    for c in range(1, 8):
        d = np.array([(c >> 2) & 1, (c >> 1) & 1, c & 1], np.int64)
        ci = lo + d
        f = ci.astype(np.float32)
        w = (one - np.abs(f[:, 0] - g[:, 0])) * (one - np.abs(f[:, 1] - g[:, 1]))
        w = (w * (one - np.abs(f[:, 2] - g[:, 2]))).astype(np.float32)
        cells.append(ci)
        wts.append(w)
    return np.stack(cells), np.stack(wts)


def q(f):
    return np.rint(np.asarray(f, np.float64) * Q).astype(np.int64)


def fuse_reference(parts, N, Nz, vs):
    """parts: list of dicts with idx [n,3], tsdf, w [n] f32, occ [n] int, optional color [n,3] f32, R [3,3], T [3] and
    optional sign (+1 add, -1 remove).  -> dict(idx int32 [m,3], tsdf, w f32 [m], occ int8 [m], color f32 [m,3] or
    None, splatted, skipped), rows in lexicographic idx order."""
    hN, hNz = N // 2, Nz // 2
    textured = any(p.get("color") is not None for p in parts)
    keys, cols = [], {k: [] for k in ("wt", "w", "co", "c0", "c1", "c2")}
    splatted = skipped = 0
    for p in parts:
        idx = np.asarray(p["idx"], np.int64).reshape(-1, 3)
        if idx.shape[0] == 0:
            continue
        sign = int(p.get("sign", 1))
        W = np.asarray(p["w"], np.float32)
        T = np.asarray(p["tsdf"], np.float32)
        occ = np.asarray(p["occ"], np.int64)
        C = np.asarray(p["color"], np.float32).reshape(-1, 3) if textured else None
        g, lo = place(idx, p["R"], p["T"], vs)
        cells, wts = corners(g, lo)
        inb = ((cells[..., 0] >= -hN) & (cells[..., 0] < N - hN) & (cells[..., 1] >= -hN) & (cells[..., 1] < N - hN) &
               (cells[..., 2] >= -hNz) & (cells[..., 2] < Nz - hNz))
        with np.errstate(all="ignore"):
            w = (W[None, :] * wts).astype(np.float32)
            terms = [w, (w * T[None, :]).astype(np.float32)]
            if textured:
                terms += [(w * C[None, :, a]).astype(np.float32) for a in range(3)]
            bad = np.zeros(w.shape, bool)
            for t in terms:
                bad |= ~(np.abs(t) < FMAX)
        bad_vox = (bad & inb).any(0)
        skipped += int(bad_vox.sum())
        splatted += int((~bad_vox).sum())
        use = inb & ~bad_vox[None, :]
        keys.append(cells[use])
        s = np.int64(sign)
        cols["w"].append(s * q(terms[0][use]))
        cols["wt"].append(s * q(terms[1][use]))
        cols["co"].append(s * ((np.int64(1) << np.int64(32)) + np.broadcast_to(occ[None, :], use.shape)[use]))
        if textured:
            for a in range(3):
                cols[f"c{a}"].append(s * q(terms[2 + a][use]))
    if not keys or sum(k.shape[0] for k in keys) == 0:
        e = np.zeros(0, np.float32)
        return dict(idx=np.zeros((0, 3), np.int32), tsdf=e, w=e, occ=np.zeros(0, np.int8),
                    color=np.zeros((0, 3), np.float32) if textured else None, splatted=splatted, skipped=skipped)
    K = np.concatenate(keys)
    uk, inv = np.unique(K, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    sums = {}
    for k, v in cols.items():
        if not v:
            continue
        acc = np.zeros(uk.shape[0], np.int64)
        with np.errstate(over="ignore"):
            np.add.at(acc, inv, np.concatenate(v))
        sums[k] = acc
    co = sums["co"]
    cnt = (co + (np.int64(1) << np.int64(31))) >> np.int64(32)
    socc = co - (cnt << np.int64(32))
    keep = cnt != 0
    sw = sums["w"][keep].astype(np.float64)
    with np.errstate(all="ignore"):
        t = (sums["wt"][keep].astype(np.float64) / sw).astype(np.float32)
        col = np.stack([(sums[f"c{a}"][keep].astype(np.float64) / sw).astype(np.float32) for a in range(3)], 1) if textured else None
    wout = (sw * 2.0 ** -24).astype(np.float32)
    occ_out = np.clip(socc[keep], -128, 127).astype(np.int8)
    idx_out = uk[keep].astype(np.int32)
    o = np.lexsort((idx_out[:, 2], idx_out[:, 1], idx_out[:, 0]))
    return dict(idx=idx_out[o], tsdf=t[o], w=wout[o], occ=occ_out[o], color=None if col is None else col[o],
                splatted=splatted, skipped=skipped)


def same_values(a, b):
    """Arrays equal bit for bit, except that any NaN equals any NaN (the device and numpy spell 0 / 0 differently)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def same_rows(gpu, ref):
    """gather() rows (idx, tsdf, w, occ[, color]) of the device against fuse_reference's dict, in key order."""
    o = np.lexsort((gpu[0][:, 2], gpu[0][:, 1], gpu[0][:, 0]))
    rows = [np.asarray(a)[o] for a in gpu]
    ok = (same_values(rows[0].astype(np.int32), ref["idx"]) and same_values(rows[1], ref["tsdf"]) and same_values(rows[2], ref["w"])
          and same_values(rows[3].astype(np.int8), ref["occ"]))
    if len(rows) > 4:
        ok = ok and same_values(rows[4], ref["color"])
    return ok
