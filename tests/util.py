"""Shared helpers for the parity tests."""
import numpy as np


def rot_xyz(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def key_sort(idx):
    """Lexicographic row order of an [n,3] int array."""
    return np.lexsort((idx[:, 2], idx[:, 1], idx[:, 0]))


def as_dict_rows(idx, *cols):
    o = key_sort(idx)
    return (idx[o],) + tuple(c[o] for c in cols)


def compare_voxels(gpu, orc, tol=1e-4, check_occ=True):
    """gpu/orc = (idx, tsdf, w, occ).  Index set and occupy bit-exact, values within tol."""
    gi, gt, gw, go = as_dict_rows(*gpu)
    oi, ot, ow, oo = as_dict_rows(*orc)
    assert gi.shape == oi.shape, f"voxel count differs: gpu {gi.shape[0]} oracle {oi.shape[0]}"
    assert np.array_equal(gi, oi), "observed voxel index sets differ"
    if check_occ:
        assert np.array_equal(go.astype(np.int32), oo.astype(np.int32)), "occupy differs"
    fin = np.isfinite(ot)
    assert np.array_equal(np.isfinite(gt), fin)
    dt = np.abs(gt[fin] - ot[fin])
    dw = np.abs(gw - ow)
    assert dt.max(initial=0.0) <= tol, f"max |dTSDF| = {dt.max()}"
    # weights: relative tolerance (W grows to 1000)
    assert np.all(dw <= tol * np.maximum(1.0, np.abs(ow))), f"max |dW| = {dw.max()}"
    return float(dt.max(initial=0.0)), float(dw.max(initial=0.0))


F32_U = 2.0 ** -24  # unit roundoff of f32
ref_wmax = 1000.0   # Wmax (dense_tsdf.py:8)


def march_bounds(ref, sequential=False):
    """Per-voxel bounds (bW, bT) on |W - W_ref| and |TSDF - TSDF_ref| for one launch, ref = march_reference output.

    S = sum w, A = sum w*ds, T = A/S, c = samples of the voxel; u = 2^-24.  A march adds some samples as integers
    x = rint(v * 2^k) for v = w and v = w*ds and the others through f32 reductions unquantised (DESIGN §4 "Fixed point
    per launch"):
      * binned march (tslam_march.cu): every sample is quantised at the launch's scale k, except rays with
        w * 2^k < MB_MIN_WQ and samples on block faces, which may take the global f32 path;
      * textured march (k_raymarch): samples in the 16^3 window around the sensor origin are quantised at the scale of
        their round of 512 rays (>= the launch's k, and w * 2^k_r >= MB_MIN_WQ); all others are f32 reductions.
    The reference reports per voxel the sum of the fixed-point bounds (q), the reductions that may reach it (n_red) and
    the rounding of the kernels' sample values (eval).  Error sources of W:
      * fixed point: <= 2^-(k_r+1) per quantised sample                                 -> q
      * the kernels' weight 1/(z*z) in f32 of the 2^-20-quantised z, not 1/|p|^2        -> sum |w32 - w|   (measured)
      * f32 rounding of each reduction that reaches the voxel (item flushes, global-path samples) and of the
        commit, each of a partial sum <= S                                              -> (n_red + 1) * u * S
    Error sources of A, besides the same fixed-point term:
      * the sample value (binned: L - j*vs; textured: |P - x_| * sign in f32) instead of the exact |P - x_| * sign
                                                                                        -> sum w*|ds_kernel - ds| (measured)
      * f32 rounding in forming each summand (binned: fma(-j0, vs, L), fma(-k, vs, L0), times w, and the global path's
        conversion, four roundings of values <= L + j*vs; textured: w * ds)            -> eval
      * w32 instead of w                                                                 -> sum |w32 - w| * |ds|
      * f32 reductions of partial sums <= sum w*|ds|                                     -> (n_red + 1) * u * sum w*|ds|
    TSDF = A'/S' with |A' - A| <= bA, |S' - S| <= bW: |T' - T| <= (bA + |T| bW) / S to first order, plus the commit
    division and the final f32 rounding: 3u |T|.  The Wmax clamp is 1-Lipschitz: the W bound holds for min(S, 1000).
    sequential=True: an f32 running average (the literal oracle, dense_tsdf.py:264-267) instead of sums - every
    sample is its own reduction (n_red = c), its weight is 1/(z*z) of the unquantised f32 z (3u more), and each
    update T' = (T W + w ds)/(W + w) adds <= 4u max|ds|.
    """
    c = ref["count"].astype(np.float64)
    n_red = c if sequential else ref["n_red"]
    q = ref["q"]
    S, T = ref["sw"], np.abs(ref["tsdf"])
    # (sequential: the weight is 1/(z*z) of the unquantised f32 z, within 3u of w)
    ew = (n_red + 1.0 + (3.0 if sequential else 0.0)) * F32_U
    bW = q + ref["dw"] + ew * S
    bA = q + ref["dds"] + ref["eval"] + ref["dwd"] + ew * ref["swabsd"]
    bT = (bA + T * bW) / S + 3.0 * F32_U * T
    if sequential:  # once the clamp binds mid-frame the running average is no longer the weighted mean: unbounded
        bT = np.where(S < ref_wmax, bT + c * 4.0 * F32_U * ref["max_absd"], np.inf)
    return bW, bT


def one_sample_effect(ref):
    """What one sample more or less changes at each voxel: mean weight S/c in W, and the spread of ds over c in TSDF
    (sqrt(sum w ds^2 / S - T^2) / c)."""
    c = ref["count"].astype(np.float64)
    S = ref["sw"]
    sd = np.sqrt(np.maximum(ref["swd2"] / S - ref["tsdf"] ** 2, 0.0))
    return S / c, sd / c


def compare_to_reference(got, ref, sequential=False, sharp=True):
    """got = (idx, tsdf, w[, occ]) of one launch vs march_reference output: same voxel set, W and TSDF within
    march_bounds.  sharp: the bounds at the hottest voxel must also be well below the effect of one sample there, so
    that a bound grown too loose fails instead of passing."""
    gi, gt, gw = as_dict_rows(*got[:3])
    assert gi.shape == ref["idx"].shape, f"voxel count differs: got {gi.shape[0]} reference {ref['idx'].shape[0]}"
    assert np.array_equal(gi, ref["idx"]), "observed voxel index sets differ"
    bW, bT = march_bounds(ref, sequential)
    dW = np.abs(gw.astype(np.float64) - ref["W"])
    dT = np.abs(gt.astype(np.float64) - ref["tsdf"])
    assert np.all(dW <= bW), f"W off the reference at {int((dW > bW).sum())} voxels, worst {np.max(dW / bW):.3g}x the bound"
    assert np.all(dT <= bT), f"TSDF off the reference at {int((dT > bT).sum())} voxels, worst {np.max(dT / bT):.3g}x the bound"
    if sharp:
        h = int(np.argmax(ref["count"]))
        eW, eT = one_sample_effect(ref)
        assert bW[h] < 0.1 * eW[h], f"W bound {bW[h]:.3g} not well below one sample ({eW[h]:.3g}) at the hottest voxel"
        # (eT = 0: every sample of the voxel carries the same ds, and no sample count changes its TSDF)
        assert eT[h] == 0.0 or bT[h] < 0.5 * eT[h], f"TSDF bound {bT[h]:.3g} not well below one sample ({eT[h]:.3g}) at the hottest voxel"
    with np.errstate(invalid="ignore", divide="ignore"):  # (bound 0 where the sums are exact, and so is the result)
        return float(np.max(np.where(bW > 0, dW / bW, 0.0))), float(np.max(np.where(bT > 0, dT / bT, 0.0)))


def tri_multiset(verts, decimals=5):
    """Canonical sorted array of triangles (each triangle's 3 vertices kept in emission order)."""
    t = np.round(verts.reshape(-1, 9).astype(np.float64), decimals)
    o = np.lexsort(t.T[::-1])
    return t[o]
