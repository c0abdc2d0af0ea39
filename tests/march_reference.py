"""f64 reference of process_new_pcl (dense_tsdf.py:236-270) for point clouds whose every point is alone in its bucket.

Input contract: the points lie on the 2^-20 m grid the bucket kernels sum in, no two share a bucket (round(p/vs)), and
they are integrated with R = I.  Then a bucket's mean is its point, exactly, in every implementation, and the ray of a
bucket needs no bucket emulation.

Per ray, the quantities that decide WHICH voxel a sample lands in are reproduced in float32, in the source's order, so
that the voxel indices come out bit for bit as the CUDA kernels and the oracle compute them (:244-254):
    L = |p|,  u = p / L,  n = int(min(L/vs + internal_voxels, max_ray_length/vs)),  x_ = (u*j)*vs + T,
    index = round_half_away(x_/vs)      (the f32 quotient, rounded in f64)
Everything that is ACCUMULATED is f64: w = 1/z^2 with z = |p|, the exact signed distance ds = |P - x_| * sign((P - x_).p)
of the f32 sample point x_, and per voxel the sample count, sum w and sum w*ds.  The Wmax clamp is applied once, at
commit: the reference reports the unclamped sums and W = min(sum w, Wmax).

Beside the sums it reports what tests/util.py::march_bounds needs to bound the distance of an implementation from it:
the fixed-point scale k of the launch (as k_seg_scan derives it), the weight as the kernels round it, the distance
between the kernels' sample value and the exact ds, and an upper bound on the number of f32 reductions that reach each
voxel.  Two marches are described (`path`):
  * "binned" (tslam_march.cu, untextured maps): sample value L - j*vs, fixed-point sums per work item of a block;
  * "textured" (k_raymarch, tslam_integrate.cu): sample value |P - x_| * sign in f32, formed here as the kernel forms
    it; fixed-point sums only in a 16^3 window around the sensor origin (steps 1-18 of rays of the window's submap),
    at a scale chosen per round of 512 rays; every other sample is an f32 reduction.
With `rgb` (uint8 [n,3], one colour per point) it also reports the colour word every voxel ends with (the largest
[seq:22 | 4095 - min(4095, |ds|/vs*16):12 | rgb 3x10] over its samples, ds in f32 as the kernels and the oracle form it),
and the voxels where the exact ds would have put a sample's closeness in another bin and changed the winner.
"""
import numpy as np

WMAX = 1000.0
FIXQ = 2.0 ** 20      # bucket fixed point (per-frame sums of the bucket kernels)
MR_CHUNK = 4096       # segments per work item of the binned march
MB_MIN_WQ = 16384     # rays below this many fixed-point units take f32 global reductions
TS_B = 16             # voxel block edge of the CUDA map
F32_U = 2.0 ** -24    # unit roundoff of f32
RM_THREADS = 512      # rays per round of k_raymarch (one window per round)
RM_WIN = 16           # window edge (voxels) of k_raymarch, origin round(T/vs) - 8
RM_WIN_STEPS = 18     # steps of a ray that can fall into the window

_f = np.float32
_SUMS = ("count", "sw", "swd", "swabsd", "swd2", "dw", "dwd", "dds", "eval", "q", "glob", "nwin")


def round_half_away(q):
    """ti.round / roundf of an f32 quotient, done in f64."""
    q = q.astype(np.float64)
    return (np.sign(q) * np.floor(np.abs(q) + 0.5)).astype(np.int64)


def ray_setup(pts, vs, internal_voxels, max_ray_length):
    """f32 ray set-up of :240-251 and the launch's fixed-point scale (k_seg_scan).  pts: f32 [n,3], R = I."""
    p = np.ascontiguousarray(pts, dtype=np.float32)
    vs32 = _f(vs)
    L = np.sqrt((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2])          # :244, also z = pt.norm() (:176)
    keep = L < _f(max_ray_length)                                                      # :177
    p, L = p[keep], L[keep]
    u = p / L[:, None]                                                                 # :245
    max_steps = _f(max_ray_length / vs)                                                # python-float constant (:249)
    n = np.minimum(L / vs32 + _f(internal_voxels), max_steps).astype(np.int64)         # :249-251, range(float) truncates
    # the weight as the kernels form it: the mean z of a one-point bucket passes the 2^-20 fixed point, then 1/(z*z) in f32
    zq = (np.rint(L.astype(np.float64) * FIXQ) / FIXQ).astype(np.float32)
    wf = _f(1.0) / (zq * zq)
    z64 = np.sqrt((p.astype(np.float64) ** 2).sum(1))
    # fixed-point scale: the largest k with max(w, w*dmax) * 2^k < 2^30, clamped to [0, 48] (tslam_march.cu ray_setup, k_seg_scan)
    dmax = np.maximum(L, n.astype(np.float32) * vs32 - L) + vs32
    fm = np.minimum(np.maximum(wf, wf * dmax), _f(3.0e38)).astype(np.float64)
    fmax = float(fm.max(initial=0.0))
    k = 30 - int(np.frexp(fmax)[1]) if fmax > 0 else 30
    k = max(0, min(48, k))
    tiny = np.rint(wf.astype(np.float64) * 2.0 ** k) < MB_MIN_WQ
    # the largest scale a round of k_raymarch holding the ray can have: the ray's own
    k_ray = np.clip(30 - np.frexp(fm)[1], 0, 48)
    return dict(p=p, L=L, u=u, n=n, w=1.0 / (z64 * z64), w32=wf.astype(np.float64), k=k, tiny=tiny, keep=keep,
                tiny_ray=np.rint(wf.astype(np.float64) * np.exp2(k_ray)) < MB_MIN_WQ)


def _samples(rays, sel, vs, T):
    """All samples of the rays `sel`, ray by ray in step order: ray, step j, voxel index, exact ds, the f32 sample values
    of the binned march (L - j*vs) and of k_raymarch, and L + j*vs."""
    vs32 = _f(vs)
    T32 = np.asarray(T, np.float32)
    n = rays["n"][sel]
    ray = np.repeat(sel, n)
    j = np.arange(ray.shape[0], dtype=np.int64) - np.repeat(np.cumsum(n) - n, n) + 1
    u = rays["u"][ray]
    x = (u * j.astype(np.float32)[:, None]) * vs32 + T32                                 # :253 (f32, source order)
    idx = round_half_away(x / vs32)                                                      # :254
    p = rays["p"][ray].astype(np.float64)
    v = (p + T32.astype(np.float64)) - x.astype(np.float64)                             # :258 P - x_ (exact in f64)
    ds = np.sqrt((v * v).sum(1)) * np.sign((v * p).sum(1))                              # :259-260
    jv = j * np.float64(vs32)
    L = rays["L"][ray].astype(np.float64)
    # k_raymarch's value, in f32 and source order (P = f32(mean + T)): d = sqrtf((vx*vx + vy*vy) + vz*vz), times sgnf
    m = rays["p"][ray]
    vf = (m + T32) - x
    df = np.sqrt((vf[:, 0] * vf[:, 0] + vf[:, 1] * vf[:, 1]) + vf[:, 2] * vf[:, 2])
    sf = (vf[:, 0] * m[:, 0] + vf[:, 1] * m[:, 1]) + vf[:, 2] * m[:, 2]
    ds_t = df * np.sign(sf).astype(np.float32)
    return ray, j, idx, ds, L - jv, ds_t, L + jv


def color_words(rgb, ray, ds, vs, seq):
    """The colour word of each sample (k_raymarch, oracle color_word): the point's colour / 255 quantised to 10 bits in
    f32, closeness from |ds| / vs * 16 (ds f32: f32 division, truncation; ds f64: the exact bin)."""
    c = rgb.astype(np.float32)
    q = np.minimum(1023, ((c / _f(1.0)) / _f(255.0) * _f(1023.0) + _f(0.5)).astype(np.int64)).astype(np.uint64)
    q = (q[:, 0] << np.uint64(20)) | (q[:, 1] << np.uint64(10)) | q[:, 2]
    if ds.dtype == np.float32:
        cl = np.minimum(4095, (np.abs(ds) / _f(vs) * _f(16.0)).astype(np.int64))
    else:
        cl = np.minimum(4095, np.floor(np.abs(ds) / np.float64(_f(vs)) * 16.0).astype(np.int64))
    return (np.uint64(seq) << np.uint64(42)) | ((4095 - cl).astype(np.uint64) << np.uint64(30)) | q[ray]


def reference_march(pts, T, vs, N, Nz, internal_voxels=10, max_ray_length=10.0, chunk=1 << 22, path="binned", rgb=None,
                    seq=1):
    """What one integrate_points(pts, I, T) call adds to each voxel of an N x N x Nz map, marched by `path` ("binned" or
    "textured"), with the colour words of frame `seq` when `rgb` is given.  Per-voxel arrays are in lexicographic
    voxel-index order."""
    assert path in ("binned", "textured")
    rays = ray_setup(pts, vs, internal_voxels, max_ray_length)
    if rgb is not None:
        rgb = np.asarray(rgb, np.uint8)[rays["keep"]]
    lo = np.array([-(N // 2), -(N // 2), -(Nz // 2)], np.int64)
    dims = np.array([N, N, Nz], np.int64)
    nb = dims // TS_B + 3
    win_lo = round_half_away(np.asarray(T, np.float32) / _f(vs)) - RM_WIN // 2  # k_raymarch: iroundf(T / vs) - 8
    keys, sums, vblocks, run_blocks, words = [], [], [], [], []
    n_in = n_oob = n_tiny = 0
    cum = np.cumsum(rays["n"])
    nr, start = cum.shape[0], 0
    while start < nr:
        base = cum[start - 1] if start else 0
        stop = min(nr, max(start + 1, int(np.searchsorted(cum, base + chunk, side="right"))))
        ray, j, idx, ds, ds_k, ds_t, span = _samples(rays, np.arange(start, stop), vs, T)
        start = stop
        inb = np.all((idx >= lo) & (idx < lo + dims), axis=1)
        n_in += int(inb.sum())
        n_oob += int((~inb).sum())
        blk = np.floor_divide(idx - lo, TS_B) + 1
        bkey = (blk[:, 0] * nb[1] + blk[:, 1]) * nb[2] + blk[:, 2]
        # a run of consecutive in-bounds samples of one ray in one block: what the segment walk makes segments of
        run = inb & ((j == 1) | np.r_[True, (bkey[1:] != bkey[:-1]) | ~inb[:-1]])
        ray, j, idx, ds, ds_k, ds_t, span, bkey, run = (a[inb] for a in (ray, j, idx, ds, ds_k, ds_t, span, bkey, run))
        run_blocks.append(bkey[run])
        w, w32, tiny = rays["w"][ray], rays["w32"][ray], rays["tiny"][ray]
        key = ((idx[:, 0] - lo[0]) * dims[1] + (idx[:, 1] - lo[1])) * dims[2] + (idx[:, 2] - lo[2])
        uk, first, inv = np.unique(key, return_index=True, return_inverse=True)
        common = dict(count=np.ones_like(w), sw=w, swd=w * ds, swabsd=w * np.abs(ds), swd2=w * ds * ds,
                      dw=np.abs(w32 - w), dwd=np.abs(w32 - w) * np.abs(ds))
        if path == "binned":
            n_tiny += int(tiny.sum())
            loc = np.mod(idx, TS_B)
            face = np.any((loc == 0) | (loc == TS_B - 1), axis=1)
            # the chain fma(-j0, vs, L), fma(-k, vs, L0), times w, and the global path's conversion: four roundings
            terms = dict(dds=w * np.abs(ds_k - ds), eval=4.0 * F32_U * w * span,
                         q=(~tiny) * 2.0 ** -(rays["k"] + 1), glob=(face | tiny).astype(np.float64), nwin=np.zeros_like(w))
            dsv = ds_k
        else:
            # window samples: steps 1-18 inside the window (one frame, one submap here).  A round's scale k_r lies between
            # the launch's k (every ray in the round) and the ray's own; a ray is quantised iff w * 2^k_r >= MB_MIN_WQ.
            # Window samples of rays that may go either way are counted in both error models.
            cand = (j <= RM_WIN_STEPS) & np.all((idx - win_lo >= 0) & (idx - win_lo < RM_WIN), axis=1)
            maybe_q = cand & ~rays["tiny_ray"][ray]
            maybe_f = ~cand | tiny
            n_tiny += int((cand & tiny).sum())
            # quantised at k_r >= k with w * 2^k_r >= MB_MIN_WQ - 1/2: error <= min(2^-(k+1), w / (2 MB_MIN_WQ - 1))
            qs = np.minimum(2.0 ** -(rays["k"] + 1), w32 / (2 * MB_MIN_WQ - 1))
            terms = dict(dds=w * np.abs(ds_t.astype(np.float64) - ds), eval=F32_U * w32 * np.abs(ds_t),  # a = w * ds in f32
                         q=maybe_q * qs, glob=maybe_f.astype(np.float64), nwin=maybe_q.astype(np.float64))
            dsv = ds_t
        terms.update(common)
        sums.append({nm: np.bincount(inv, weights=t, minlength=uk.shape[0]) for nm, t in terms.items()})
        for nm, t in (("max_dds", np.abs(dsv.astype(np.float64) - ds)), ("max_absd", np.abs(ds))):
            mx = np.zeros(uk.shape[0])
            np.maximum.at(mx, inv, t)
            sums[-1][nm] = mx
        if rgb is not None:
            cw = np.zeros((2, uk.shape[0]), np.uint64)
            np.maximum.at(cw[0], inv, color_words(rgb, ray, ds_t, vs, seq))
            np.maximum.at(cw[1], inv, color_words(rgb, ray, ds, vs, seq))
            words.append(cw)
        keys.append(uk)
        vblocks.append(bkey[first])
    keys = np.concatenate(keys) if keys else np.zeros(0, np.int64)
    uk, first, inv = np.unique(keys, return_index=True, return_inverse=True)
    out = {nm: np.bincount(inv, weights=np.concatenate([s[nm] for s in sums]), minlength=uk.shape[0]) if sums else np.zeros(0)
           for nm in _SUMS}
    for nm in ("max_dds", "max_absd"):
        out[nm] = np.zeros(uk.shape[0])
        if sums:
            np.maximum.at(out[nm], inv, np.concatenate([s[nm] for s in sums]))
    if rgb is not None:
        cw = np.zeros((2, uk.shape[0]), np.uint64)
        for r in range(2):
            np.maximum.at(cw[r], inv, np.concatenate([c[r] for c in words]) if words else np.zeros(0, np.uint64))
        out["cword"] = cw[0]
        out["color"] = np.stack([(cw[0] >> np.uint64(s)) & np.uint64(1023) for s in (20, 10, 0)], 1).astype(np.float32) / _f(1023.0)
        out["color_amb"] = cw[0] != cw[1]
    if path == "binned":
        vblk = np.concatenate(vblocks)[first] if vblocks else np.zeros(0, np.int64)
        ub, segs = np.unique(np.concatenate(run_blocks) if run_blocks else np.zeros(0, np.int64), return_counts=True)
        seg_v = segs[np.searchsorted(ub, vblk)] if ub.size else np.zeros(0)
        # f32 reductions that reach a voxel: one flush per work item (<= MR_CHUNK segments) of its block, plus one per
        # sample that may take the global path (block faces, tiny weights).  A run of <= 28 samples is one segment; the
        # walk's block-crossing hints may be a step off, so a block may also hold a stray one-step segment per
        # neighbouring run: segments <= 2 x runs.
        out["n_red"] = np.minimum(out["count"], np.ceil(2.0 * seg_v / MR_CHUNK) + 1.0 + out["glob"])
    else:
        # one f32 reduction per far sample, one flush per round of 512 rays that put a window sample there, and the
        # conversions of the flushed window sums to f32 (together <= u * sum w)
        rounds = np.ceil(nr / RM_THREADS)
        out["n_red"] = out["glob"] + np.minimum(out["nwin"], rounds) + (out["nwin"] > 0)
    out["count"] = out["count"].astype(np.int64)
    iz, iy, ix = uk % dims[2], (uk // dims[2]) % dims[1], uk // (dims[2] * dims[1])
    out["idx"] = np.stack([ix + lo[0], iy + lo[1], iz + lo[2]], 1).astype(np.int32)
    with np.errstate(invalid="ignore", divide="ignore"):
        out["tsdf"] = out["swd"] / out["sw"]
    out["W"] = np.minimum(out["sw"], WMAX)
    out.update(n_updates=n_in, n_oob=n_oob, n_rays=int(nr), k=rays["k"], n_tiny=n_tiny, w32=rays["w32"], path=path)
    return out
