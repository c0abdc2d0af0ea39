// libtslam.so - the TSDF integrate path: depth frames / point clouds -> per-frame buckets -> ray march -> commit.
// The kernels and the one host sequence that launches them (ts_integrate_launch).  sm_90a.
//
// Reference semantics: taichi_slam/mapping/dense_tsdf.py (cited per kernel).
// Compiled with -fmad=false: the index-forming arithmetic must round exactly like
// the strict-IEEE statement of the reference source (voxel indices are compared
// bit-for-bit by the parity tests).
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <cmath>
#include "tslam_internal.cuh"
#include "tslam_bucket.cuh"

// bucket index entry: [launch epoch : 25 - S][record slot + 1 : S][bx + 4096 : 13][by + 4096 : 13][bz + 4096 : 13],
// S = TsBucketLaunch::slot_bits.  An entry whose epoch is not the launch's counts as empty, so nobody clears the index
// between launches: the host clears it once when the epoch wraps (ts_bucket_launch).  A handle whose record slots
// leave fewer than TS_BK_MIN_EPOCH_BITS for the epoch runs in clearing mode instead: S = 25, no epoch, and the ray
// set-up zeroes the entry of every record it reads (TsBucketLaunch::bpos).
#define BK_OFF 4096
#define BK_KEY_BITS 39
#define BK_KEY_MASK ((1ull << BK_KEY_BITS) - 1ull)
__device__ __forceinline__ unsigned long long bucket_key(int bx, int by, int bz) {
  return ((unsigned long long)(bx + BK_OFF) << 26) | ((unsigned long long)(by + BK_OFF) << 13) | (unsigned long long)(bz + BK_OFF);
}
__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.b64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// release: the opener's record stores are visible to whoever reads the entry; acquire: a lane that loses the race
// reads the winner's entry and then adds into the winner's record
__device__ __forceinline__ unsigned long long cas_acq_rel_u64(unsigned long long* p, unsigned long long cmp, unsigned long long val) {
  unsigned long long old;
  asm volatile("atom.acq_rel.gpu.global.cas.b64 %0, [%1], %2, %3;" : "=l"(old) : "l"(p), "l"(cmp), "l"(val) : "memory");
  return old;
}

#define BK_CTA_TAB 512  // CTA bucket table: open addressing, twice the 256 keys a CTA can bring
#define BK_ROW 13       // words of a CTA bucket's sums: lo x, y, z, d; hi x, y, z, d; count; r, g, b (13: odd row stride)

// S from lo = S mod 2^32 and hi = sum(x >> 16) over fewer than 2^16 int32 addends x (as mb_sum, tslam_march.cu)
__device__ __forceinline__ long long bk_row_sum(unsigned int lo, unsigned int hi) {
  return (long long)(int)hi * 65536ll + (long long)(unsigned int)(lo - (hi << 16));
}

// accumulate one unprojected point per thread into the frame's bucket grid.
// process_point (dense_tsdf.py:227-234) with exact fixed-point sums.  Points that fall into the same bucket
// (neighbouring pixels usually do) are merged on chip in two stages before anyone touches the index: lanes of a warp
// (match.any, per-warp slots), then the warps of the CTA (a shared-memory table keyed by the bucket, exact two-word
// sums).  One probe and one set of reductions per distinct bucket per CTA instead of per pixel.  The index maps the
// bucket's voxel to a RECORD slot.  Slots need no allocator: every CTA owns the 256 records [slot_base, slot_base + 256)
// (it holds at most 256 distinct buckets), the thread that owns a bucket's CTA sums brings the slot of its thread index
// along and publishes it with the key in ONE 64-bit CAS, so nobody ever waits for a slot.  The slot is private until
// that CAS publishes it, so the thread STORES its CTA's sums there first (the record needs no zeroing); threads that
// find the bucket open add into its record.  A thread that loses the race leaves its slot written but unnamed.
// Must be called by all 256 threads of the CTA; `valid` masks threads without a point.  Returns the record slot when
// this thread OPENED a bucket (the bucket becomes one ray; the caller appends it to the ray list), else -1.
__device__ __forceinline__ int bucket_accumulate(bool valid, unsigned long long* idx, uint32_t cap_mask, uint32_t idx_base, TsBucket* recs,
                                                 uint4* cols, uint32_t* cnts, uint32_t rec_cap, uint32_t slot_base, const TsBucketLaunch& bl, float px,
                                                 float py, float pz, float dep, float vs, float rvs, bool agg_ok, int* err, bool tex = false,
                                                 int cr = 0, int cg = 0, int cb = 0) {
  // xyz_to_ijk mapping_common.py:240-243; div_vs is the correctly rounded px / vs
  const int bx = iroundf(div_vs(px, vs, rvs)), by = iroundf(div_vs(py, vs, rvs)), bz = iroundf(div_vs(pz, vs, rvs));
  if (valid && ((unsigned)(bx + (BK_OFF - 1)) > 2u * (BK_OFF - 1) || (unsigned)(by + (BK_OFF - 1)) > 2u * (BK_OFF - 1) ||
                (unsigned)(bz + (BK_OFF - 1)) > 2u * (BK_OFF - 1))) {
    atomicOr(err, TS_ERR_BUCKET_RANGE);
    valid = false;
  }
  const unsigned long long key = bucket_key(bx, by, bz);
  long long qx = __float2ll_rn(px * FIXQ), qy = __float2ll_rn(py * FIXQ), qz = __float2ll_rn(pz * FIXQ), qd = __float2ll_rn(dep * FIXQ);
  int cnt = 1;
  bool act = valid;  // this thread probes and adds
  const unsigned vmask = __ballot_sync(0xffffffffu, valid);
  const uint32_t hk = ts_hash(key);
  if (agg_ok) {  // |q| < 2^26 (max_ray < 64 m): a 32-lane sum fits int32
    // every lane adds its point to the shared-memory slot of its group's first lane (native 32-bit ATOMS; slots of
    // different groups sit in different banks: stride 9 words), the leaders read the totals back.  (The
    // redux-per-group loop this replaces was 17 % of the kernel's instructions.)
    __shared__ int s_agg[8][32][9];
    // CTA stage: the table maps a key to the thread that owns the bucket's row, entry = key << 8 | owner (~0: empty)
    __shared__ unsigned long long s_tab[BK_CTA_TAB];
    __shared__ unsigned int s_row[256][BK_ROW];
    const int lane = threadIdx.x & 31, wid = (threadIdx.x >> 5) & 7;
    int* mine = s_agg[wid][lane];
    mine[0] = 0; mine[1] = 0; mine[2] = 0; mine[3] = 0; mine[4] = 0;
    if (tex) { mine[5] = 0; mine[6] = 0; mine[7] = 0; }
    unsigned int* row = s_row[threadIdx.x];
    for (int e = 0; e < 9; e++) row[e] = 0u;
    if (tex) { row[9] = 0u; row[10] = 0u; row[11] = 0u; }
    s_tab[threadIdx.x] = ~0ull;
    s_tab[threadIdx.x + 256] = ~0ull;
    __syncwarp();
    if (valid) {
      const unsigned grp = __match_any_sync(vmask, key);
      const int lead = __ffs(grp) - 1;
      act = lane == lead;
      // the index entry this bucket will probe: an index line is rarely in L2 (64 frames x 1 MB), so its DRAM fetch
      // starts here and overlaps the merge and its two barriers instead of following them
      if (act) asm volatile("prefetch.global.L2 [%0];" ::"l"(idx + (hk & cap_mask)));
      cnt = __popc(grp);
      int* slot = s_agg[wid][lead];
      if (grp & (grp - 1u)) {  // more than one lane in the bucket
        atomicAdd(&slot[0], (int)qx); atomicAdd(&slot[1], (int)qy); atomicAdd(&slot[2], (int)qz); atomicAdd(&slot[3], (int)qd);
        if (tex) { atomicAdd(&slot[5], cr); atomicAdd(&slot[6], cg); atomicAdd(&slot[7], cb); }
      }
    }
    __syncwarp();
    if (valid && act && cnt > 1) {
      qx = (long long)mine[0]; qy = (long long)mine[1]; qz = (long long)mine[2]; qd = (long long)mine[3];
      if (tex) { cr = mine[5]; cg = mine[6]; cb = mine[7]; }
    }
    __syncthreads();  // the CTA table and rows are cleared
    if (valid && act) {  // warp leaders: at most one per warp and bucket, so a row sums at most 8 addends
      const unsigned long long want = (key << 8) | (unsigned long long)threadIdx.x;
      uint32_t hs = hk & (BK_CTA_TAB - 1);
      int own;
      for (;;) {  // 256 keys at most in 512 entries: an empty entry is always found
        const unsigned long long prev = atomicCAS(&s_tab[hs], ~0ull, want);
        if (prev == ~0ull) { own = (int)threadIdx.x; break; }
        if ((prev >> 8) == key) { own = (int)(prev & 255ull); break; }
        hs = (hs + 1) & (BK_CTA_TAB - 1);
      }
      unsigned int* o = s_row[own];
      const int wx = (int)qx, wy = (int)qy, wz = (int)qz, wd = (int)qd;
      atomicAdd(&o[0], (unsigned)wx); atomicAdd(&o[1], (unsigned)wy); atomicAdd(&o[2], (unsigned)wz); atomicAdd(&o[3], (unsigned)wd);
      atomicAdd(&o[4], (unsigned)(wx >> 16)); atomicAdd(&o[5], (unsigned)(wy >> 16)); atomicAdd(&o[6], (unsigned)(wz >> 16));
      atomicAdd(&o[7], (unsigned)(wd >> 16));
      atomicAdd(&o[8], (unsigned)cnt);
      if (tex) { atomicAdd(&o[9], (unsigned)cr); atomicAdd(&o[10], (unsigned)cg); atomicAdd(&o[11], (unsigned)cb); }
      act = own == (int)threadIdx.x;
    }
    __syncthreads();  // the CTA's sums are complete
    if (act) {
      qx = bk_row_sum(row[0], row[4]); qy = bk_row_sum(row[1], row[5]); qz = bk_row_sum(row[2], row[6]); qd = bk_row_sum(row[3], row[7]);
      cnt = (int)row[8];
      if (tex) { cr = (int)row[9]; cg = (int)row[10]; cb = (int)row[11]; }
    }
  }
  uint32_t h = hk & cap_mask;
  if (!act) return -1;
  const uint32_t my_slot = slot_base + threadIdx.x;
  if (my_slot >= rec_cap) { atomicOr(err, TS_ERR_RAYLIST_FULL); return -1; }
  // qd >= 0; with a count plane the word holds the depth sum alone
  const unsigned long long cd = (cnts ? 0ull : (unsigned long long)cnt << bl.cnt_shift) + (unsigned long long)qd;
  const unsigned long long emask = bl.slot_bits >= TS_BK_SLOT_FIELD ? 0ull : ~0ull << (BK_KEY_BITS + bl.slot_bits);
  const unsigned long long smask = (1ull << bl.slot_bits) - 1ull;
  const unsigned long long mine = bl.etag | ((unsigned long long)(my_slot + 1) << BK_KEY_BITS) | key;
  unsigned long long cur = ld_acquire_u64(&idx[h]);
  bool stored = false;
  int slot = -1, fresh = -1;
  for (uint32_t probe = 0; probe <= cap_mask; ++probe) {
    if (cur == 0ull || (cur & emask) != bl.etag) {  // empty, or left by an earlier launch
      if (!stored) {
        uint4* q = reinterpret_cast<uint4*>(&recs[my_slot]);
        q[0] = make_uint4((unsigned)qx, (unsigned)((unsigned long long)qx >> 32), (unsigned)qy, (unsigned)((unsigned long long)qy >> 32));
        q[1] = make_uint4((unsigned)qz, (unsigned)((unsigned long long)qz >> 32), (unsigned)cd, (unsigned)(cd >> 32));
        if (cols) cols[my_slot] = make_uint4((unsigned)cr, (unsigned)cg, (unsigned)cb, 0u);  // textured map: zero without colours
        if (cnts) cnts[my_slot] = (unsigned)cnt;
        stored = true;
      }
      const unsigned long long prev = cas_acq_rel_u64(&idx[h], cur, mine);
      if (prev == cur) {  // this point opened the bucket: it becomes one ray
        fresh = (int)my_slot;
        if (bl.bpos) bl.bpos[idx_base + my_slot] = idx_base + h;  // where the consumer clears the index
        return fresh;
      }
      cur = prev;  // the winner's entry, of this launch
    }
    if ((cur & BK_KEY_MASK) == key) { slot = (int)((cur >> BK_KEY_BITS) & smask) - 1; break; }
    h = (h + 1) & cap_mask;
    cur = ld_acquire_u64(&idx[h]);
  }
  if (slot < 0) { atomicOr(err, TS_ERR_TABLE_FULL); return -1; }
  TsBucket* b = &recs[slot];
  red_add_u64((unsigned long long*)&b->sx, (unsigned long long)qx);
  red_add_u64((unsigned long long*)&b->sy, (unsigned long long)qy);
  red_add_u64((unsigned long long*)&b->sz, (unsigned long long)qz);
  red_add_u64(&b->cd, cd);
  if (cnts) red_add_u32(&cnts[slot], (unsigned int)cnt);
  if (tex) {  // new_pcl_sum_color += rgb (dense_tsdf.py:233-234), exact integer sums
    red_add_u32(&cols[slot].x, (unsigned int)cr);
    red_add_u32(&cols[slot].y, (unsigned int)cg);
    red_add_u32(&cols[slot].z, (unsigned int)cb);
  }
  return fresh;
}

// CTA-aggregated append of the buckets opened by this CTA (one atomic on the global ray counter per CTA instead
// of one per ray; the rays of a pixel tile stay contiguous in the list).  Must be reached by all threads.
__device__ __forceinline__ void append_rays_cta(int fresh_slot, uint32_t tab_base, unsigned n_valid_warp, uint32_t* ray_list,
                                                int* n_rays, uint32_t ray_cap, TsCounters* ctr, int* err) {
  __shared__ unsigned int s_cnt[8], s_val[8];
  __shared__ unsigned int s_base;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned m = __ballot_sync(0xffffffffu, fresh_slot >= 0);
  if (lane == 0) { s_cnt[wid] = __popc(m); s_val[wid] = n_valid_warp; }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned tot = 0, nv = 0;
    for (int w = 0; w < 8; w++) { const unsigned c = s_cnt[w]; s_cnt[w] = tot; tot += c; nv += s_val[w]; }
    s_base = tot ? (unsigned)atomicAdd(n_rays, (int)tot) : 0u;
    if (nv) atomicAdd(&ctr->n_valid, (unsigned long long)nv);
  }
  __syncthreads();
  if (fresh_slot >= 0) {
    const uint32_t p = s_base + s_cnt[wid] + __popc(m & ((1u << lane) - 1));
    if (p < ray_cap) ray_list[p] = tab_base + (uint32_t)fresh_slot; else atomicOr(err, TS_ERR_RAYLIST_FULL);
  }
}

// ---------------------------------------------------------------------------
// K1a: depth frames -> per-frame buckets.
// recast_depth_to_map_kernel phase 1 (dense_tsdf.py:188-213) + unproject_point_dep
// (mapping_common.py:31-41).  One thread per SAMPLED pixel (the reference walks a
// row per thread, :192-194); a warp covers an 8x4 tile of sampled pixels, a CTA 32x8;
// blockIdx.z = frame of the batch.  Six CTAs per SM (40 registers): each CTA is one chain of dependent round trips
// (depth load, index probe, CAS, ray append), so resident CTAs, not bandwidth, set the kernel's rate.
//
// Both bucket kernels are launched with programmatic dependent launch (ts_launch_pdl) after the previous launch's
// commit (or march), so their grid is dispatched while that kernel finishes.  They wait for it at entry, before the
// first load.  What the kernel reads or writes that an earlier kernel on the stream may still own:
//   * the frames / points: the caller's device memory may come from the caller's own kernel right before this launch
//     (PDL relaxes exactly that dependency), so even the depth load waits.  Host batches and queued frames are copied
//     into the staging buffers by a copy the stream waits for in full (memcpy, event wait: an ordinary launch);
//   * n_rays: set back to 0 by the previous launch's march tail (k_march_blocks, last CTA) or by k_reset_counters.
//     k_march_blocks triggers no early launch, so every wait of the chain after it covers its whole grid;
//   * the bucket index: cleared by a memset when the epoch wraps (every 15 launches; an ordinary launch again) and
//     probed / written by the previous launch's bucket kernel and set-up, two kernels back;
//   * staging buffer 0 (host batches) and ev_free[0]: the host waits on ev_free before it refills a buffer, and
//     k_gather_rows runs on the copy stream behind ev_copied: neither is a kernel this one follows;
//   * rm_reserve only sizes the march grid on the host.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 6) k_bucket_depth(const uint16_t* __restrict__ depth, int frame_stride, int row_mul, int w, int hh, int ww,
                                                       const __grid_constant__ TsBatch batch, TsIntrin in, int agg_ok,
                                                       TsBucket* buckets, uint4* bcol, unsigned long long* bidx, uint32_t bucket_cap,
                                                       TsBucketLaunch bl, uint32_t* ray_list, int* n_rays, uint32_t ray_cap, TsCounters* ctr, int* err,
                                                       const uint8_t* __restrict__ tex, int th, int tw, unsigned long long* prof) {
  ts_stamp_begin(prof, TS_K_BUCKET);
  cudaGridDependencySynchronize();
  const int tz = blockIdx.z;    // frame of the batch = its bucket grid
  const int f = tz;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int ii = blockIdx.x * 32 + (wid & 3) * 8 + (lane & 7);
  const int jj = blockIdx.y * 8 + (wid >> 2) * 4 + (lane >> 3);
  bool valid = false;
  float px = 0.f, py = 0.f, pz = 0.f, dep = 0.f;
  int cr = 0, cg = 0, cb = 0;
  if (ii < ww && jj < hh) {
    const int j = jj * in.step, i = ii * in.step;
    // row_mul = recast_step for full frames, 1 when the staging copy already dropped the unsampled rows
    const uint16_t d = depth[(size_t)f * frame_stride + (size_t)(jj * row_mul) * w + i];
    if (ts_depth_kept(in, d)) {  // :196-199
      valid = true;
      const float3 c = ts_unproject(in, i, j, d);            // :201, mapping_common.py:37-40
      const float x = c.x, y = c.y;
      dep = c.z;
      const TsFrame& fr = batch.f[f];
      px = (fr.R[0] * x + fr.R[1] * y) + fr.R[2] * dep;     // :203 input_R @ pt (rotation only)
      py = (fr.R[3] * x + fr.R[4] * y) + fr.R[5] * dep;
      pz = (fr.R[6] * x + fr.R[7] * y) + fr.R[8] * dep;
      if (tex) {
        int tj, ti;  // texture[j, i] (:206) or color_ind_from_depth_pt (:209)
        if (ts_color_pixel(in, i, j, th, tw, ti, tj)) {
          const uint8_t* p = tex + ((size_t)f * th * tw + (size_t)tj * tw + ti) * 3;
          cr = p[0]; cg = p[1]; cb = p[2];
        }
      }
    }
  }
  const unsigned nv = __popc(__ballot_sync(0xffffffffu, valid));
  const int fresh = bucket_accumulate(valid, bidx + (size_t)tz * bucket_cap, bucket_cap - 1, (uint32_t)tz * bucket_cap, buckets + (size_t)tz * bucket_cap,
                                      bcol ? bcol + (size_t)tz * bucket_cap : nullptr, bl.cnt ? bl.cnt + (size_t)tz * bucket_cap : nullptr, bucket_cap,
                                      (blockIdx.y * gridDim.x + blockIdx.x) * 256u, bl, px, py, pz, dep, in.vs, in.rvs, agg_ok != 0, err,
                                      tex != nullptr, cr, cg, cb);
  append_rays_cta(fresh, (uint32_t)tz * bucket_cap, nv, ray_list, n_rays, ray_cap, ctr, err);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) atomicAdd(&ctr->n_px, (unsigned long long)(hh * ww));
  ts_stamp_end(prof, TS_K_BUCKET);
}

// K1b: point cloud -> buckets.  recast_pcl_to_map_kernel (dense_tsdf.py:167-185).
__global__ void __launch_bounds__(256, 6) k_bucket_points(const float* __restrict__ xyz, int n, const __grid_constant__ TsBatch batch,
                                                        TsIntrin in, int agg_ok, TsBucket* buckets, uint4* bcol, unsigned long long* bidx,
                                                        uint32_t bucket_cap, uint32_t rec_cap, TsBucketLaunch bl, uint32_t* ray_list, int* n_rays, uint32_t ray_cap, TsCounters* ctr,
                                                        int* err, const uint8_t* __restrict__ rgb, unsigned long long* prof) {
  ts_stamp_begin(prof, TS_K_BUCKET);
  cudaGridDependencySynchronize();  // as k_bucket_depth
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  int cr = 0, cg = 0, cb = 0;
  bool valid = false;
  float px = 0.f, py = 0.f, pz = 0.f, len = 0.f;
  if (t < n) {
    const float x = xyz[3 * (size_t)t], y = xyz[3 * (size_t)t + 1], z = xyz[3 * (size_t)t + 2];
    const TsFrame& fr = batch.f[0];
    px = (fr.R[0] * x + fr.R[1] * y) + fr.R[2] * z;  // :175
    py = (fr.R[3] * x + fr.R[4] * y) + fr.R[5] * z;
    pz = (fr.R[6] * x + fr.R[7] * y) + fr.R[8] * z;
    len = sqrtf((px * px + py * py) + pz * pz);       // :176
    valid = len < in.max_ray;                          // :177
    if (rgb) { cr = rgb[3 * (size_t)t]; cg = rgb[3 * (size_t)t + 1]; cb = rgb[3 * (size_t)t + 2]; }  // :179-182
  }
  const unsigned nv = __popc(__ballot_sync(0xffffffffu, valid));
  const int fresh = bucket_accumulate(valid, bidx, bucket_cap - 1, 0u, buckets, bcol, bl.cnt, rec_cap, blockIdx.x * 256u, bl, px, py, pz, len, in.vs,
                                      in.rvs, agg_ok != 0, err, rgb != nullptr, cr, cg, cb);  // :183/:185
  append_rays_cta(fresh, 0u, nv, ray_list, n_rays, ray_cap, ctr, err);
  if (t == 0) atomicAdd(&ctr->n_px, (unsigned long long)n);
  ts_stamp_end(prof, TS_K_BUCKET);
}

// ---------------------------------------------------------------------------
// K2: ray march of textured maps.  process_new_pcl (dense_tsdf.py:236-270) incl. the colour
// (:268-269).  One thread per live bucket (= ray) of any frame of the batch; every step adds
// (w*d, w) to the voxel's pending sums - the reference's racy RMW (:264-267) becomes an
// order-independent sum that k_commit_tma folds into (TSDF, W) - and raises the voxel's colour
// word.  Untextured maps march with tslam_march.cu.
//
// Two accumulation paths:
//  * far field: one 8-byte vector reduction REDG.E.ADD.F32x2 per step into the block's
//    `acc` plane (block pointer cached across steps, hash lookup through L1 on a change);
//  * near field: every ray of a frame - and, with a slowly moving camera, of the whole
//    batch - starts in the same handful of voxels, and same-address reductions
//    serialise in L2 (a ray-like pattern reaches a fraction of the scattered update rate,
//    tools/ubench/red_bench.cu).  Each CTA therefore keeps a 16^3-voxel WINDOW around
//    the sensor origin in shared memory, accumulates samples that fall inside it with
//    native 32-bit integer shared atomics (exact fixed point, lo/hi words), and
//    flushes one reduction per touched window voxel per round.
// The fixed-point scale 2^k is chosen per round from the round's rays, as k_seg_scan chooses it per launch: the largest
// k with max(w, w*dmax) * 2^k < 2^30 (one sample's integer fits 31 bits), so that long rays with small weights keep their
// precision.  A ray with w * 2^k < MB_MIN_WQ (fewer than 14 significant bits) marches on the far path instead.
// ---------------------------------------------------------------------------
#define RM_THREADS 512
#define RM_WIN 16
#define RM_WIN3 4096
#define RM_WIN_STEPS 18      // a sample >= 18 voxels from the sensor origin lies outside the +-8 voxel window on some axis
#define RM_SMEM (RM_WIN3 * 24 + RM_TAB * 8)  // A, B (lo/hi words) and the 64-bit colour word per window voxel, block table

__device__ __forceinline__ void win_add(unsigned int* lo, int* hi, int x) {
  const unsigned int ux = (unsigned int)x;
  const unsigned int old = atomicAdd(lo, ux);
  const int c = (x >> 31) + ((old + ux) < old ? 1 : 0);  // sign extension + carry into the high word
  if (c) atomicAdd(hi, c);
}

__global__ void __launch_bounds__(RM_THREADS, 2) k_raymarch(const __grid_constant__ TsBatch batch, TsIntrin in, TsGrid g,
                                                              const TsBucket* buckets, const uint4* bcol, unsigned long long* bidx,
                                                              uint32_t bucket_shift, TsBucketLaunch bl, const uint32_t* __restrict__ ray_list, const int* __restrict__ n_rays_p, uint32_t ray_cap,
                                                              TsCounters* ctr, unsigned long long* prof) {
  ts_stamp_begin(prof, TS_K_MARCH);
  extern __shared__ __align__(16) unsigned int win[];  // [4][4096]: A.lo, A.hi, B.lo, B.hi
  unsigned int* const w_alo = win;
  int* const w_ahi = (int*)(win + RM_WIN3);
  unsigned int* const w_blo = win + 2 * RM_WIN3;
  int* const w_bhi = (int*)(win + 3 * RM_WIN3);
  unsigned long long* const btab = (unsigned long long*)(win + 4 * RM_WIN3);
  unsigned long long* const w_cw = btab + RM_TAB;  // colour word of every window voxel
  __shared__ int s_org[4];   // window origin (voxels) and submap
  __shared__ unsigned s_fmax;  // round's largest max(w, w*dmax), as bits (non-negative floats order like their bits)
  __shared__ int s_blk[8];   // the <= 8 blocks the window overlaps

  const uint32_t n_rays = min((uint32_t)*n_rays_p, ray_cap);
  const float vs = in.vs;
  const uint32_t lane = threadIdx.x & 31u;
  unsigned int my_updates = 0, my_oob = 0, my_rays = 0;
  const float rvs = in.rvs;
  for (int e = threadIdx.x; e < 4 * RM_WIN3; e += RM_THREADS) win[e] = 0u;
  for (int e = threadIdx.x; e < RM_TAB; e += RM_THREADS) btab[e] = TS_EMPTY;
  for (int e = threadIdx.x; e < RM_WIN3; e += RM_THREADS) w_cw[e] = 0ull;

  // control flow is kept WARP-UNIFORM (32 consecutive rays per warp, march to the longest ray, predicated lanes)
  for (uint32_t base = blockIdx.x * RM_THREADS; base < n_rays; base += gridDim.x * RM_THREADS) {
    if (threadIdx.x == 0) {  // window of this round: around the sensor origin of the round's first ray
      const TsFrame& f0 = batch.f[ray_list[base] >> bucket_shift];
      s_org[0] = iroundf(f0.T[0] / vs) - RM_WIN / 2;
      s_org[1] = iroundf(f0.T[1] / vs) - RM_WIN / 2;
      s_org[2] = iroundf(f0.T[2] / vs) - RM_WIN / 2;
      s_org[3] = f0.submap;
      s_fmax = 0u;
    }
    __syncthreads();
    const int wx = s_org[0], wy = s_org[1], wz = s_org[2], ws = s_org[3];
    const uint32_t r = base + threadIdx.x;
    bool live = r < n_rays;
    int cnt = 0, s = 0, n = 0;
    unsigned int ccr = 0, ccg = 0, ccb = 0;
    uint32_t f = 0;
    TsBucketSums b = {};
    if (live) {
      const uint32_t id = ray_list[r];
      f = id >> bucket_shift;
      b = ts_read_bucket(buckets, bidx, bl, id);
      cnt = b.cnt;
      const uint4 c = bcol[id];
      ccr = c.x; ccg = c.y; ccb = c.z;
      live = cnt > 0;  // :240
    }
    float mx = 0.f, my = 0.f, mz = 0.f, ux = 0.f, uy = 0.f, uz = 0.f, Tx = 0.f, Ty = 0.f, Tz = 0.f, Px = 0.f, Py = 0.f, Pz = 0.f,
          wgt = 0.f, Lr = 0.f;
    unsigned long long cur_key = TS_EMPTY;
    int cur_blk = -1;
    if (live) {
      my_rays++;
      const TsFrame& fr = batch.f[f];
      s = fr.submap;
      TsRayGeom rg;
      if (ts_ray_geom(b, fr.T, in, rg)) {
        mx = rg.mx; my = rg.my; mz = rg.mz;
        ux = rg.ux; uy = rg.uy; uz = rg.uz;
        Tx = fr.T[0]; Ty = fr.T[1]; Tz = fr.T[2];
        Px = rg.Px; Py = rg.Py; Pz = rg.Pz;
        if (ts_in_bounds(g, rg.oi, rg.oj, rg.ok)) {  // occupy[sxyz_to_ijk(pos_p)] = 1 (:248)
          cur_key = ts_pack_key(s, rg.oi >> TS_BSHIFT, rg.oj >> TS_BSHIFT, rg.ok >> TS_BSHIFT);
          cur_blk = ts_get_or_alloc_cached(g, cur_key);
          if (cur_blk >= 0) {
            g.occ[(size_t)cur_blk * TS_B3 + ts_voxel_off(rg.oi, rg.oj, rg.ok)] = 1;
            ts_mark_dirty(g, cur_blk);  // touched blocks are listed even when only `occupy` changed
          }
        }
        n = rg.n;
        wgt = rg.w;
        Lr = rg.L;
      }
    }
    {  // the round's fixed-point scale (tslam_march.cu ray_setup and k_seg_scan form the same bound per launch)
      const float dmax = fmaxf(Lr, (float)n * vs - Lr) + vs;
      unsigned fb = __float_as_uint(fminf(fmaxf(wgt, wgt * dmax), 3.0e38f));
      fb = __reduce_max_sync(0xffffffffu, fb);
      if (lane == 0 && fb) atomicMax(&s_fmax, fb);
    }
    __syncthreads();
    int sk = 30;
    if (s_fmax) {
      int ex;
      frexpf(__uint_as_float(s_fmax), &ex);  // fmax < 2^ex
      sk = 30 - ex;
    }
    sk = max(0, min(48, sk));
    const float fix = __uint_as_float((unsigned)(127 + sk) << 23);  // 2^k
    const int wq = __float2int_rn(wgt * fix);
    const bool win_ok = (s == ws) && wq >= MB_MIN_WQ;
    // every sample also raises the voxel's colour word [frame seq : 22][closeness : 12][rgb : 30] (atomicMax; decoded
    // by the commit) - in the window's shared-memory copy for near-field samples
    unsigned long long cw_hi = 0ull;
    if (live) {
      const float c = (float)cnt;
      const int qr = min(1023, (int)((((float)ccr / c) / 255.0f) * 1023.0f + 0.5f));  // sum_color/c/255 (:269), 10 bits
      const int qg = min(1023, (int)((((float)ccg / c) / 255.0f) * 1023.0f + 0.5f));
      const int qb = min(1023, (int)((((float)ccb / c) / 255.0f) * 1023.0f + 0.5f));
      cw_hi = ((unsigned long long)batch.f[f].seq << 42) | ((unsigned long long)qr << 20) | ((unsigned long long)qg << 10) | (unsigned long long)qb;
    }
    const int nmax = __reduce_max_sync(0xffffffffu, n);
    // voxel of the previous far-field sample: a new block is looked up only when a coordinate leaves its 16-cell
    // (bits >= 4 differ).  Starts at the occupy voxel's block (cur_blk), or at a value no in-bounds voxel shares.
    int pxi = 0x40000000, pyi = 0x40000000, pzi = 0x40000000;
    if (cur_blk >= 0) {
      int ks, kx, ky, kz;
      ts_unpack_key(cur_key, ks, kx, ky, kz);
      pxi = kx << TS_BSHIFT; pyi = ky << TS_BSHIFT; pzi = kz << TS_BSHIFT;
    }
    const unsigned uN = (unsigned)g.N, uNz = (unsigned)g.Nz;
    float jf = 0.0f;
    // One step of the march (:252-267).  WIN: the sample may fall into the shared-memory window (only the first
    // RM_WIN_STEPS steps can: the window reaches 8 voxels from the sensor origin).
    auto step = [&](const int it, const bool WIN) __attribute__((always_inline)) {
      jf += 1.0f;  // :252
      const float x = (ux * jf) * vs + Tx, y = (uy * jf) * vs + Ty, z = (uz * jf) * vs + Tz;  // :253
      const int xi = iroundf(div_vs(x, vs, rvs)), yi = iroundf(div_vs(y, vs, rvs)), zi = iroundf(div_vs(z, vs, rvs));  // :254
      // (ds = L - j*vs would be cheaper and equal up to ~1e-6 m, but it was measured to buy nothing - the kernel is
      // bound by the reductions - and it moves marching-cubes topology where |TSDF| ~ 1e-6: the reference's formula stays.)
      const float vx = Px - x, vy = Py - y, vz = Pz - z;                                       // :258
      const float d = sqrtf((vx * vx + vy * vy) + vz * vz);                                     // :259
      const float ds = d * sgnf((vx * mx + vy * my) + vz * mz);                                 // :260
      const float a = wgt * ds;                                                                 // :264
      const bool stepping = it < n;
      const bool inb = stepping && (unsigned)(xi + g.hN) < uN && (unsigned)(yi + g.hN) < uN && (unsigned)(zi + g.hNz) < uNz;
      my_oob += (stepping && !inb) ? 1u : 0u;
      bool far = inb;
      if (WIN) {
        const unsigned dx = (unsigned)(xi - wx), dy = (unsigned)(yi - wy), dz = (unsigned)(zi - wz);
        const bool in_win = inb && win_ok && dx < RM_WIN && dy < RM_WIN && dz < RM_WIN;
        if (in_win) {  // near field: exact fixed-point sums in shared memory
          const int e = (int)((dx << 8) | (dy << 4) | dz);
          win_add(&w_alo[e], &w_ahi[e], __float2int_rn(a * fix));
          win_add(&w_blo[e], &w_bhi[e], wq);
          const int cl = min(4095, (int)(fabsf(ds) / vs * 16.0f));
          atomicMax(&w_cw[e], cw_hi | ((unsigned long long)(4095 - cl) << 30));
          my_updates++;
        }
        far = inb && !in_win;
      }
      if (far && ((((xi ^ pxi) | (yi ^ pyi) | (zi ^ pzi)) >> TS_BSHIFT) != 0)) {  // block boundary crossed: ~ every 10th step of a lane
        pxi = xi; pyi = yi; pzi = zi;
        cur_blk = rm_lookup(g, btab, ts_pack_key(s, xi >> TS_BSHIFT, yi >> TS_BSHIFT, zi >> TS_BSHIFT), xi >> TS_BSHIFT, yi >> TS_BSHIFT,
                            zi >> TS_BSHIFT);
      }
      __syncwarp();
      if (far && cur_blk >= 0) {  // cur_blk < 0: pool exhausted (error flag raised)
        const size_t vo = (size_t)cur_blk * TS_B3 + ts_voxel_off(xi, yi, zi);
        red_add_f32x2(&g.acc[vo], a, wgt);  // :264,:267
        // color[xi] = ray colour (:268-269): latest frame, then the sample closest to its surface point
        const int cl = min(4095, (int)(fabsf(ds) / vs * 16.0f));
        ts_red_max_u64(&g.cword[vo], cw_hi | ((unsigned long long)(4095 - cl) << 30));
        my_updates++;
      }
    };
    const int n1 = min(nmax, RM_WIN_STEPS);
    int it = 0;
    for (; it < n1; ++it) step(it, true);
#pragma unroll 2
    for (; it < nmax; ++it) step(it, false);
    // flush the window: one reduction per touched voxel.  Pass 1 finds which of the <= 8 overlapped blocks hold
    // touched voxels, 8 threads resolve (activate) exactly those, pass 2 emits the reductions.
    __syncthreads();
    if (threadIdx.x < 8) s_blk[threadIdx.x] = 0;
    __syncthreads();
    {
      unsigned need = 0;
      for (int e = threadIdx.x; e < RM_WIN3; e += RM_THREADS) {
        if (w_blo[e] == 0u && w_bhi[e] == 0) continue;  // B > 0 for every sample (w > 0)
        const int xi = wx + (e >> 8), yi = wy + ((e >> 4) & 15), zi = wz + (e & 15);
        need |= 1u << ((((xi >> TS_BSHIFT) - (wx >> TS_BSHIFT)) << 2) | (((yi >> TS_BSHIFT) - (wy >> TS_BSHIFT)) << 1) |
                       ((zi >> TS_BSHIFT) - (wz >> TS_BSHIFT)));
      }
      need = __reduce_or_sync(0xffffffffu, need);
      if (lane == 0) {
        for (int b8 = 0; b8 < 8; b8++)
          if (need & (1u << b8)) atomicOr((unsigned int*)&s_blk[b8], 1u);
      }
    }
    __syncthreads();
    if (threadIdx.x < 8) {
      int blk = -1;
      if (s_blk[threadIdx.x]) {
        blk = ts_get_or_alloc_cached(g, ts_pack_key(ws, (wx >> TS_BSHIFT) + ((threadIdx.x >> 2) & 1), (wy >> TS_BSHIFT) + ((threadIdx.x >> 1) & 1),
                                                    (wz >> TS_BSHIFT) + (threadIdx.x & 1)));
        if (blk >= 0) ts_mark_dirty(g, blk);
      }
      s_blk[threadIdx.x] = blk;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < RM_WIN3; e += RM_THREADS) {
      const unsigned int blo = w_blo[e];
      const int bhi = w_bhi[e];
      if (blo == 0u && bhi == 0) continue;
      const unsigned int alo = w_alo[e];
      const int ahi = w_ahi[e];
      w_alo[e] = 0u; w_ahi[e] = 0; w_blo[e] = 0u; w_bhi[e] = 0;
      const int xi = wx + (e >> 8), yi = wy + ((e >> 4) & 15), zi = wz + (e & 15);
      const int bsel = (((xi >> TS_BSHIFT) - (wx >> TS_BSHIFT)) << 2) | (((yi >> TS_BSHIFT) - (wy >> TS_BSHIFT)) << 1) |
                       ((zi >> TS_BSHIFT) - (wz >> TS_BSHIFT));
      const int blk = s_blk[bsel];
      if (blk < 0) continue;  // pool exhausted (error flag raised)
      const double rfix = __hiloint2double((1023 - sk) << 20, 0);  // 2^-k
      const float A = (float)(((double)ahi * 4294967296.0 + (double)alo) * rfix);
      const float B = (float)(((double)bhi * 4294967296.0 + (double)blo) * rfix);
      red_add_f32x2(&g.acc[(size_t)blk * TS_B3 + ts_voxel_off(xi, yi, zi)], A, B);
      ts_red_max_u64(&g.cword[(size_t)blk * TS_B3 + ts_voxel_off(xi, yi, zi)], w_cw[e]);
      w_cw[e] = 0ull;
    }
    __syncthreads();
  }
  // statistics: one atomic per warp
  for (int o = 16; o > 0; o >>= 1) {
    my_updates += __shfl_xor_sync(0xffffffffu, my_updates, o);
    my_oob += __shfl_xor_sync(0xffffffffu, my_oob, o);
    my_rays += __shfl_xor_sync(0xffffffffu, my_rays, o);
  }
  if (lane == 0) {
    if (my_updates) atomicAdd(&ctr->n_updates, (unsigned long long)my_updates);
    if (my_oob) atomicAdd(&ctr->n_oob, (unsigned long long)my_oob);
    if (my_rays) atomicAdd(&ctr->n_rays, (unsigned long long)my_rays);
  }
  ts_stamp_end(prof, TS_K_MARCH);
}

// ---------------------------------------------------------------------------
// K3: commit.  Folds the pending (sum w*d, sum w) of every dirty block into
// (TSDF, W_TSDF):  T' = (T*W + A)/(W + B), W' = min(W + B, Wmax), observed = 1
// (dense_tsdf.py:264-267 applied once per voxel per batch).  clamp=0 is the fusion variant (:274-278).
// Each dirty block's two 32 KB planes are moved by the bulk-copy engine (cp.async.bulk: SASS UBLKCP) instead of
// per-thread loads/stores: one elected thread arms an mbarrier with the expected byte count and issues two
// global->shared bulk copies; the CTA waits on the barrier, folds the sums in shared memory, and the elected thread
// streams the updated (TSDF, W) plane and a zeroed accumulator plane back with shared->global bulk stores.  Textured
// maps also set the colour of every touched voxel, per thread in global memory (the colour planes are not copied).
// ---------------------------------------------------------------------------
// The last CTA to finish (every CTA read n_dirty at its start) sets the dirty-list count and `ticket` back to zero.
// It also stamps the end of the commit (prof).
__device__ __forceinline__ void commit_done(const TsGrid& g, int* ticket, unsigned long long* prof) {
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = atomicAdd(ticket, 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    *g.n_dirty = 0;
    *ticket = 0;
    ts_stamp_end_thread(prof, TS_K_COMMIT);
  }
}
#define CM_PLANE_BYTES (TS_B3 * 8)
#define CM_SMEM (2 * CM_PLANE_BYTES + 16)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(void* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(void* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(void* bar, unsigned phase) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(phase)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, void* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, const void* src_smem, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}

__global__ void __launch_bounds__(256) k_commit_tma(TsGrid g, int clamp, int fused_obs, unsigned long long* stamp, unsigned long long seq, int* ticket,
                                                    unsigned long long* prof) {
  extern __shared__ __align__(128) unsigned char cm_smem[];
  ts_stamp_begin(prof, TS_K_COMMIT);
  float2* s_acc = reinterpret_cast<float2*>(cm_smem);
  float2* s_tw = reinterpret_cast<float2*>(cm_smem + CM_PLANE_BYTES);
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(cm_smem + 2 * CM_PLANE_BYTES);
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  cudaGridDependencySynchronize();  // the dirty list comes from k_collect_dirty
  const int nd = *g.n_dirty;
  unsigned phase = 0;
  for (int q = blockIdx.x; q < nd; q += gridDim.x) {
    const int blk = g.dirty_list[q];
    float2* acc = g.acc + (size_t)blk * TS_B3;
    float2* tw = g.tw + (size_t)blk * TS_B3;
    uint8_t* obs = g.obs + (size_t)blk * TS_B3;
    if (threadIdx.x == 0) {
      mbar_expect_tx(bar, 2 * CM_PLANE_BYTES);
      bulk_g2s(s_acc, acc, CM_PLANE_BYTES, bar);
      bulk_g2s(s_tw, tw, CM_PLANE_BYTES, bar);
    }
    mbar_wait(bar, phase);
    phase ^= 1;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const float2 a = s_acc[v];
      // integrate: a voxel is touched iff sum w > 0.  fusion: also voxels whose observed
      // flag was raised by a zero-weight corner (0/0 = NaN is reference behaviour).
      const bool touched = fused_obs ? (a.y != 0.0f || a.x != 0.0f || obs[v] == 2) : (a.y > 0.0f);
      if (touched) {
        const float2 o = s_tw[v];
        const float wn = o.y + a.y;
        float2 r;
        r.x = (o.x * o.y + a.x) / wn;
        r.y = clamp ? fminf(wn, WMAX) : wn;
        s_tw[v] = r;
        obs[v] = 1;
        s_acc[v] = make_float2(0.0f, 0.0f);
        if (g.col) {
          float4* col = g.col + (size_t)blk * TS_B3;
          if (fused_obs) {  // fusion: col holds sum(w*c) (:277) -> weighted mean
            float4 c = col[v];
            c.x = c.x / wn; c.y = c.y / wn; c.z = c.z / wn;
            col[v] = c;
          } else {
            const unsigned long long cw = g.cword[(size_t)blk * TS_B3 + v];
            if (cw) col[v] = make_float4((float)((cw >> 20) & 1023) / 1023.0f, (float)((cw >> 10) & 1023) / 1023.0f, (float)(cw & 1023) / 1023.0f, 0.0f);
          }
        }
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy smem writes -> visible to the bulk engine
    __syncthreads();
    if (threadIdx.x == 0) {
      bulk_s2g(tw, s_tw, CM_PLANE_BYTES);
      bulk_s2g(acc, s_acc, CM_PLANE_BYTES);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // smem may be overwritten by the next block's loads
      g.dirty_flag[blk] = 0;
      g.esdf_dirty[blk] = 1;
      stamp[blk] = seq;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  commit_done(g, ticket, prof);
}

// compact the per-block dirty flags into dirty_list (warp-aggregated append)
__global__ void __launch_bounds__(256) k_collect_dirty(TsGrid g, unsigned long long* prof) {
  ts_stamp_begin(prof, TS_K_COLLECT);
  cudaGridDependencySynchronize();  // the flags are set by the kernels before it
  const int nb = min(*g.n_blocks, g.max_blocks);
  const int stride = gridDim.x * blockDim.x;
  const int iters = (nb + stride - 1) / stride;
  for (int it = 0; it < iters; ++it) {
    const int b = it * stride + blockIdx.x * blockDim.x + threadIdx.x;
    const bool want = b < nb && g.dirty_flag[b] != 0;
    const int row = warp_append_i32(want, g.n_dirty);
    if (want) g.dirty_list[row] = b;
  }
  ts_stamp_end(prof, TS_K_COLLECT);
}
__global__ void k_reset_counters(int* n_rays) { *n_rays = 0; }

// the kernels of this file that need more dynamic shared memory than the default limit
int ts_integrate_init() {
  TS_CUDA(cudaFuncSetAttribute(k_raymarch, cudaFuncAttributeMaxDynamicSharedMemorySize, RM_SMEM));
  TS_CUDA(cudaFuncSetAttribute(k_commit_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, CM_SMEM));
  return TSLAM_OK;
}

// ---------------------------------------------------------------------------
// host: integrate
// ---------------------------------------------------------------------------
// k_collect_dirty, then the commit, whose last CTA sets the dirty-list count back to zero (ticket: scratch_i[4]).  Both
// are launched with programmatic dependent launch (ts_launch_pdl).
int ts_collect_dirty(tslam_tsdf* m, cudaStream_t st, unsigned long long* prof) {
  const int gc = (m->g.max_blocks + 255) / 256 < m->sm_count * 4 ? (m->g.max_blocks + 255) / 256 : m->sm_count * 4;
  TS_CUDA(ts_launch_pdl(k_collect_dirty, gc, 256, 0, st, m->g, prof));
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
int ts_launch_commit(tslam_tsdf* m, cudaStream_t st, int clamp, int fused, unsigned long long* prof) {
  { int rc = ts_collect_dirty(m, st, prof); if (rc) return rc; }
  const unsigned long long seq = ++m->commit_seq;  // stamp of every block this commit writes (incremental mesh)
  TS_CUDA(ts_launch_pdl(k_commit_tma, m->sm_count * 3, 256, CM_SMEM, st, m->g, clamp, fused, m->blk_stamp, seq, m->scratch_i + 4, prof));
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

int ts_flush_pending(tslam_tsdf* m, cudaStream_t st, unsigned long long* prof) {
  if (m->q_n > 0) {  // frames queued by the per-frame API
    int rc = ts_launch_queue(m, st);
    if (rc) return rc;
  }
  if (m->n_integrate_calls > 0) {  // something may be pending
    int rc = ts_launch_commit(m, st, m->clamp_on_commit ? 1 : 0, 0, prof);
    if (rc) return rc;
    m->n_integrate_calls = 0;
  }
  return TSLAM_OK;
}

int ts_check_deferred(tslam_tsdf* m) {
  int err = 0;
  TS_CUDA(cudaMemcpy(&err, m->g.err, 4, cudaMemcpyDeviceToHost));
  if (err) {
    int zero = 0;
    cudaMemcpy(m->g.err, &zero, 4, cudaMemcpyHostToDevice);
    if (err & TS_ERR_POOL_FULL) { ts_set_error("voxel-block pool exhausted (max_blocks=%d): samples were dropped", m->g.max_blocks); return TSLAM_E_POOL_FULL; }
    if (err & TS_ERR_BUCKET_RANGE) { ts_set_error("a point lies more than 4095 voxels from the sensor origin (bucket key range): dropped"); return TSLAM_E_CAPACITY; }
    ts_set_error("device error flags 0x%x (hash table / ray list capacity)", err);
    return TSLAM_E_CAPACITY;
  }
  return TSLAM_OK;
}

// same, ordered on `st` (flush / exporters: the error word is read after the kernels that may have raised it)
int ts_check_deferred_async(tslam_tsdf* m, cudaStream_t st) {
  int err = 0;
  TS_CUDA(cudaMemcpyAsync(&err, m->g.err, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (!err) return TSLAM_OK;
  return ts_check_deferred(m);
}

extern "C" int tslam_tsdf_commit(tslam_tsdf_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  return ts_flush_pending(m, (cudaStream_t)stream);
}

// the commit of sums left pending by tslam_tsdf_fuse_pending (multi-GPU building block, see tslam_dist.cu)
extern "C" int tslam_tsdf_commit_fused(tslam_tsdf_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  return ts_launch_commit(m, (cudaStream_t)stream, 0, 1);
}

static void ts_fill_frame(tslam_tsdf* m, TsFrame& fr, const float* R9, const float* T3, int submap) {
  memcpy(fr.R, R9, 36);
  memcpy(fr.T, T3, 12);
  fr.submap = submap;
  fz_written(m->ver, submap);
  m->frame_seq++;  // 1, 2, ... (texture: later frames win); < 2^22 - TSLAM_MAX_BATCH (ts_seq_renorm runs before that)
  fr.seq = m->frame_seq;
}

extern "C" int tslam_tsdf_integrate_depth(tslam_tsdf_t* m, const uint16_t* depth, int mem, int32_t n_frames, int32_t h, int32_t w,
                                          const float* R9s, const float* T3s, const int32_t* submap_ids, int flags, void* stream) {
  if (m && m->q_n > 0) { int rcq = ts_launch_queue(m, (cudaStream_t)stream); if (rcq) return rcq; }  // frames queued earlier are integrated first
  return ts_integrate_depth_impl(m, depth, mem, n_frames, h, w, R9s, T3s, submap_ids, flags, stream);
}
int ts_check_tex(tslam_tsdf* m, const uint8_t* tex, int th, int tw) {
  if (!tex) return TSLAM_OK;
  if (!m->g.cword) { ts_set_error("colour image given but the map was created with texture_enabled=0"); return TSLAM_E_INVALID; }
  if (th <= 0 || tw <= 0 || (long long)th * tw > m->cfg.max_image_pixels) { ts_set_error("texture %dx%d exceeds max_image_pixels=%d", th, tw, m->cfg.max_image_pixels); return TSLAM_E_INVALID; }
  return TSLAM_OK;
}
extern "C" int tslam_tsdf_integrate_depth_tex(tslam_tsdf_t* m, const uint16_t* depth, const uint8_t* tex, int mem, int32_t n_frames, int32_t h,
                                              int32_t w, int32_t th, int32_t tw, const float* R9s, const float* T3s,
                                              const int32_t* submap_ids, int flags, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  int rc = ts_check_tex(m, tex, th, tw);
  if (rc) return rc;
  if (m->q_n > 0) { rc = ts_launch_queue(m, (cudaStream_t)stream); if (rc) return rc; }
  return ts_integrate_depth_impl(m, depth, mem, n_frames, h, w, R9s, T3s, submap_ids, flags, stream, tex, th, tw);
}
// The colour word of a voxel starts with the 22-bit sequence number of the frame that wrote it ("later frame wins").
// Before the counter could run out (4.2 M frames) every stored word is reset to sequence 0 and counting restarts:
// any later frame still beats every stored colour, which is all the rule needs.
__global__ void __launch_bounds__(256) k_cword_renorm(TsGrid g) {
  const size_t n = (size_t)min(*g.n_blocks, g.max_blocks) * TS_B3;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) g.cword[i] &= (1ull << 42) - 1ull;
}
static int ts_seq_renorm(tslam_tsdf* m, cudaStream_t st, int n_new) {
  if (m->frame_seq + (unsigned)n_new < (1u << 22) - 1u) return TSLAM_OK;
  if (m->g.cword) {
    int rc = ts_flush_pending(m, st);
    if (rc) return rc;
    k_cword_renorm<<<m->sm_count * 8, 256, 0, st>>>(m->g);
    TS_LAUNCH_CHECK(m);
  }
  m->frame_seq = 0;
  return TSLAM_OK;
}

// largest depth (or point-cloud ray length) a bucket sum can add, in metres
double ts_bucket_dmax(const tslam_tsdf* m) {
  return std::max((double)m->in.dmax_mm / 1000.0, (double)m->in.max_ray) * (1.0 + 1e-6);
}

// Bucket index and record parameters of the next launch, in which one bucket can collect at most n points.  Advances
// the launch epoch, and clears the index when it wraps.
static int ts_bucket_launch(tslam_tsdf* m, cudaStream_t st, uint64_t n, TsBucketLaunch& bl) {
  const int shift = ts_bucket_cnt_shift(n, ts_bucket_dmax(m));
  bl.cnt_shift = shift < 0 ? 0 : shift;
  bl.cnt = shift < 0 ? m->bcnt : nullptr;
  if (shift < 0 && !m->bcnt) {  // the plane is sized at create time for the largest launch the handle accepts
    ts_set_error("bucket count plane missing for a launch of %llu points", (unsigned long long)n);
    return TSLAM_E_INVALID;
  }
  bl.slot_bits = m->bk_slot_bits;
  bl.bpos = m->bpos;
  bl.etag = 0ull;
  if (m->bpos) return TSLAM_OK;
  if (++m->bk_epoch > m->bk_epoch_max) {
    TS_CUDA(cudaMemsetAsync(m->bidx, 0, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * 8, st));
    m->bk_epoch = 1;
  }
  bl.etag = (unsigned long long)m->bk_epoch << (BK_KEY_BITS + m->bk_slot_bits);
  return TSLAM_OK;
}
// A launch that stops between the bucket kernel and the ray set-up leaves index entries behind: harmless with epochs
// (the next launch has a new one), cleared here in clearing mode.
static int ts_bucket_abandon(tslam_tsdf* m, cudaStream_t st, int rc) {
  if (m->bpos) TS_CUDA(cudaMemsetAsync(m->bidx, 0, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * 8, st));
  return rc;
}

// One integrate launch on st: the bucket kernel, the ray march of the buckets it opened, and the commit when flags
// holds TSLAM_F_COMMIT.  launch_bucket(bl, agg_ok, prof) enqueues k_bucket_depth or k_bucket_points, the only step that
// differs between depth frames and point clouds; n_bucket_points is the most points one bucket can collect.
// Nothing but kernels goes on the stream between the bucket kernel and the commit, so every boundary of the untextured
// chain is a programmatic dependent launch.  With profiling on, the kernels stamp the launch's row of the profiling
// ring themselves (TS_PROF_WORDS): no event record breaks the chain.
template <class F>
static int ts_integrate_launch(tslam_tsdf* m, cudaStream_t st, const TsBatch& batch, uint32_t bshift, uint64_t n_bucket_points, int flags,
                               F launch_bucket) {
  const long long prow = m->prof_launches % TS_PROF_RING;
  unsigned long long* prof = m->profiling ? m->prof + TS_PROF_WORDS * prow : nullptr;
  const int agg_ok = m->cfg.max_ray_length < 30.0 ? 1 : 0;  // 32-lane int32 sums: |p| <= max_ray * sqrt(1 + tan^2) < 64 m even at 60 deg half-FOV
  TsBucketLaunch bl;
  { int rcb = ts_bucket_launch(m, st, n_bucket_points, bl); if (rcb) return rcb; }
  TS_CUDA(launch_bucket(bl, agg_ok, prof));
  TS_LAUNCH_CHECK(m);
  unsigned ran = 1u << TS_K_BUCKET;
  if (!m->g.cword) {  // untextured maps: the block-binned march (tslam_march.cu)
    int rcm = ts_march_launch(m, st, batch, bshift, bl, prof);  // clears n_rays itself
    if (rcm) return ts_bucket_abandon(m, st, rcm);
    ran |= (1u << TS_K_COUNT) | (1u << TS_K_CLASS_SCAN) | (1u << TS_K_SCATTER) | (1u << TS_K_MARCH);
  } else {
    k_raymarch <<<m->sm_count, RM_THREADS, RM_SMEM, st>>>(batch, m->in, m->g, m->buckets, m->bcol, m->bidx, bshift, bl, m->ray_list, m->n_rays,
                                                         m->ray_list_cap, m->counters, prof);
    TS_LAUNCH_CHECK(m);
    k_reset_counters<<<1, 1, 0, st>>>(m->n_rays);
    TS_LAUNCH_CHECK(m);
    ran |= 1u << TS_K_MARCH;
  }
  m->n_integrate_calls++;
  if (flags & TSLAM_F_COMMIT) {  // commits this launch (it is pending): k_collect_dirty + k_commit_tma
    int rc = ts_flush_pending(m, st, prof);
    if (rc) return rc;
    ran |= (1u << TS_K_COLLECT) | (1u << TS_K_COMMIT);
  }
  if (prof) { m->prof_ran[prow] = (unsigned char)ran; m->prof_launches++; }
  return TSLAM_OK;
}

int ts_integrate_depth_impl(tslam_tsdf_t* m, const uint16_t* depth, int mem, int32_t n_frames, int32_t h, int32_t w, const float* R9s,
                            const float* T3s, const int32_t* submap_ids, int flags, void* stream, const uint8_t* tex, int th, int tw) {
  if (!m || !depth || !R9s || !T3s || n_frames < 0 || h <= 0 || w <= 0) { ts_set_error("bad argument"); return TSLAM_E_INVALID; }
  if ((long long)h * w > m->cfg.max_image_pixels) { ts_set_error("frame %dx%d exceeds max_image_pixels=%d", h, w, m->cfg.max_image_pixels); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const int step = m->cfg.recast_step;
  const int hh = (int)((double)h / step), ww = (int)((double)w / step);  // range(0, h/step) (dense_tsdf.py:192,194)
  if (hh <= 0 || ww <= 0) return TSLAM_OK;
  uint32_t bshift = 0;
  while ((1u << bshift) < m->bucket_cap) bshift++;
  for (int base = 0; base < n_frames; base += TSLAM_MAX_BATCH) {
    const int nf = (n_frames - base < TSLAM_MAX_BATCH) ? (n_frames - base) : TSLAM_MAX_BATCH;
    { int rcs = ts_seq_renorm(m, st, nf); if (rcs) return rcs; }
    TsBatch batch;
    for (int q = 0; q < nf; q++) {
      const int sid = submap_ids ? submap_ids[base + q] : 0;
      if (sid < 0 || sid >= m->cfg.max_submaps) { ts_set_error("bad submap id %d", sid); return TSLAM_E_INVALID; }
      ts_fill_frame(m, batch.f[q], R9s + 9 * (size_t)(base + q), T3s + 3 * (size_t)(base + q), sid);
    }
    const uint16_t* src = depth + (size_t)base * h * w;
    const bool stage0 = mem == TSLAM_MEM_HOST;  // host batches are staged in buffer 0 of the per-frame queue's staging area
    if (stage0) {
      if (m->ev_free_valid[0]) TS_CUDA(cudaStreamWaitEvent(st, m->ev_free[0], 0));  // kernels of an earlier queue launch still read it
      TS_CUDA(cudaMemcpyAsync(m->depth_stage, src, (size_t)nf * h * w * 2, cudaMemcpyHostToDevice, st));
      src = m->depth_stage;
    }
    const uint8_t* tsrc = tex ? tex + (size_t)base * th * tw * 3 : nullptr;
    if (tex && mem == TSLAM_MEM_HOST) {
      TS_CUDA(cudaMemcpyAsync(m->tex_stage, tsrc, (size_t)nf * th * tw * 3, cudaMemcpyHostToDevice, st));
      tsrc = m->tex_stage;
    }
    dim3 grid1((ww + 31) / 32, (hh + 7) / 8, nf);
    if ((size_t)grid1.x * grid1.y * 256 > m->bucket_cap) {  // every 32x8-pixel CTA tile owns 256 bucket records of its frame
      ts_set_error("frame %dx%d (sampled %dx%d) has too many partial pixel tiles for max_image_pixels=%d", h, w, hh, ww, m->cfg.max_image_pixels);
      return TSLAM_E_INVALID;
    }
    int rc = ts_integrate_launch(m, st, batch, bshift, (uint64_t)hh * ww, flags, [&](const TsBucketLaunch& bl, int agg_ok, unsigned long long* prof) {
      return ts_launch_pdl(k_bucket_depth, grid1, 256, 0, st, (const uint16_t*)src, h * w, step, w, hh, ww, batch, m->in, agg_ok, m->buckets, m->bcol,
                           m->bidx, m->bucket_cap, bl, m->ray_list, m->n_rays, m->ray_list_cap, m->counters, m->g.err, tsrc, th, tw, prof);
    });
    if (rc) return rc;
    if (stage0) {  // the queue must not refill buffer 0 before these kernels have read it
      TS_CUDA(cudaEventRecord(m->ev_free[0], st));
      m->ev_free_valid[0] = true;
    }
  }
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_integrate_points(tslam_tsdf_t* m, const float* xyz, int mem, int32_t n, const float* R9, const float* T3,
                                           int32_t submap, int flags, void* stream) {
  return tslam_tsdf_integrate_points_rgb(m, xyz, nullptr, mem, n, R9, T3, submap, flags, stream);
}
extern "C" int tslam_tsdf_integrate_points_rgb(tslam_tsdf_t* m, const float* xyz, const uint8_t* rgb, int mem, int32_t n, const float* R9,
                                               const float* T3, int32_t submap, int flags, void* stream) {
  if (m && rgb && !m->g.cword) { ts_set_error("point colours given but the map was created with texture_enabled=0"); return TSLAM_E_INVALID; }
  if (!m || (!xyz && n > 0) || !R9 || !T3 || n < 0) { ts_set_error("bad argument"); return TSLAM_E_INVALID; }
  if (n > m->cfg.max_points) { ts_set_error("n=%d exceeds max_points=%d", n, m->cfg.max_points); return TSLAM_E_INVALID; }
  if (submap < 0 || submap >= m->cfg.max_submaps) { ts_set_error("bad submap id %d", submap); return TSLAM_E_INVALID; }
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  { int rcs = ts_seq_renorm(m, st, 1); if (rcs) return rcs; }
  TsBatch batch;
  ts_fill_frame(m, batch.f[0], R9, T3, submap);
  const float* src = xyz;
  if (mem == TSLAM_MEM_HOST) {
    TS_CUDA(cudaMemcpyAsync(m->points_stage, xyz, (size_t)n * 12, cudaMemcpyHostToDevice, st));
    src = m->points_stage;
  }
  const uint8_t* csrc = rgb;
  if (rgb && mem == TSLAM_MEM_HOST) {
    TS_CUDA(cudaMemcpyAsync(m->rgb_stage, rgb, (size_t)n * 3, cudaMemcpyHostToDevice, st));
    csrc = m->rgb_stage;
  }
  const uint32_t bshift = 31;  // every ray belongs to batch.f[0]
  const uint32_t cap_total = (uint32_t)TSLAM_MAX_BATCH * m->bucket_cap;  // power of two
  const uint32_t rec_cap = (uint32_t)n;  // a bucket's record slot is the index of the point whose thread owns its CTA sums
  return ts_integrate_launch(m, st, batch, bshift, (uint64_t)n, flags, [&](const TsBucketLaunch& bl, int agg_ok, unsigned long long* prof) {
    return ts_launch_pdl(k_bucket_points, (n + 255) / 256, 256, 0, st, src, n, batch, m->in, agg_ok, m->buckets, m->bcol, m->bidx, cap_total, rec_cap, bl,
                         m->ray_list, m->n_rays, m->ray_list_cap, m->counters, m->g.err, csrc, prof);
  });
}
