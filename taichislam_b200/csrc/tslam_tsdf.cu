// libtslam.so - TSDF map: hash grid of 16^3 voxel blocks, depth / point-cloud
// integration (bucket -> ray-march -> commit), I/O and export kernels.  sm_90a.
//
// Reference semantics: taichi_slam/mapping/dense_tsdf.py (cited per kernel).
// Compiled with -fmad=false: the index-forming arithmetic must round exactly like
// the strict-IEEE statement of the reference source (voxel indices are compared
// bit-for-bit by the parity tests).
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <cmath>
#include <vector>
#include <cuda_fp16.h>
#include "tslam_internal.cuh"
#include "tslam_bucket.cuh"

// ---------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------
static thread_local char g_err[512] = "";
void ts_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int ts_cuda_fail(cudaError_t e, const char* what) {
  ts_set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) ? TSLAM_E_NOGPU : TSLAM_E_CUDA;
}
extern "C" const char* tslam_last_error(void) { return g_err; }
extern "C" int tslam_abi_version(void) { return TSLAM_ABI_VERSION; }
extern "C" int tslam_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

// bucket index entry: [launch epoch : 25 - S][record slot + 1 : S][bx + 4096 : 13][by + 4096 : 13][bz + 4096 : 13],
// S = TsBucketLaunch::slot_bits.  An entry whose epoch is not the launch's counts as empty, so nobody clears the index
// between launches: the host clears it once when the epoch wraps (ts_bucket_launch).  A handle whose record slots
// leave fewer than TS_BK_MIN_EPOCH_BITS for the epoch runs in clearing mode instead: S = 25, no epoch, and the ray
// set-up zeroes the entry of every record it reads (TsBucketLaunch::bpos).
#define BK_OFF 4096
#define BK_KEY_BITS 39
#define BK_KEY_MASK ((1ull << BK_KEY_BITS) - 1ull)
#define BK_MAX_SLOTS ((1u << 25) - 2u)
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

// accumulate one unprojected point per lane into the frame's bucket grid.
// process_point (dense_tsdf.py:227-234) with exact fixed-point sums.  Lanes of a warp that fall into
// the same bucket (neighbouring pixels usually do) are merged first (match.any + redux): one probe and
// one set of reductions per distinct bucket per warp instead of per pixel.  The index maps the bucket's
// voxel to a RECORD slot.  Slots need no allocator: every warp owns the 32 records [slot_base, slot_base + 32)
// (it holds at most 32 distinct buckets), a probing lane brings the slot of its rank along and publishes it
// with the key in ONE 64-bit CAS, so nobody ever waits for a slot.  The slot is private until that CAS publishes it,
// so the lane STORES its warp's sums there first (the record needs no zeroing); lanes that find the bucket open add
// into its record.  A lane that loses the race leaves its slot written but unnamed: nobody reads it.
// Must be called by all 32 lanes; `valid` masks lanes without a point.  Returns the record slot when this
// lane OPENED a bucket (the bucket becomes one ray; the caller appends it to the ray list), else -1.
__device__ __forceinline__ int bucket_accumulate(bool valid, unsigned long long* idx, uint32_t cap_mask, uint32_t idx_base, TsBucket* recs,
                                                 uint4* cols, uint32_t* cnts, uint32_t rec_cap, uint32_t slot_base, const TsBucketLaunch& bl, float px,
                                                 float py, float pz, float dep, float vs, bool agg_ok, int* err, bool tex = false, int cr = 0,
                                                 int cg = 0, int cb = 0) {
  const int bx = iroundf(px / vs), by = iroundf(py / vs), bz = iroundf(pz / vs);  // xyz_to_ijk mapping_common.py:240-243
  if (valid && ((unsigned)(bx + (BK_OFF - 1)) > 2u * (BK_OFF - 1) || (unsigned)(by + (BK_OFF - 1)) > 2u * (BK_OFF - 1) ||
                (unsigned)(bz + (BK_OFF - 1)) > 2u * (BK_OFF - 1))) {
    atomicOr(err, TS_ERR_BUCKET_RANGE);
    valid = false;
  }
  const unsigned long long key = bucket_key(bx, by, bz);
  long long qx = __float2ll_rn(px * FIXQ), qy = __float2ll_rn(py * FIXQ), qz = __float2ll_rn(pz * FIXQ), qd = __float2ll_rn(dep * FIXQ);
  int cnt = 1;
  bool act = valid;  // this lane probes and adds
  const unsigned vmask = __ballot_sync(0xffffffffu, valid);
  if (agg_ok) {  // |q| < 2^26 (max_ray < 64 m): a 32-lane sum fits int32
    // every lane adds its point to the shared-memory slot of its group's first lane (native 32-bit ATOMS; slots of
    // different groups sit in different banks: stride 9 words), the leaders read the totals back.  (The
    // redux-per-group loop this replaces was 17 % of the kernel's instructions.)
    __shared__ int s_agg[8][32][9];
    const int lane = threadIdx.x & 31, wid = (threadIdx.x >> 5) & 7;
    int* mine = s_agg[wid][lane];
    mine[0] = 0; mine[1] = 0; mine[2] = 0; mine[3] = 0; mine[4] = 0;
    if (tex) { mine[5] = 0; mine[6] = 0; mine[7] = 0; }
    __syncwarp();
    if (valid) {
      const unsigned grp = __match_any_sync(vmask, key);
      const int lead = __ffs(grp) - 1;
      act = lane == lead;
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
  }
  uint32_t h = ts_hash(key) & cap_mask;
  const unsigned amask = __ballot_sync(0xffffffffu, act);
  if (!act) return -1;
  const uint32_t my_slot = slot_base + (uint32_t)__popc(amask & ((1u << (threadIdx.x & 31)) - 1u));
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
// blockIdx.z = frame of the batch.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_bucket_depth(const uint16_t* __restrict__ depth, int frame_stride, int row_mul, int w, int hh, int ww,
                                                       const __grid_constant__ TsBatch batch, TsIntrin in, int agg_ok,
                                                       TsBucket* buckets, uint4* bcol, unsigned long long* bidx, uint32_t bucket_cap,
                                                       TsBucketLaunch bl, uint32_t* ray_list, int* n_rays, uint32_t ray_cap, TsCounters* ctr, int* err,
                                                       const uint8_t* __restrict__ tex, int th, int tw) {
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
    const float df = (float)d;
    if (d != 0 && !(df > in.dmax_mm || df < in.dmin_mm)) {  // :196-199
      valid = true;
      dep = df / 1000.0f;                                    // :201
      const float x = ((float)i - in.cx) * dep / in.fx;     // mapping_common.py:37-40
      const float y = ((float)j - in.cy) * dep / in.fy;
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
                                      ((blockIdx.y * gridDim.x + blockIdx.x) * 8u + (uint32_t)wid) * 32u, bl, px, py, pz, dep, in.vs, agg_ok != 0,
                                      err, tex != nullptr, cr, cg, cb);
  append_rays_cta(fresh, (uint32_t)tz * bucket_cap, nv, ray_list, n_rays, ray_cap, ctr, err);
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) atomicAdd(&ctr->n_px, (unsigned long long)(hh * ww));
}

// K1b: point cloud -> buckets.  recast_pcl_to_map_kernel (dense_tsdf.py:167-185).
__global__ void __launch_bounds__(256) k_bucket_points(const float* __restrict__ xyz, int n, const __grid_constant__ TsBatch batch,
                                                        TsIntrin in, int agg_ok, TsBucket* buckets, uint4* bcol, unsigned long long* bidx,
                                                        uint32_t bucket_cap, uint32_t rec_cap, TsBucketLaunch bl, uint32_t* ray_list, int* n_rays, uint32_t ray_cap, TsCounters* ctr,
                                                        int* err, const uint8_t* __restrict__ rgb) {
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
  const int fresh = bucket_accumulate(valid, bidx, bucket_cap - 1, 0u, buckets, bcol, bl.cnt, rec_cap, (uint32_t)(t & ~31), bl, px, py, pz, len, in.vs,
                                      agg_ok != 0, err, rgb != nullptr, cr, cg, cb);  // :183/:185
  append_rays_cta(fresh, 0u, nv, ray_list, n_rays, ray_cap, ctr, err);
  if (t == 0) atomicAdd(&ctr->n_px, (unsigned long long)n);
}

// ---------------------------------------------------------------------------
// K2: ray march.  process_new_pcl (dense_tsdf.py:236-270).  One thread per live
// bucket (= ray) of any frame of the batch; every step adds (w*d, w) to the voxel's
// pending sums - the reference's racy RMW (:264-267) becomes an order-independent
// sum that k_commit folds into (TSDF, W).
//
// Two accumulation paths:
//  * far field: one 8-byte vector reduction REDG.E.ADD.F32x2 per step into the block's
//    `acc` plane (block pointer cached across steps, hash lookup through L1 on a change);
//  * near field: every ray of a frame - and, with a slowly moving camera, of the whole
//    batch - starts in the same handful of voxels, and same-address reductions
//    serialise in L2 (a ray-like pattern reaches a fraction of the scattered update rate,
//    tools/ubench/red_bench.cu).  Each CTA therefore keeps a 16^3-voxel WINDOW around
//    the sensor origin in shared memory, accumulates samples that fall inside it with
//    native 32-bit integer shared atomics (exact 2^-24 fixed point, lo/hi words), and
//    flushes one reduction per touched window voxel per round.
// ---------------------------------------------------------------------------
#define RM_THREADS 512
#define RM_WIN 16
#define RM_WIN3 4096
#define RM_FIX 16777216.0f   // 2^24
#define RM_WIN_STEPS 18      // a sample >= 18 voxels from the sensor origin lies outside the +-8 voxel window on some axis
#define RM_SMEM (RM_WIN3 * 16 + RM_TAB * 8)
#define RM_SMEM_TEX (RM_SMEM + RM_WIN3 * 8)  // textured maps: + one 64-bit colour word per window voxel

__device__ __forceinline__ void win_add(unsigned int* lo, int* hi, int x) {
  const unsigned int ux = (unsigned int)x;
  const unsigned int old = atomicAdd(lo, ux);
  const int c = (x >> 31) + ((old + ux) < old ? 1 : 0);  // sign extension + carry into the high word
  if (c) atomicAdd(hi, c);
}

template <bool TEX>
__global__ void __launch_bounds__(RM_THREADS, 2) k_raymarch(const __grid_constant__ TsBatch batch, TsIntrin in, TsGrid g,
                                                              const TsBucket* buckets, const uint4* bcol, unsigned long long* bidx,
                                                              uint32_t bucket_shift, TsBucketLaunch bl, const uint32_t* __restrict__ ray_list, const int* __restrict__ n_rays_p, uint32_t ray_cap,
                                                              TsCounters* ctr) {
  extern __shared__ __align__(16) unsigned int win[];  // [4][4096]: A.lo, A.hi, B.lo, B.hi
  unsigned int* const w_alo = win;
  int* const w_ahi = (int*)(win + RM_WIN3);
  unsigned int* const w_blo = win + 2 * RM_WIN3;
  int* const w_bhi = (int*)(win + 3 * RM_WIN3);
  unsigned long long* const btab = (unsigned long long*)(win + 4 * RM_WIN3);
  unsigned long long* const w_cw = btab + RM_TAB;  // TEX only: colour word of every window voxel
  __shared__ int s_org[4];   // window origin (voxels) and submap
  __shared__ int s_blk[8];   // the <= 8 blocks the window overlaps

  const uint32_t n_rays = min((uint32_t)*n_rays_p, ray_cap);
  const float vs = in.vs;
  const uint32_t lane = threadIdx.x & 31u;
  unsigned int my_updates = 0, my_oob = 0, my_rays = 0;
  const float rvs = in.rvs;
  for (int e = threadIdx.x; e < 4 * RM_WIN3; e += RM_THREADS) win[e] = 0u;
  for (int e = threadIdx.x; e < RM_TAB; e += RM_THREADS) btab[e] = TS_EMPTY;
  if (TEX)
    for (int e = threadIdx.x; e < RM_WIN3; e += RM_THREADS) w_cw[e] = 0ull;

  // control flow is kept WARP-UNIFORM (32 consecutive rays per warp, march to the longest ray, predicated lanes)
  for (uint32_t base = blockIdx.x * RM_THREADS; base < n_rays; base += gridDim.x * RM_THREADS) {
    if (threadIdx.x == 0) {  // window of this round: around the sensor origin of the round's first ray
      const TsFrame& f0 = batch.f[ray_list[base] >> bucket_shift];
      s_org[0] = iroundf(f0.T[0] / vs) - RM_WIN / 2;
      s_org[1] = iroundf(f0.T[1] / vs) - RM_WIN / 2;
      s_org[2] = iroundf(f0.T[2] / vs) - RM_WIN / 2;
      s_org[3] = f0.submap;
    }
    __syncthreads();
    const int wx = s_org[0], wy = s_org[1], wz = s_org[2], ws = s_org[3];
    const uint32_t r = base + threadIdx.x;
    bool live = r < n_rays;
    int cnt = 0, s = 0, n = 0;
    long long sx = 0, sy = 0, sz = 0, sd = 0;
    unsigned int ccr = 0, ccg = 0, ccb = 0;
    uint32_t f = 0;
    if (live) {
      const uint32_t id = ray_list[r];
      f = id >> bucket_shift;
      const TsBucket* bk = &buckets[id];
      sx = bk->sx; sy = bk->sy; sz = bk->sz;
      const unsigned long long cd = bk->cd;
      cnt = bl.cnt ? (int)bl.cnt[id] : (int)(cd >> bl.cnt_shift);
      sd = bl.cnt ? (long long)cd : (long long)(cd & ((1ull << bl.cnt_shift) - 1ull));
      if (TEX) { const uint4 c = bcol[id]; ccr = c.x; ccg = c.y; ccb = c.z; }
      // PCLroot.deactivate_all() (:163): clearing mode hands the index entry back zeroed
      if (bl.bpos) bidx[bl.bpos[id]] = 0ull;
      live = cnt > 0;  // :240
    }
    float mx = 0.f, my = 0.f, mz = 0.f, ux = 0.f, uy = 0.f, uz = 0.f, Tx = 0.f, Ty = 0.f, Tz = 0.f, Px = 0.f, Py = 0.f, Pz = 0.f,
          wgt = 0.f;
    unsigned long long cur_key = TS_EMPTY;
    int cur_blk = -1;
    if (live) {
      my_rays++;
      const TsFrame& fr = batch.f[f];
      s = fr.submap;
      const double den = (double)cnt * FIXQ_D;
      mx = (float)((double)sx / den);  // pos_s2p = sum/c (:243), exact mean
      my = (float)((double)sy / den);
      mz = (float)((double)sz / den);
      const float zc = (float)((double)sd / den);  // z = new_pcl_z/c (:247)
      const float L = sqrtf((mx * mx + my * my) + mz * mz);  // :244
      if (L > 0.0f) {
        ux = mx / L; uy = my / L; uz = mz / L;  // :245
        Tx = fr.T[0]; Ty = fr.T[1]; Tz = fr.T[2];
        Px = mx + Tx; Py = my + Ty; Pz = mz + Tz;  // :246
        // occupy[sxyz_to_ijk(pos_p)] = 1 (:248)
        const int oi = iroundf(Px / vs), oj = iroundf(Py / vs), ok = iroundf(Pz / vs);
        if (ts_in_bounds(g, oi, oj, ok)) {
          cur_key = ts_pack_key(s, oi >> TS_BSHIFT, oj >> TS_BSHIFT, ok >> TS_BSHIFT);
          cur_blk = ts_get_or_alloc_cached(g, cur_key);
          if (cur_blk >= 0) {
            g.occ[(size_t)cur_blk * TS_B3 + ts_voxel_off(oi, oj, ok)] = 1;
            ts_mark_dirty(g, cur_blk);  // touched blocks are listed even when only `occupy` changed
          }
        }
        n = (int)fminf(L / vs + (float)in.internal_voxels, in.max_steps);  // :249-251
        wgt = 1.0f / (zc * zc);  // w_x_p(d>=0, z) (:216-225, :262)
      }
    }
    const bool win_ok = (s == ws) && wgt < 120.0f;  // fixed-point range of the window words
    // textured maps: every sample also raises the voxel's colour word [frame seq : 22][closeness : 12][rgb : 30]
    // (atomicMax; decoded by k_commit) - in the window's shared-memory copy for near-field samples
    unsigned long long cw_hi = 0ull;
    if (TEX && live && cnt > 0) {
      const float c = (float)cnt;
      const int qr = min(1023, (int)((((float)ccr / c) / 255.0f) * 1023.0f + 0.5f));  // sum_color/c/255 (:269), 10 bits
      const int qg = min(1023, (int)((((float)ccg / c) / 255.0f) * 1023.0f + 0.5f));
      const int qb = min(1023, (int)((((float)ccb / c) / 255.0f) * 1023.0f + 0.5f));
      cw_hi = ((unsigned long long)batch.f[f].seq << 42) | ((unsigned long long)qr << 20) | ((unsigned long long)qg << 10) | (unsigned long long)qb;
    }
    const int wq = __float2int_rn(wgt * RM_FIX);
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
        const bool in_win = inb && win_ok && dx < RM_WIN && dy < RM_WIN && dz < RM_WIN && fabsf(a) < 120.0f;
        if (in_win) {  // near field: exact fixed-point sums in shared memory
          const int e = (int)((dx << 8) | (dy << 4) | dz);
          win_add(&w_alo[e], &w_ahi[e], __float2int_rn(a * RM_FIX));
          win_add(&w_blo[e], &w_bhi[e], wq);
          if (TEX) {
            const int cl = min(4095, (int)(fabsf(ds) / vs * 16.0f));
            atomicMax(&w_cw[e], cw_hi | ((unsigned long long)(4095 - cl) << 30));
          }
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
        if (TEX) {  // color[xi] = ray colour (:268-269): latest frame, then the sample closest to its surface point
          const int cl = min(4095, (int)(fabsf(ds) / vs * 16.0f));
          ts_red_max_u64(&g.cword[vo], cw_hi | ((unsigned long long)(4095 - cl) << 30));
        }
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
      const float A = (float)(((double)ahi * 4294967296.0 + (double)alo) * (1.0 / 16777216.0));
      const float B = (float)(((double)bhi * 4294967296.0 + (double)blo) * (1.0 / 16777216.0));
      red_add_f32x2(&g.acc[(size_t)blk * TS_B3 + ts_voxel_off(xi, yi, zi)], A, B);
      if (TEX) {
        ts_red_max_u64(&g.cword[(size_t)blk * TS_B3 + ts_voxel_off(xi, yi, zi)], w_cw[e]);
        w_cw[e] = 0ull;
      }
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
}

// ---------------------------------------------------------------------------
// K3: commit.  Folds the pending (sum w*d, sum w) of every dirty block into
// (TSDF, W_TSDF):  T' = (T*W + A)/(W + B), W' = min(W + B, Wmax), observed = 1
// (dense_tsdf.py:264-267 applied once per voxel per batch).  One CTA per block,
// fully coalesced float2 streams.  clamp=0 is the fusion variant (:274-278).
// ---------------------------------------------------------------------------
// The last CTA to finish (every CTA read n_dirty at its start) sets the dirty-list count and `ticket` back to zero.
__device__ __forceinline__ void commit_done(const TsGrid& g, int* ticket) {
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = atomicAdd(ticket, 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) { *g.n_dirty = 0; *ticket = 0; }
}
__global__ void __launch_bounds__(256) k_commit(TsGrid g, int clamp, int fused_obs, unsigned long long* stamp, unsigned long long seq, int* ticket) {
  cudaGridDependencySynchronize();  // the dirty list comes from k_collect_dirty
  const int nd = *g.n_dirty;
  for (int q = blockIdx.x; q < nd; q += gridDim.x) {
    const int blk = g.dirty_list[q];
    float2* acc = g.acc + (size_t)blk * TS_B3;
    float2* tw = g.tw + (size_t)blk * TS_B3;
    uint8_t* obs = g.obs + (size_t)blk * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const float2 a = acc[v];
      // integrate: a voxel is touched iff sum w > 0.  fusion: also voxels whose observed
      // flag was raised by a zero-weight corner (0/0 = NaN is reference behaviour).
      const bool touched = fused_obs ? (a.y != 0.0f || a.x != 0.0f || obs[v] == 2) : (a.y > 0.0f);
      if (touched) {
        const float2 o = tw[v];
        const float wn = o.y + a.y;
        float2 r;
        r.x = (o.x * o.y + a.x) / wn;
        r.y = clamp ? fminf(wn, WMAX) : wn;
        tw[v] = r;
        obs[v] = 1;
        acc[v] = make_float2(0.0f, 0.0f);
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
    if (threadIdx.x == 0) { g.dirty_flag[blk] = 0; g.esdf_dirty[blk] = 1; stamp[blk] = seq; }
  }
  commit_done(g, ticket);
}
// ---------------------------------------------------------------------------
// K3 (TMA variant): the same commit, with each dirty block's two 32 KB planes moved by the bulk-copy engine
// (cp.async.bulk: SASS UBLKCP) instead of per-thread loads/stores: one elected thread arms an mbarrier with the
// expected byte count and issues two global->shared bulk copies; the CTA waits on the barrier, folds the sums in
// shared memory, and the elected thread streams the updated (TSDF, W) plane and a zeroed accumulator plane back
// with shared->global bulk stores.
// ---------------------------------------------------------------------------
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

__global__ void __launch_bounds__(256) k_commit_tma(TsGrid g, int clamp, int fused_obs, unsigned long long* stamp, unsigned long long seq, int* ticket) {
  extern __shared__ __align__(128) unsigned char cm_smem[];
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
  commit_done(g, ticket);
}

// compact the per-block dirty flags into dirty_list (warp-aggregated append)
__global__ void __launch_bounds__(256) k_collect_dirty(TsGrid g) {
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
}
__global__ void k_reset_counters(int* a, int* b) {
  if (a) *a = 0;
  if (b) *b = 0;
}

// ---------------------------------------------------------------------------
// host: create / destroy / reset
// ---------------------------------------------------------------------------
static size_t next_pow2(size_t v) {
  size_t p = 1;
  while (p < v) p <<= 1;
  return p;
}

static void fill_jet_host(float* cm) {
  // colormap[i] = matplotlib.cm.jet(i/1024) (mapping_common.py:158-163) = 256-entry LUT of
  // the piecewise-linear jet segment data, sampled at i//4.
  static const float r[][2] = {{0, 0}, {0.35f, 0}, {0.66f, 1}, {0.89f, 1}, {1, 0.5f}};
  static const float gg[][2] = {{0, 0}, {0.125f, 0}, {0.375f, 1}, {0.64f, 1}, {0.91f, 0}, {1, 0}};
  static const float b[][2] = {{0, 0.5f}, {0.11f, 1}, {0.34f, 1}, {0.65f, 0}, {1, 0}};
  auto seg = [](const float (*d)[2], int n, float x) {
    for (int i = 1; i < n; i++)
      if (x <= d[i][0]) {
        float t = (x - d[i - 1][0]) / (d[i][0] - d[i - 1][0]);
        return d[i - 1][1] + t * (d[i][1] - d[i - 1][1]);
      }
    return d[n - 1][1];
  };
  for (int i = 0; i < 1024; i++) {
    float x = (float)(i / 4) / 255.0f;
    cm[3 * i] = seg(r, 5, x);
    cm[3 * i + 1] = seg(gg, 6, x);
    cm[3 * i + 2] = seg(b, 5, x);
  }
}

static void ts_fill_intrin(tslam_tsdf* m) {
  const tslam_tsdf_config_t& c = m->cfg;
  m->in.fx = (float)c.fx; m->in.fy = (float)c.fy; m->in.cx = (float)c.cx; m->in.cy = (float)c.cy;
  m->in.dmin_mm = (float)(c.min_ray_length * 1000.0);
  m->in.dmax_mm = (float)(c.max_ray_length * 1000.0);
  m->in.vs = (float)c.voxel_scale;
  m->in.rvs = 1.0f / m->in.vs;
  m->in.max_steps = (float)(c.max_ray_length / c.voxel_scale);
  m->in.max_ray = (float)c.max_ray_length;
  m->in.internal_voxels = c.internal_voxels;
  m->in.step = c.recast_step;
  m->in.tex = c.texture_enabled;
}

// largest depth (or point-cloud ray length) a bucket sum can add, in metres
static double ts_bucket_dmax(const tslam_tsdf* m) {
  return std::max((double)m->in.dmax_mm / 1000.0, (double)m->in.max_ray) * (1.0 + 1e-6);
}

extern "C" int tslam_tsdf_create(const tslam_tsdf_config_t* cfg, tslam_tsdf_t** out) {
  if (!cfg || !out) { ts_set_error("null argument"); return TSLAM_E_INVALID; }
  *out = nullptr;
  if (cfg->voxel_scale <= 0 || cfg->N <= 0 || cfg->Nz <= 0 || cfg->recast_step <= 0 || cfg->N > 16384 || cfg->Nz > 16384) {
    ts_set_error("invalid config (voxel_scale/N/Nz/recast_step)");
    return TSLAM_E_INVALID;
  }
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    ts_set_error("no CUDA device visible: libtslam has no CPU fallback");
    return TSLAM_E_NOGPU;
  }
  tslam_tsdf* m = new tslam_tsdf();
  memset(m, 0, sizeof(*m));
  m->cfg = *cfg;
  TS_CUDA(cudaGetDevice(&m->device));
  cudaDeviceProp prop;
  TS_CUDA(cudaGetDeviceProperties(&prop, m->device));
  m->sm_count = prop.multiProcessorCount;
  if (m->cfg.max_submaps <= 0) m->cfg.max_submaps = 1024;
  if (m->cfg.max_submaps > 1024) m->cfg.max_submaps = 1024;
  if (m->cfg.max_image_pixels <= 0) m->cfg.max_image_pixels = 640 * 480;
  if (m->cfg.max_points <= 0) m->cfg.max_points = 1 << 20;
  // block pool capacity: the dense block count when that is small, else 32768 blocks
  const long long nb = (long long)((cfg->N + TS_B - 1) / TS_B + 1);
  const long long nbz = (long long)((cfg->Nz + TS_B - 1) / TS_B + 1);
  long long dense_blocks = nb * nb * nbz * (cfg->is_global_map ? 1 : 4);
  // default pool: the dense block count, at least 32768 blocks (2.4 GB: a submap collection keeps growing with every
  // keyframe - the reference's pointer SNodes grow on demand), at most 131072 (9.4 GB); callers that know better pass
  // max_blocks.  Exhaustion drops samples and raises a sticky TSLAM_E_POOL_FULL on the next flush / reader.
  if (m->cfg.max_blocks <= 0) m->cfg.max_blocks = (int)(dense_blocks < 32768 ? 32768 : (dense_blocks > 131072 ? 131072 : dense_blocks));
  if (m->cfg.max_blocks > TS_MAX_BLOCKS) m->cfg.max_blocks = TS_MAX_BLOCKS;
  ts_fill_intrin(m);
  m->clamp_on_commit = true;

  TsGrid& g = m->g;
  g.max_blocks = m->cfg.max_blocks;
  g.N = cfg->N; g.Nz = cfg->Nz; g.hN = cfg->N / 2; g.hNz = cfg->Nz / 2;
  m->table_cap = next_pow2((size_t)g.max_blocks * 2 + 64);
  g.table_mask = (uint32_t)(m->table_cap - 1);
  const size_t nv = (size_t)g.max_blocks * TS_B3;
  TS_CUDA(cudaMalloc(&g.table, m->table_cap * 8));
  TS_CUDA(cudaMemset(g.table, 0xFF, m->table_cap * 8));
  TS_CUDA(cudaMalloc(&g.block_key, (size_t)g.max_blocks * 8));
  TS_CUDA(cudaMalloc(&g.acc, nv * sizeof(float2)));
  TS_CUDA(cudaMalloc(&g.tw, nv * sizeof(float2)));
  TS_CUDA(cudaMalloc(&g.obs, nv));
  TS_CUDA(cudaMalloc(&g.occ, nv));
  TS_CUDA(cudaMemset(g.acc, 0, nv * sizeof(float2)));
  TS_CUDA(cudaMemset(g.tw, 0, nv * sizeof(float2)));
  TS_CUDA(cudaMemset(g.obs, 0, nv));
  TS_CUDA(cudaMemset(g.occ, 0, nv));
  g.esdf = nullptr;
  g.cword = nullptr;
  g.col = nullptr;
  if (m->cfg.texture_enabled) {
    TS_CUDA(cudaMalloc(&g.cword, nv * 8));
    TS_CUDA(cudaMalloc(&g.col, nv * 16));
    TS_CUDA(cudaMemset(g.cword, 0, nv * 8));
    TS_CUDA(cudaMemset(g.col, 0, nv * 16));
  }
  TS_CUDA(cudaMalloc(&g.ghost, (size_t)g.max_blocks));
  TS_CUDA(cudaMemset(g.ghost, 0, (size_t)g.max_blocks));
  TS_CUDA(cudaMalloc(&g.dirty_flag, (size_t)g.max_blocks * 4));
  TS_CUDA(cudaMalloc(&g.dirty_list, (size_t)g.max_blocks * 4));
  TS_CUDA(cudaMemset(g.dirty_flag, 0, (size_t)g.max_blocks * 4));
  TS_CUDA(cudaMalloc(&g.esdf_dirty, (size_t)g.max_blocks * 4));
  TS_CUDA(cudaMemset(g.esdf_dirty, 0, (size_t)g.max_blocks * 4));
  TS_CUDA(cudaMalloc(&m->blk_stamp, (size_t)g.max_blocks * 8));
  TS_CUDA(cudaMemset(m->blk_stamp, 0, (size_t)g.max_blocks * 8));
  TS_CUDA(cudaMalloc(&m->scratch_i, 64 * sizeof(int)));
  TS_CUDA(cudaMemset(m->scratch_i, 0, 64 * sizeof(int)));
  g.n_blocks = m->scratch_i + 0;
  g.n_dirty = m->scratch_i + 1;
  g.err = m->scratch_i + 2;
  m->n_rays = m->scratch_i + 3;

  // integrate workspace
  const int step = m->cfg.recast_step;
  size_t sampled = (size_t)m->cfg.max_image_pixels / ((size_t)step * step) + 1024;
  m->bucket_cap = (uint32_t)next_pow2(sampled + sampled / 2);
  if (const char* bc = getenv("TSLAM_BUCKET_CAP")) { if (atoi(bc) >= 1024) m->bucket_cap = (uint32_t)next_pow2((size_t)atoi(bc)); }  // experiment
  // the point-cloud path treats the TSLAM_MAX_BATCH per-frame tables as ONE table
  if ((size_t)m->cfg.max_points * 3 / 2 > (size_t)TSLAM_MAX_BATCH * m->bucket_cap || (size_t)m->cfg.max_points > BK_MAX_SLOTS || m->bucket_cap > BK_MAX_SLOTS) {
    ts_set_error("max_points=%d too large for the bucket workspace", m->cfg.max_points);
    return TSLAM_E_INVALID;
  }
  TS_CUDA(cudaMalloc(&m->buckets, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * sizeof(TsBucket)));
  if (m->cfg.texture_enabled) TS_CUDA(cudaMalloc(&m->bcol, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * sizeof(uint4)));
  TS_CUDA(cudaMalloc(&m->bidx, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * 8));
  TS_CUDA(cudaMemset(m->bidx, 0, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * 8));
  m->bk_slot_bits = ts_bucket_slot_bits(m->bucket_cap, (uint32_t)m->cfg.max_points);
  if (m->bk_slot_bits >= TS_BK_SLOT_FIELD) TS_CUDA(cudaMalloc(&m->bpos, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * 4));
  m->bk_epoch_max = m->bk_slot_bits >= TS_BK_SLOT_FIELD ? 0u : (1u << (TS_BK_SLOT_FIELD - m->bk_slot_bits)) - 1u;
  m->bk_epoch = 0;
  {  // a launch in which one bucket can collect more points than the packed count word holds keeps its counts in a plane
    const uint64_t n_max = std::max((uint64_t)m->cfg.max_image_pixels / ((uint64_t)step * step), (uint64_t)m->cfg.max_points);
    if (ts_bucket_cnt_shift(n_max, ts_bucket_dmax(m)) < 0) TS_CUDA(cudaMalloc(&m->bcnt, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * 4));
  }
  m->ray_list_cap = (uint32_t)((size_t)TSLAM_MAX_BATCH * sampled);
  if (m->ray_list_cap < (uint32_t)m->cfg.max_points) m->ray_list_cap = (uint32_t)m->cfg.max_points;
  TS_CUDA(cudaMalloc(&m->ray_list, (size_t)m->ray_list_cap * 4));
  TS_CUDA(cudaMalloc(&m->depth_stage, (size_t)2 * TSLAM_MAX_BATCH * m->cfg.max_image_pixels * 2));  // double buffered
  {
    int prio_lo = 0, prio_hi = 0;  // highest priority: the gather kernel's few CTAs go first when SM slots free up
    TS_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    TS_CUDA(cudaStreamCreateWithPriority(&m->copy_stream, cudaStreamNonBlocking, prio_hi));
  }
  {
    // Page-locked frames are COPIED at call time by default (the reference's semantics: recast_depth_to_map has
    // consumed the array when it returns).  Borrowing them instead - the GPU reads the sampled rows straight from
    // host memory a few calls later - is opt-in: tslam_tsdf_set_frame_mode(m, 1) or TSLAM_ZERO_COPY=1.
    const char* zc = getenv("TSLAM_ZERO_COPY");
    m->zero_copy = (zc && zc[0] == '1') ? 1 : 0;
    const char* fc = getenv("TSLAM_FRAME_COPY");  // "dma": pageable frames through cudaMemcpyAsync too (A/B against the ring)
    m->stage_mode = (fc && strcmp(fc, "dma") == 0) ? 0 : 1;
    // page-locked frames in copy mode: awaited cudaMemcpyAsync (default; A/B: "ring" = through the host ring like
    // pageable frames, "fetch" = awaited row fetch).  On one H100 SXM (400 W power limit, one rank,
    // bench.py e2e arms, three runs): dma 32.0-35.5 k, ring 13.4-14.8 k, fetch 25.1-27.6 k frames/s - the copy engine is the
    // one that neither depends on the host's memcpy bandwidth (8 ranks share it) nor on the PCIe read latency
    const char* pc = getenv("TSLAM_PINNED_COPY");
    m->pinned_mode = (pc && strcmp(pc, "ring") == 0) ? 0 : (pc && strcmp(pc, "fetch") == 0) ? 1 : 2;
    m->trace = getenv("TSLAM_TRACE") != nullptr;
    if (m->trace) {
      for (int i = 0; i < 2; i++)
        for (int k = 0; k < 4; k++) TS_CUDA(cudaEventCreate(&m->tr_ev[i][k]));
      TS_CUDA(cudaEventCreate(&m->tr_base));
      TS_CUDA(cudaEventRecord(m->tr_base, 0));
    }
    // frames per queue launch, alternating a, b, a, b, ...: half a batch each by default, so that the kernels of the
    // first half run while the caller is still handing over the second half.  (16,48 and 24,40 were measured too: with
    // page-locked frames the step is bound by the PCIe reads of the row gather, the split hardly matters.)
    m->queue_launch[0] = TSLAM_MAX_BATCH / 2;
    m->queue_launch[1] = TSLAM_MAX_BATCH / 2;
    const char* ql = getenv("TSLAM_QUEUE_LAUNCH");
    if (ql) {
      int a = 0, b = 0;
      const int k = sscanf(ql, "%d,%d", &a, &b);
      if (k == 1) b = a;
      if (k >= 1 && a >= 1 && a <= TSLAM_MAX_BATCH && b >= 1 && b <= TSLAM_MAX_BATCH) { m->queue_launch[0] = a; m->queue_launch[1] = b; }
    }
  }
  for (int i = 0; i < 2; i++) {
    TS_CUDA(cudaEventCreateWithFlags(&m->ev_copied[i], cudaEventDisableTiming));
    TS_CUDA(cudaEventCreateWithFlags(&m->ev_free[i], cudaEventDisableTiming));
  }
  TS_CUDA(cudaMalloc(&m->points_stage, (size_t)m->cfg.max_points * 12));
  if (m->cfg.texture_enabled) {
    TS_CUDA(cudaMalloc(&m->tex_stage, (size_t)2 * TSLAM_MAX_BATCH * m->cfg.max_image_pixels * 3));
    TS_CUDA(cudaMalloc(&m->rgb_stage, (size_t)m->cfg.max_points * 3));
  }
  TS_CUDA(cudaMalloc(&m->counters, sizeof(TsCounters)));
  TS_CUDA(cudaMemset(m->counters, 0, sizeof(TsCounters)));
  TS_CUDA(cudaMalloc(&m->pose_R, (size_t)m->cfg.max_submaps * 9 * 4));
  TS_CUDA(cudaMalloc(&m->pose_T, (size_t)m->cfg.max_submaps * 3 * 4));
  TS_CUDA(cudaMemset(m->pose_R, 0, (size_t)m->cfg.max_submaps * 9 * 4));  // ti fields start at zero
  TS_CUDA(cudaMemset(m->pose_T, 0, (size_t)m->cfg.max_submaps * 3 * 4));
  std::vector<float> cm(1024 * 3);
  fill_jet_host(cm.data());
  TS_CUDA(cudaMalloc(&m->colormap, cm.size() * 4));
  TS_CUDA(cudaMemcpy(m->colormap, cm.data(), cm.size() * 4, cudaMemcpyHostToDevice));
  {
    // ray march: block-binned shared-memory accumulation (tslam_march.cu) for untextured maps; TSLAM_MARCH=legacy
    // keeps the round-1 kernel (one global reduction per sample) for A/B runs.  Textured maps use k_raymarch<true>.
    const char* mm = getenv("TSLAM_MARCH");
    m->march_mode = (m->cfg.texture_enabled || (mm && mm[0] == 'l') || m->cfg.max_ray_length / m->cfg.voxel_scale > 60000.0) ? 0 : 1;
    m->march_verify = getenv("TSLAM_MARCH_VERIFY") != nullptr;
    // (the march workspace - ~2 GB for 640x480 frames - is allocated by the first integrate launch: global maps that are
    // only ever fused into never pay for it)
  }
  TS_CUDA(cudaFuncSetAttribute(k_raymarch<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, RM_SMEM));
  TS_CUDA(cudaFuncSetAttribute(k_raymarch<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, RM_SMEM_TEX));
  TS_CUDA(cudaFuncSetAttribute(k_commit_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, CM_SMEM));
  TS_CUDA(cudaDeviceSynchronize());
  *out = m;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_destroy(tslam_tsdf_t* m) {
  if (!m) return TSLAM_OK;
  cudaDeviceSynchronize();
  TsGrid& g = m->g;
  cudaFree(g.table); cudaFree(g.block_key); cudaFree(g.acc); cudaFree(g.tw); cudaFree(g.obs); cudaFree(g.occ);
  if (g.esdf) cudaFree(g.esdf);
  if (m->esdf_aux) cudaFree(m->esdf_aux);
  if (m->mc_scratch) cudaFree(m->mc_scratch);
  if (m->tile_hist) cudaFree(m->tile_hist);
  if (m->reg_blk) cudaFree(m->reg_blk);
  if (m->reg_pts) cudaFree(m->reg_pts);
  if (g.cword) cudaFree(g.cword);
  if (g.col) cudaFree(g.col);
  if (m->tex_stage) cudaFree(m->tex_stage);
  if (m->rgb_stage) cudaFree(m->rgb_stage);
  cudaFree(g.ghost); cudaFree(g.dirty_flag); cudaFree(g.esdf_dirty); cudaFree(m->blk_stamp); cudaFree(g.dirty_list); cudaFree(m->scratch_i);
  cudaFree(m->buckets); cudaFree(m->bidx); cudaFree(m->ray_list);
  if (m->bcol) cudaFree(m->bcol);
  if (m->bpos) cudaFree(m->bpos);
  if (m->bcnt) cudaFree(m->bcnt);
  cudaFree(m->depth_stage); cudaFree(m->points_stage);
  cudaStreamDestroy(m->copy_stream);
  if (m->h_ring) cudaFreeHost(m->h_ring);
  for (int i = 0; i < 2; i++) { cudaEventDestroy(m->ev_copied[i]); cudaEventDestroy(m->ev_free[i]); }
  if (m->mw.rays) ts_march_free(m);
  cudaFree(m->counters); cudaFree(m->pose_R); cudaFree(m->pose_T); cudaFree(m->colormap);
  if (m->ev) { for (int i = 0; i < TS_PROF_EV * TS_PROF_RING; i++) cudaEventDestroy(m->ev[i]); delete[] m->ev; }
  delete m;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_reset(tslam_tsdf_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  TsGrid& g = m->g;
  int nb = 0;
  m->n_integrate_calls = 0;  // pending sums are discarded with the blocks
  m->esdf_full_needed = 1;   // ... and the ESDF state
  m->mesh_epoch++;           // ... and the incremental mesh (planes cleared and pool slots recycled without stamps)
  m->q_n = 0;                // ... and so are queued frames
  m->q_gathered = 0;
  TS_CUDA(cudaMemcpyAsync(&nb, g.n_blocks, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (nb > g.max_blocks) nb = g.max_blocks;
  const size_t nv = (size_t)nb * TS_B3;
  TS_CUDA(cudaMemsetAsync(g.table, 0xFF, m->table_cap * 8, st));
  if (nv) {
    TS_CUDA(cudaMemsetAsync(g.acc, 0, nv * sizeof(float2), st));
    TS_CUDA(cudaMemsetAsync(g.tw, 0, nv * sizeof(float2), st));
    TS_CUDA(cudaMemsetAsync(g.obs, 0, nv, st));
    TS_CUDA(cudaMemsetAsync(g.occ, 0, nv, st));
    if (g.esdf) TS_CUDA(cudaMemsetAsync(g.esdf, 0, nv * 4, st));
    TS_CUDA(cudaMemsetAsync(g.dirty_flag, 0, (size_t)nb * 4, st));
    TS_CUDA(cudaMemsetAsync(g.ghost, 0, (size_t)nb, st));
    if (g.cword) TS_CUDA(cudaMemsetAsync(g.cword, 0, nv * 8, st));
    if (g.col) TS_CUDA(cudaMemsetAsync(g.col, 0, nv * 16, st));
  }
  TS_CUDA(cudaMemsetAsync(m->scratch_i, 0, 4 * sizeof(int), st));  // n_blocks, n_dirty, err, n_rays
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_set_intrinsics(tslam_tsdf_t* m, double fx, double fy, double cx, double cy) {
  if (!m) return TSLAM_E_INVALID;
  m->cfg.fx = fx; m->cfg.fy = fy; m->cfg.cx = cx; m->cfg.cy = cy;
  ts_fill_intrin(m);
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_set_color_intrinsics(tslam_tsdf_t* m, double fx, double fy, double cx, double cy, int color_same_proj) {
  if (!m) return TSLAM_E_INVALID;
  m->in.fxc = (float)fx; m->in.fyc = (float)fy; m->in.cxc = (float)cx; m->in.cyc = (float)cy;
  m->in.same_proj = color_same_proj ? 1 : 0;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_set_submap_pose(tslam_tsdf_t* m, int32_t s, const float* R9, const float* T3) {
  if (!m || !R9 || !T3 || s < 0 || s >= m->cfg.max_submaps) { ts_set_error("bad submap id %d", s); return TSLAM_E_INVALID; }
  TS_CUDA(cudaMemcpy(m->pose_R + 9 * (size_t)s, R9, 36, cudaMemcpyHostToDevice));
  TS_CUDA(cudaMemcpy(m->pose_T + 3 * (size_t)s, T3, 12, cudaMemcpyHostToDevice));
  return TSLAM_OK;
}

// ---------------------------------------------------------------------------
// host: integrate
// ---------------------------------------------------------------------------
// k_collect_dirty, then the commit, whose last CTA sets the dirty-list count back to zero (ticket: scratch_i[4]).  Both
// are launched with programmatic dependent launch (ts_launch_pdl).
static int ts_launch_commit(tslam_tsdf* m, cudaStream_t st, int clamp, int fused) {
  int grid = m->sm_count * 8;
  const int gc = (m->g.max_blocks + 255) / 256 < m->sm_count * 4 ? (m->g.max_blocks + 255) / 256 : m->sm_count * 4;
  TS_CUDA(ts_launch_pdl(k_collect_dirty, gc, 256, 0, st, m->g));
  TS_LAUNCH_CHECK(m);
  static const bool plain_env = getenv("TSLAM_COMMIT_PLAIN") != nullptr;  // A/B switch for the non-TMA variant
  const bool plain = plain_env || m->g.col != nullptr;  // textured maps: the per-thread variant also folds the colours
  const unsigned long long seq = ++m->commit_seq;        // stamp of every block this commit writes (incremental mesh)
  int* ticket = m->scratch_i + 4;
  if (plain) TS_CUDA(ts_launch_pdl(k_commit, grid, 256, 0, st, m->g, clamp, fused, m->blk_stamp, seq, ticket));
  else TS_CUDA(ts_launch_pdl(k_commit_tma, m->sm_count * 3, 256, CM_SMEM, st, m->g, clamp, fused, m->blk_stamp, seq, ticket));
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

static int ts_launch_queue(tslam_tsdf* m, cudaStream_t st);
int ts_flush_pending(tslam_tsdf* m, cudaStream_t st) {
  if (m->q_n > 0) {  // frames queued by the per-frame API
    int rc = ts_launch_queue(m, st);
    if (rc) return rc;
  }
  if (m->n_integrate_calls > 0) {  // something may be pending
    int rc = ts_launch_commit(m, st, m->clamp_on_commit ? 1 : 0, 0);
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

static void ts_fill_frame(tslam_tsdf* m, TsFrame& fr, const float* R9, const float* T3, int submap) {
  memcpy(fr.R, R9, 36);
  memcpy(fr.T, T3, 12);
  fr.submap = submap;
  m->frame_seq++;  // 1, 2, ... (texture: later frames win); < 2^22 - TSLAM_MAX_BATCH (ts_seq_renorm runs before that)
  fr.seq = m->frame_seq;
}

static int ts_integrate_depth_impl(tslam_tsdf_t* m, const uint16_t* depth, int mem, int32_t n_frames, int32_t h, int32_t w,
                                   const float* R9s, const float* T3s, const int32_t* submap_ids, int flags, void* stream, int rows_compacted,
                                   const uint8_t* tex = nullptr, int th = 0, int tw = 0);
extern "C" int tslam_tsdf_integrate_depth(tslam_tsdf_t* m, const uint16_t* depth, int mem, int32_t n_frames, int32_t h, int32_t w,
                                          const float* R9s, const float* T3s, const int32_t* submap_ids, int flags, void* stream) {
  if (m && m->q_n > 0) { int rcq = ts_launch_queue(m, (cudaStream_t)stream); if (rcq) return rcq; }  // frames queued earlier are integrated first
  return ts_integrate_depth_impl(m, depth, mem, n_frames, h, w, R9s, T3s, submap_ids, flags, stream, 0);
}
static int ts_check_tex(tslam_tsdf* m, const uint8_t* tex, int th, int tw) {
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
  return ts_integrate_depth_impl(m, depth, mem, n_frames, h, w, R9s, T3s, submap_ids, flags, stream, 0, tex, th, tw);
}
// rows_compacted: the frames hold only the sampled rows (hh = h/step rows of w pixels each) - the per-frame queue
// stages them that way with a strided 2-D copy, halving the host->device bytes for recast_step 2.
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

static int ts_integrate_depth_impl(tslam_tsdf_t* m, const uint16_t* depth, int mem, int32_t n_frames, int32_t h, int32_t w,
                                   const float* R9s, const float* T3s, const int32_t* submap_ids, int flags, void* stream, int rows_compacted,
                                   const uint8_t* tex, int th, int tw) {
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
    const int rows_stored = rows_compacted ? hh : h;
    const uint16_t* src = depth + (size_t)base * rows_stored * w;
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
    cudaEvent_t* pe = m->profiling ? m->ev + TS_PROF_EV * (m->prof_launches % TS_PROF_RING) : nullptr;
    if (pe) TS_CUDA(cudaEventRecord(pe[0], st));
    const int agg_ok = m->cfg.max_ray_length < 30.0 ? 1 : 0;  // 32-lane int32 sums: |p| <= max_ray * sqrt(1 + tan^2) < 64 m even at 60 deg half-FOV
    dim3 grid1((ww + 31) / 32, (hh + 7) / 8, nf);
    if ((size_t)grid1.x * grid1.y * 256 > m->bucket_cap) {  // every 8x4-pixel warp tile owns 32 bucket records of its frame
      ts_set_error("frame %dx%d (sampled %dx%d) has too many partial pixel tiles for max_image_pixels=%d", h, w, hh, ww, m->cfg.max_image_pixels);
      return TSLAM_E_INVALID;
    }
    TsBucketLaunch bl;
    { int rcb = ts_bucket_launch(m, st, (uint64_t)hh * ww, bl); if (rcb) return rcb; }
    k_bucket_depth<<<grid1, 256, 0, st>>>(src, rows_stored * w, rows_compacted ? 1 : step, w, hh, ww, batch, m->in, agg_ok, m->buckets, m->bcol,
                                          m->bidx, m->bucket_cap, bl, m->ray_list, m->n_rays, m->ray_list_cap, m->counters, m->g.err, tsrc, th, tw);
    TS_LAUNCH_CHECK(m);
    if (pe) TS_CUDA(cudaEventRecord(pe[1], st));
    if (!m->g.cword && m->march_mode) {
      int rcs = ts_march_setup(m, st, batch, bshift);
      if (rcs) return ts_bucket_abandon(m, st, rcs);
      int rcm = ts_march_launch(m, st, batch, bshift, bl, pe ? pe + 4 : nullptr);  // clears n_rays itself
      if (rcm) return ts_bucket_abandon(m, st, rcm);
      if (pe) TS_CUDA(cudaEventRecord(pe[2], st));
    } else {
      if (m->g.cword) {
        k_raymarch<true><<<m->sm_count, RM_THREADS, RM_SMEM_TEX, st>>>(batch, m->in, m->g, m->buckets, m->bcol, m->bidx, bshift, bl, m->ray_list,
                                                                       m->n_rays, m->ray_list_cap, m->counters);
      } else {
        k_raymarch<false><<<(m->sm_count - m->rm_reserve) * 2, RM_THREADS, RM_SMEM, st>>>(batch, m->in, m->g, m->buckets, m->bcol, m->bidx, bshift,
                                                                                       bl, m->ray_list, m->n_rays, m->ray_list_cap, m->counters);
      }
      TS_LAUNCH_CHECK(m);
      if (pe) TS_CUDA(cudaEventRecord(pe[2], st));
      k_reset_counters<<<1, 1, 0, st>>>(m->n_rays, nullptr);
      TS_LAUNCH_CHECK(m);
    }
    m->n_integrate_calls++;
    if (flags & TSLAM_F_COMMIT) {
      int rc = ts_flush_pending(m, st);
      if (rc) return rc;
    }
    if (stage0) {  // the queue must not refill buffer 0 before these kernels have read it
      TS_CUDA(cudaEventRecord(m->ev_free[0], st));
      m->ev_free_valid[0] = true;
    }
    if (pe) { TS_CUDA(cudaEventRecord(pe[3], st)); m->prof_launches++; }
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
  const uint32_t rec_cap = ((uint32_t)n + 31u) & ~31u;  // a warp's slots start at its first point
  cudaEvent_t* pe = m->profiling ? m->ev + TS_PROF_EV * (m->prof_launches % TS_PROF_RING) : nullptr;
    if (pe) TS_CUDA(cudaEventRecord(pe[0], st));
  const int agg_ok = m->cfg.max_ray_length < 30.0 ? 1 : 0;  // 32-lane int32 sums: |p| <= max_ray * sqrt(1 + tan^2) < 64 m even at 60 deg half-FOV
  TsBucketLaunch bl;
  { int rcb = ts_bucket_launch(m, st, (uint64_t)n, bl); if (rcb) return rcb; }
  k_bucket_points<<<(n + 255) / 256, 256, 0, st>>>(src, n, batch, m->in, agg_ok, m->buckets, m->bcol, m->bidx, cap_total, rec_cap, bl, m->ray_list,
                                                    m->n_rays, m->ray_list_cap, m->counters, m->g.err, csrc);
  TS_LAUNCH_CHECK(m);
  if (pe) TS_CUDA(cudaEventRecord(pe[1], st));
  if (!m->g.cword && m->march_mode) {
    int rcm = ts_march_setup(m, st, batch, bshift);
    if (rcm) return ts_bucket_abandon(m, st, rcm);
    rcm = ts_march_launch(m, st, batch, bshift, bl, pe ? pe + 4 : nullptr);  // clears n_rays itself
    if (rcm) return ts_bucket_abandon(m, st, rcm);
    if (pe) TS_CUDA(cudaEventRecord(pe[2], st));
  } else {
    if (m->g.cword)
      k_raymarch<true><<<m->sm_count, RM_THREADS, RM_SMEM_TEX, st>>>(batch, m->in, m->g, m->buckets, m->bcol, m->bidx, bshift, bl, m->ray_list,
                                                                     m->n_rays, m->ray_list_cap, m->counters);
    else
      k_raymarch<false><<<m->sm_count * 2, RM_THREADS, RM_SMEM, st>>>(batch, m->in, m->g, m->buckets, m->bcol, m->bidx, bshift, bl, m->ray_list,
                                                                      m->n_rays, m->ray_list_cap, m->counters);
    TS_LAUNCH_CHECK(m);
    if (pe) TS_CUDA(cudaEventRecord(pe[2], st));
    k_reset_counters<<<1, 1, 0, st>>>(m->n_rays, nullptr);
    TS_LAUNCH_CHECK(m);
  }
  m->n_integrate_calls++;
  if (flags & TSLAM_F_COMMIT) {
    int rc = ts_flush_pending(m, st);
    if (rc) return rc;
  }
  if (pe) { TS_CUDA(cudaEventRecord(pe[3], st)); m->prof_launches++; }
  return TSLAM_OK;
}

// ---------------------------------------------------------------------------
// per-frame queue: the reference API hands over ONE frame per call (recast_depth_to_map, dense_tsdf.py:162-165).
// tslam_tsdf_queue_depth copies the frame to a device staging slot on a copy stream (overlapping the kernels of
// the previous batch) and records its pose; a full queue (TSLAM_MAX_BATCH frames) or tslam_tsdf_flush launches
// the batch: bucket -> ray march -> commit.
// ---------------------------------------------------------------------------
// Pinned (page-locked) host frames: instead of a DMA copy of the whole 614 KB frame, a small kernel reads ONLY THE
// SAMPLED ROWS (every recast_step-th row, :192) straight from host memory over PCIe - 16-byte loads, a warp covers
// 512 contiguous bytes - and drops them at their place in the device staging frame.  Half the PCIe bytes for
// recast_step 2, one launch per TS_GATHER_GROUP frames instead of one copy call per frame.
#define TS_GATHER_GROUP 8
struct TsGatherArgs {
  const uint4* src[TS_GATHER_GROUP];
  uint4* dst[TS_GATHER_GROUP];
  int sstride[TS_GATHER_GROUP];  // source row stride (16-byte units): recast_step rows for a caller's frame, 1 row for the ring
};
__global__ void __launch_bounds__(256) k_gather_rows(const __grid_constant__ TsGatherArgs ga, int hh, int row_u4, int row_stride_u4) {
  const uint4* __restrict__ src = ga.src[blockIdx.y];
  uint4* __restrict__ dst = ga.dst[blockIdx.y];
  const int sstride = ga.sstride[blockIdx.y];
  const int total = hh * row_u4;
  const int base = (blockIdx.x * 256 + threadIdx.x) * 4;
  uint4 v[4];
  int off[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {  // 4 independent 16-byte PCIe reads in flight per thread
    const int i = base + k;
    off[k] = -1;
    if (i < total) {
      const int jj = i / row_u4, c = i - jj * row_u4;
      off[k] = jj * row_stride_u4 + c;
      v[k] = __ldcs(src + (jj * sstride + c));
    }
  }
#pragma unroll
  for (int k = 0; k < 4; k++)
    if (off[k] >= 0) dst[off[k]] = v[k];
}

// hand the queued zero-copy frames [q_gathered, q_n) to gather launches on the copy stream
static int ts_gather_pending(tslam_tsdf* m) {
  const int b = m->q_buf;
  const int step = m->cfg.recast_step;
  const int hh = (int)((double)m->q_h / step), row_u4 = m->q_w / 8;
  while (m->q_gathered < m->q_n) {
    TsGatherArgs ga;
    int k = 0;
    while (m->q_gathered < m->q_n && k < TS_GATHER_GROUP) {
      const int q = m->q_gathered++;
      if (!m->q_hptr[q]) continue;
      ga.src[k] = (const uint4*)m->q_hptr[q];
      ga.sstride[k] = m->q_sstride[q];
      ga.dst[k] = (uint4*)(m->depth_stage + (size_t)b * TSLAM_MAX_BATCH * m->cfg.max_image_pixels + (size_t)q * m->q_h * m->q_w);
      k++;
    }
    if (k == 0 || hh <= 0) continue;
    dim3 grid((hh * row_u4 + 1023) / 1024, k);
    k_gather_rows<<<grid, 256, 0, m->copy_stream>>>(ga, hh, row_u4, step * row_u4);
    TS_LAUNCH_CHECK(m);
  }
  return TSLAM_OK;
}

static int ts_launch_queue(tslam_tsdf* m, cudaStream_t st) {
  if (m->q_open) {  // a hand-over that was begun and never ended (the caller failed in between): the frame is dropped
    m->q_open = 0;
    if (m->q_await) { m->q_await = 0; TS_CUDA(cudaStreamSynchronize(m->copy_stream)); }
  }
  m->q_phase = 0;  // any launch that is not the queue's own threshold (flush, reader, geometry change) restarts the pattern
  const int n = m->q_n;
  if (n == 0) return TSLAM_OK;
  const int b = m->q_buf;
  {
    int rcg = ts_gather_pending(m);
    if (rcg) return rcg;
  }
  m->q_gathered = 0;
  if (m->trace) TS_CUDA(cudaEventRecord(m->tr_ev[b][1], m->copy_stream));
  TS_CUDA(cudaEventRecord(m->ev_copied[b], m->copy_stream));
  TS_CUDA(cudaStreamWaitEvent(st, m->ev_copied[b], 0));
  if (m->trace) TS_CUDA(cudaEventRecord(m->tr_ev[b][2], st));
  const uint16_t* src = m->depth_stage + (size_t)b * TSLAM_MAX_BATCH * m->cfg.max_image_pixels;
  m->q_n = 0;  // (integrate may recurse into flush through readers; the queue is empty from here on)
  m->q_buf = b ^ 1;
  const uint8_t* tsrc = m->q_has_tex ? m->tex_stage + (size_t)b * TSLAM_MAX_BATCH * m->cfg.max_image_pixels * 3 : nullptr;
  int rc = ts_integrate_depth_impl(m, src, TSLAM_MEM_DEVICE, n, m->q_h, m->q_w, m->q_R, m->q_T, m->q_s, TSLAM_F_COMMIT, (void*)st, 0,
                                   tsrc, m->q_th, m->q_tw);
  if (rc) return rc;
  TS_CUDA(cudaEventRecord(m->ev_free[b], st));
  m->ev_free_valid[b] = true;
  if (m->trace) { TS_CUDA(cudaEventRecord(m->tr_ev[b][3], st)); m->tr_have[b] = n; }
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_set_queue_launch(tslam_tsdf_t* m, int32_t frames_a, int32_t frames_b) {
  if (!m || frames_a < 1 || frames_a > TSLAM_MAX_BATCH || frames_b < 1 || frames_b > TSLAM_MAX_BATCH) { ts_set_error("queue launch sizes must be in [1, %d]", TSLAM_MAX_BATCH); return TSLAM_E_INVALID; }
  if (m->q_n > 0) { ts_set_error("frames are queued: flush before changing the launch size"); return TSLAM_E_INVALID; }
  m->queue_launch[0] = frames_a;
  m->queue_launch[1] = frames_b;
  m->q_phase = 0;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_set_frame_mode(tslam_tsdf_t* m, int borrow_pinned) {
  if (!m) return TSLAM_E_INVALID;
  if (m->q_n > 0) { ts_set_error("frames are queued: flush before changing the frame mode"); return TSLAM_E_INVALID; }
  m->zero_copy = borrow_pinned ? 1 : 0;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_flush(tslam_tsdf_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  m->q_phase = 0;
  int rc = ts_launch_queue(m, (cudaStream_t)stream);
  if (rc) return rc;
  return ts_check_deferred_async(m, (cudaStream_t)stream);
}

extern "C" int tslam_tsdf_queue_depth(tslam_tsdf_t* m, const uint16_t* depth_host, int32_t h, int32_t w, const float* R9,
                                      const float* T3, int32_t submap, void* stream) {
  return tslam_tsdf_queue_depth_tex(m, depth_host, nullptr, h, w, 0, 0, R9, T3, submap, stream);
}
#if defined(__SSE2__) || defined(__x86_64__)
#include <emmintrin.h>
static inline void ts_stream_copy_row(uint16_t* dst, const uint16_t* src, size_t bytes) {  // dst 16-byte aligned, bytes % 16 == 0
  __m128i* d = reinterpret_cast<__m128i*>(dst);
  const __m128i* s = reinterpret_cast<const __m128i*>(src);
  const size_t n = bytes / 16;
  size_t i = 0;
  for (; i + 4 <= n; i += 4) {
    const __m128i a = _mm_loadu_si128(s + i), b = _mm_loadu_si128(s + i + 1), c = _mm_loadu_si128(s + i + 2), e = _mm_loadu_si128(s + i + 3);
    _mm_stream_si128(d + i, a); _mm_stream_si128(d + i + 1, b); _mm_stream_si128(d + i + 2, c); _mm_stream_si128(d + i + 3, e);
  }
  for (; i < n; i++) _mm_stream_si128(d + i, _mm_loadu_si128(s + i));
}
static inline void ts_stream_fence() { _mm_sfence(); }
#else
static inline void ts_stream_copy_row(uint16_t* dst, const uint16_t* src, size_t bytes) { memcpy(dst, src, bytes); }
static inline void ts_stream_fence() {}
#endif

// first half of a per-frame hand-over: the frame's copy is STARTED (page-locked source: DMA on the copy stream;
// pageable source: sampled rows into the ring; borrowed: nothing).  ts_queue_end awaits it and records the pose.
static int ts_queue_begin(tslam_tsdf* m, const uint16_t* depth_host, const uint8_t* tex_host, int32_t h, int32_t w, int32_t th, int32_t tw,
                          void* stream) {
  if (m) { int rc0 = ts_check_tex(m, tex_host, th, tw); if (rc0) return rc0; }
  if (!m || !depth_host || h <= 0 || w <= 0) { ts_set_error("bad argument"); return TSLAM_E_INVALID; }
  if ((long long)h * w > m->cfg.max_image_pixels) { ts_set_error("frame %dx%d exceeds max_image_pixels=%d", h, w, m->cfg.max_image_pixels); return TSLAM_E_INVALID; }
  m->q_open = 0;
  m->q_await = 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int has_tex = tex_host != nullptr;
  if (!has_tex) { th = 0; tw = 0; }
  // one batch = one frame geometry and either all or no frames textured
  if (m->q_n > 0 && (m->q_h != h || m->q_w != w || m->q_has_tex != has_tex || m->q_th != th || m->q_tw != tw)) {
    int rc = ts_launch_queue(m, st);
    if (rc) return rc;
  }
  const int b = m->q_buf, q = m->q_n;
  if (q == 0) {
    m->q_h = h; m->q_w = w;
    m->q_has_tex = has_tex; m->q_th = th; m->q_tw = tw;
    // the kernels that read this staging buffer (two batches ago) must be done.  Waiting on the HOST bounds how far
    // the caller can run ahead of the GPU: a pinned frame is consumed before 2*TSLAM_MAX_BATCH further frames are queued.
    if (m->ev_free_valid[b]) TS_CUDA(cudaEventSynchronize(m->ev_free[b]));
    m->q_gathered = 0;
    if (m->trace) {
      if (m->tr_have[b]) {  // timeline of the launch that used this buffer last (ms since handle creation)
        float t[4];
        for (int k = 0; k < 4; k++) cudaEventElapsedTime(&t[k], m->tr_base, m->tr_ev[b][k]);
        fprintf(stderr, "[tslam trace] buf %d frames %d: copy %.3f..%.3f  kernels %.3f..%.3f ms\n", b, m->tr_have[b], t[0], t[1], t[2], t[3]);
      }
      TS_CUDA(cudaEventRecord(m->tr_ev[b][0], m->copy_stream));
    }
  }
  // One linear copy of the whole frame.  (A strided 2-D copy of only the sampled rows halves the bytes but was
  // slower from pinned memory end to end - 240 row descriptors of 1280 B.)
  uint16_t* dst = m->depth_stage + (size_t)b * TSLAM_MAX_BATCH * m->cfg.max_image_pixels + (size_t)q * h * w;  // frames packed h*w apart
  m->q_hptr[q] = nullptr;
  const int step_q = m->cfg.recast_step;
  cudaPointerAttributes at;
  const bool src_pinned = cudaPointerGetAttributes(&at, depth_host) == cudaSuccess && at.type == cudaMemoryTypeHost;
  if (!src_pinned) cudaGetLastError();
  if (m->zero_copy && src_pinned && at.devicePointer && step_q >= 2 && (w % 8) == 0 && ((uintptr_t)depth_host % 16) == 0 && ((size_t)h * w % 8) == 0) {
    m->q_hptr[q] = (const uint16_t*)at.devicePointer;  // borrowed: the GPU reads the caller's frame itself, later
    m->q_sstride[q] = step_q * (w / 8);
  }
  if (!m->q_hptr[q] && (src_pinned ? m->pinned_mode == 0 : m->stage_mode != 0) && (w % 8) == 0) {
    // PAGEABLE source (what np.frombuffer(msg.data) gives the ROS node): the runtime would stage the whole frame through
    // its own bounce buffer inside cudaMemcpyAsync.  Instead the sampled rows (every
    // recast_step-th, :192 - half the bytes for step 2) are copied into the library's page-locked ring with streaming
    // stores - the caller's buffer is free when the call returns - and the GPU fetches them from there over PCIe while
    // the caller hands over the next frames.
    const int hh = (int)((double)h / step_q);
    if (!m->h_ring) {
      m->ring_frame_cap = ((size_t)m->cfg.max_image_pixels / (size_t)step_q + 8) & ~(size_t)7;
      TS_CUDA(cudaHostAlloc((void**)&m->h_ring, (size_t)2 * TSLAM_MAX_BATCH * m->ring_frame_cap * 2, cudaHostAllocMapped));
      TS_CUDA(cudaHostGetDevicePointer((void**)&m->h_ring_dev, m->h_ring, 0));
    }
    if ((size_t)hh * w <= m->ring_frame_cap) {
      const size_t slot = ((size_t)b * TSLAM_MAX_BATCH + (size_t)q) * m->ring_frame_cap;
      uint16_t* hdst = m->h_ring + slot;
      // streaming stores: the ring is read by the GPU over PCIe, never by this CPU - no read-for-ownership of the
      // destination lines, no cache pollution
      // (software prefetch of the rows ahead and 32-byte AVX2 stores were measured on the host: no gain / 2x slower)
      for (int j = 0; j < hh; j++) ts_stream_copy_row(hdst + (size_t)j * w, depth_host + (size_t)j * step_q * w, (size_t)w * 2);
      ts_stream_fence();
      m->q_hptr[q] = m->h_ring_dev + slot;
      m->q_sstride[q] = w / 8;
    }
  }
  if (m->q_hptr[q] && m->sm_count > 8) {
    // the persistent march kernels own every register of the SMs they run on: keep two SMs out of their grids so
    // that the row gather of the NEXT launch's frames can run (and keep PCIe busy) while they march
    m->rm_reserve = 2;
  }
  if (!m->q_hptr[q] && src_pinned && m->pinned_mode == 1 && at.devicePointer && step_q >= 2 && (w % 8) == 0 && ((uintptr_t)depth_host % 16) == 0 &&
      ((size_t)h * w % 8) == 0) {
    // page-locked source, copy mode: the SAMPLED ROWS are fetched right now by a small kernel (half the PCIe bytes of a
    // DMA copy of the frame for recast_step 2) and the fetch is awaited in ts_queue_end
    TsGatherArgs ga;
    ga.src[0] = (const uint4*)at.devicePointer;
    ga.dst[0] = (uint4*)dst;
    ga.sstride[0] = step_q * (w / 8);
    const int hh = (int)((double)h / step_q), row_u4 = w / 8;
    if (hh > 0) {
      dim3 grid((hh * row_u4 + 1023) / 1024, 1);
      k_gather_rows<<<grid, 256, 0, m->copy_stream>>>(ga, hh, row_u4, step_q * row_u4);
      TS_LAUNCH_CHECK(m);
    }
    m->q_await = 1;
    if (m->sm_count > 8) m->rm_reserve = 2;
  } else if (!m->q_hptr[q]) {
    TS_CUDA(cudaMemcpyAsync(dst, depth_host, (size_t)h * w * 2, cudaMemcpyHostToDevice, m->copy_stream));
    // a pageable source has been staged when the call returns; a page-locked one is read by the DMA engine later,
    // so the copy is awaited: the caller may reuse its buffer (camera drivers do)
    if (src_pinned) m->q_await = 1;
  }
  if (has_tex) {
    uint8_t* tdst = m->tex_stage + ((size_t)b * TSLAM_MAX_BATCH * m->cfg.max_image_pixels + (size_t)q * th * tw) * 3;
    TS_CUDA(cudaMemcpyAsync(tdst, tex_host, (size_t)th * tw * 3, cudaMemcpyHostToDevice, m->copy_stream));
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, tex_host) == cudaSuccess && at.type == cudaMemoryTypeHost) m->q_await = 1;
    else cudaGetLastError();
  }
  m->q_open = 1;
  return TSLAM_OK;
}

// second half: the copy started by ts_queue_begin is awaited (the caller's buffers are free when this returns), the pose
// recorded, the queue launched when it is full
static int ts_queue_end(tslam_tsdf* m, const float* R9, const float* T3, int32_t submap, void* stream) {
  if (!m || !R9 || !T3) { ts_set_error("bad argument"); return TSLAM_E_INVALID; }
  if (!m->q_open) { ts_set_error("tslam_tsdf_queue_depth_end without a successful tslam_tsdf_queue_depth_begin"); return TSLAM_E_INVALID; }
  m->q_open = 0;
  if (m->q_await) { m->q_await = 0; TS_CUDA(cudaStreamSynchronize(m->copy_stream)); }
  if (submap < 0 || submap >= m->cfg.max_submaps) { ts_set_error("bad submap id %d", submap); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const int q = m->q_n;
  memcpy(m->q_R + 9 * q, R9, 36);
  memcpy(m->q_T + 3 * q, T3, 12);
  m->q_s[q] = submap;
  m->q_n = q + 1;
  if (m->q_n >= m->queue_launch[m->q_phase]) {
    const int ph = m->q_phase;
    int rc = ts_launch_queue(m, st);
    m->q_phase = ph ^ 1;
    return rc;
  }
  if (m->q_n - m->q_gathered >= TS_GATHER_GROUP) return ts_gather_pending(m);
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_queue_depth_tex(tslam_tsdf_t* m, const uint16_t* depth_host, const uint8_t* tex_host, int32_t h, int32_t w,
                                          int32_t th, int32_t tw, const float* R9, const float* T3, int32_t submap, void* stream) {
  if (!R9 || !T3) { ts_set_error("bad argument"); return TSLAM_E_INVALID; }
  if (m && (submap < 0 || submap >= m->cfg.max_submaps)) { ts_set_error("bad submap id %d", submap); return TSLAM_E_INVALID; }
  int rc = ts_queue_begin(m, depth_host, tex_host, h, w, th, tw, stream);
  if (rc) return rc;
  return ts_queue_end(m, R9, T3, submap, stream);
}
extern "C" int tslam_tsdf_queue_depth_begin(tslam_tsdf_t* m, const uint16_t* depth_host, int32_t h, int32_t w, void* stream) {
  return ts_queue_begin(m, depth_host, nullptr, h, w, 0, 0, stream);
}
extern "C" int tslam_tsdf_queue_depth_end(tslam_tsdf_t* m, const float* R9, const float* T3, int32_t submap, void* stream) {
  return ts_queue_end(m, R9, T3, submap, stream);
}

// ---------------------------------------------------------------------------
// count / gather / scatter  (dense_tsdf.py:412-454)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_count_active(TsGrid g, int submap, unsigned long long* out) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  unsigned int c = 0;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap || g.ghost[b]) continue;
    const uint8_t* obs = g.obs + (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) c += obs[v] > 0;
  }
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

__global__ void __launch_bounds__(256) k_gather(TsGrid g, int submap, long long cap, int32_t* idx, float* tsdf, float* wts,
                                                 int8_t* occ, float* color, unsigned long long* counter) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap || g.ghost[b]) continue;
    const size_t base = (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const bool want = g.obs[base + v] > 0;
      const long long row = warp_append_u64(want, counter);
      if (want && row < cap) {
        idx[3 * row] = bx * TS_B + (v >> 8);
        idx[3 * row + 1] = by * TS_B + ((v >> 4) & 15);
        idx[3 * row + 2] = bz * TS_B + (v & 15);
        const float2 t = g.tw[base + v];
        tsdf[row] = t.x;
        wts[row] = t.y;
        occ[row] = g.occ[base + v];
        if (color) {  // :437-440
          const float4 c = g.col ? g.col[base + v] : make_float4(0.f, 0.f, 0.f, 0.f);
          color[3 * row] = c.x; color[3 * row + 1] = c.y; color[3 * row + 2] = c.z;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_scatter(TsGrid g, int submap, long long n, const int32_t* idx, const float* tsdf,
                                                  const float* wts, const int8_t* occ, const float* color) {
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    const int i = idx[3 * r], j = idx[3 * r + 1], k = idx[3 * r + 2];
    if (!ts_in_bounds(g, i, j, k)) continue;
    const int blk = ts_get_or_alloc(g, ts_pack_key(submap, i >> TS_BSHIFT, j >> TS_BSHIFT, k >> TS_BSHIFT));
    if (blk < 0) continue;
    const size_t o = (size_t)blk * TS_B3 + ts_voxel_off(i, j, k);
    g.tw[o] = make_float2(tsdf[r], wts[r]);  // :447-448
    g.occ[o] = occ[r];                        // :449
    g.obs[o] = 1;                             // :454
    if (color && g.col) g.col[o] = make_float4(color[3 * r], color[3 * r + 1], color[3 * r + 2], 0.0f);  // :450-453
  }
}

extern "C" int tslam_tsdf_count_active(tslam_tsdf_t* m, int32_t submap, int64_t* n_out) {
  if (!m || !n_out) return TSLAM_E_INVALID;
  cudaStream_t st = 0;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  unsigned long long* ctr = (unsigned long long*)(m->scratch_i + 8);
  TS_CUDA(cudaMemsetAsync(ctr, 0, 8, st));
  k_count_active<<<m->sm_count * 4, 256, 0, st>>>(m->g, submap, ctr);
  TS_LAUNCH_CHECK(m);
  unsigned long long v = 0;
  TS_CUDA(cudaMemcpy(&v, ctr, 8, cudaMemcpyDeviceToHost));
  *n_out = (int64_t)v;
  return ts_check_deferred(m);
}

extern "C" int tslam_tsdf_gather(tslam_tsdf_t* m, int32_t submap, int64_t cap, int32_t* idx, float* tsdf, float* w, int8_t* occ,
                                 int64_t* n_out, void* stream) {
  return tslam_tsdf_gather2(m, submap, cap, idx, tsdf, w, occ, nullptr, n_out, stream);
}
extern "C" int tslam_tsdf_gather2(tslam_tsdf_t* m, int32_t submap, int64_t cap, int32_t* idx, float* tsdf, float* w, int8_t* occ,
                                  float* color, int64_t* n_out, void* stream) {
  if (!m || !n_out) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  unsigned long long* ctr = (unsigned long long*)(m->scratch_i + 8);
  TS_CUDA(cudaMemsetAsync(ctr, 0, 8, st));
  k_gather<<<m->sm_count * 4, 256, 0, st>>>(m->g, submap, cap, idx, tsdf, w, occ, color, ctr);
  TS_LAUNCH_CHECK(m);
  unsigned long long v = 0;
  TS_CUDA(cudaMemcpyAsync(&v, ctr, 8, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  *n_out = (int64_t)v;
  rc = ts_check_deferred(m);
  if (rc) return rc;
  if ((int64_t)v > cap) { ts_set_error("gather: %lld observed voxels > capacity %lld", (long long)v, (long long)cap); return TSLAM_E_CAPACITY; }
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_scatter(tslam_tsdf_t* m, int32_t submap, int64_t n, const int32_t* idx, const float* tsdf, const float* w,
                                  const int8_t* occ, void* stream) {
  return tslam_tsdf_scatter2(m, submap, n, idx, tsdf, w, occ, nullptr, stream);
}
extern "C" int tslam_tsdf_scatter2(tslam_tsdf_t* m, int32_t submap, int64_t n, const int32_t* idx, const float* tsdf, const float* w,
                                   const int8_t* occ, const float* color, void* stream) {
  if (!m || n < 0 || submap < 0 || submap >= m->cfg.max_submaps) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  int grid = (int)((n + 255) / 256);
  if (grid > m->sm_count * 32) grid = m->sm_count * 32;
  m->esdf_full_needed = 1;  // bulk load: values change without a commit
  m->mesh_epoch++;          // (same for the incremental mesh)
  k_scatter<<<grid, 256, 0, st>>>(m->g, submap, n, idx, tsdf, w, occ, color);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

// ---------------------------------------------------------------------------
// exporters  (dense_tsdf.py:339-385)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_extract_surface(TsGrid g, int submap, int global_map, const float* pR, const float* pT,
                                                          float vs, float thres, float fl, float ce, const float* cmap,
                                                          long long cap, float* xyz, float* rgb, int* counter) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap || g.ghost[b]) continue;  // :348
    const size_t base = (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      bool want = false;
      float x = 0, y = 0, z = 0;
      if (g.obs[base + v] == 1) {                      // :349
        const float t = g.tw[base + v].x;
        if (fabsf(t) < thres) {                        // :350
          voxel_xyz(g, global_map, pR, pT, s, bx * TS_B + (v >> 8), by * TS_B + ((v >> 4) & 15), bz * TS_B + (v & 15), vs, x, y, z);
          want = !(z > ce || z < fl);                  // :356
        }
      }
      const int row = warp_append_i32(want, counter);  // :358
      if (want && row < cap) {                         // :359 (saturating, see DESIGN.md)
        xyz[3 * (size_t)row] = x; xyz[3 * (size_t)row + 1] = y; xyz[3 * (size_t)row + 2] = z;
        if (rgb && g.col) {  // enable_texture: the voxel's own colour (:360-362)
          const float4 c = g.col[base + v];
          rgb[3 * (size_t)row] = c.x; rgb[3 * (size_t)row + 1] = c.y; rgb[3 * (size_t)row + 2] = c.z;
        } else if (rgb) {
          const int ci = (int)fmaxf(fminf(((z - fl) / (ce - fl)) * 1023.0f, 1023.0f), 0.0f);  // mapping_common.py:216-219
          rgb[3 * (size_t)row] = cmap[3 * ci]; rgb[3 * (size_t)row + 1] = cmap[3 * ci + 1]; rgb[3 * (size_t)row + 2] = cmap[3 * ci + 2];
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_extract_slice(TsGrid g, int submap, int global_map, const float* pR, const float* pT,
                                                        float vs, int index, float dz, const float* cmap, long long cap,
                                                        float* xyz, float* val, float* rgb, int* counter) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap || g.ghost[b]) continue;  // :375
    const size_t base = (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const int k = bz * TS_B + (v & 15);
      const bool want = g.obs[base + v] > 0 && ((float)index - dz < (float)k) && ((float)k < (float)index + dz);  // :376-377
      const int row = warp_append_i32(want, counter);
      if (want && row < cap) {
        float x, y, z;
        voxel_xyz(g, global_map, pR, pT, s, bx * TS_B + (v >> 8), by * TS_B + ((v >> 4) & 15), k, vs, x, y, z);
        const float t = g.tw[base + v].x;
        xyz[3 * (size_t)row] = x; xyz[3 * (size_t)row + 1] = y; xyz[3 * (size_t)row + 2] = z;
        if (val) val[row] = t;  // :380
        if (rgb) {
          const int ci = (int)fmaxf(fminf(((t - (-0.5f)) / (0.5f - (-0.5f))) * 1023.0f, 1023.0f), 0.0f);  // :385
          rgb[3 * (size_t)row] = cmap[3 * ci]; rgb[3 * (size_t)row + 1] = cmap[3 * ci + 1]; rgb[3 * (size_t)row + 2] = cmap[3 * ci + 2];
        }
      }
    }
  }
}

extern "C" int tslam_tsdf_extract_surface(tslam_tsdf_t* m, int32_t submap, int64_t cap, float* xyz, float* rgb, int32_t* count_dev,
                                          void* stream) {
  if (!m || !xyz || !count_dev) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  const float thres = (float)(m->cfg.voxel_scale * 1.8);  // dense_tsdf.py:39
  k_extract_surface<<<m->sm_count * 4, 256, 0, st>>>(m->g, submap, m->cfg.is_global_map, m->pose_R, m->pose_T, m->in.vs, thres,
                                                     (float)m->cfg.disp_floor, (float)m->cfg.disp_ceiling, m->colormap, cap, xyz,
                                                     rgb, count_dev);
  TS_LAUNCH_CHECK(m);
  return ts_check_deferred_async(m, st);
}

static float h16_round(float x) {  // slice_z is an f16 field (dense_tsdf.py:72)
  __half hv = __float2half_rn(x);
  return __half2float(hv);
}

extern "C" int tslam_tsdf_extract_slice(tslam_tsdf_t* m, int32_t submap, float z, float dz, int64_t cap, float* xyz, float* val,
                                        float* rgb, int32_t* count_dev, void* stream) {
  if (!m || !xyz || !count_dev) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  const int index = (int)(h16_round(z) / m->in.vs);  // :369-370
  k_extract_slice<<<m->sm_count * 4, 256, 0, st>>>(m->g, submap, m->cfg.is_global_map, m->pose_R, m->pose_T, m->in.vs, index, dz,
                                                   m->colormap, cap, xyz, val, rgb, count_dev);
  TS_LAUNCH_CHECK(m);
  return ts_check_deferred_async(m, st);
}

// ---------------------------------------------------------------------------
// submap -> global fusion  (dense_tsdf.py:272-318)
// One CTA per SOURCE block; each observed source voxel splats into the 7 upper
// trilinear corners (:297-300) with one 8-byte reduction per corner; commit
// (no Wmax clamp, :274-278) turns the sums into (TSDF, W).
// ---------------------------------------------------------------------------
__device__ __forceinline__ void sat_add_i8(int8_t* p, int add) {
  if (add == 0) return;
  unsigned int* wp = (unsigned int*)((uintptr_t)p & ~(uintptr_t)3);
  const int sh = (int)((uintptr_t)p & 3) * 8;
  unsigned int old = *wp, assumed;
  do {
    assumed = old;
    int cur = (int)(int8_t)((assumed >> sh) & 0xFF);
    int nv = cur + add;
    nv = nv > 127 ? 127 : (nv < -128 ? -128 : nv);  // reference wraps (i8); we saturate (DESIGN.md)
    unsigned int repl = (assumed & ~(0xFFu << sh)) | (((unsigned int)(nv & 0xFF)) << sh);
    old = atomicCAS(wp, assumed, repl);
  } while (old != assumed);
}

__global__ void __launch_bounds__(256) k_fuse(TsGrid dst, TsGrid src, const float* pR, const float* pT, float vs) {
  const int nb = min(*src.n_blocks, src.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(src.block_key[b], s, bx, by, bz);
    if (src.ghost[b]) continue;
    const size_t base = (size_t)b * TS_B3;
    unsigned long long cur_key = TS_EMPTY;
    int cur_blk = -1;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      if (!(src.obs[base + v] > 0)) continue;  // :292
      const float2 t = src.tw[base + v];
      const int occ = src.occ[base + v];
      const bool tex = dst.col != nullptr && src.col != nullptr;
      float4 sc = make_float4(0.f, 0.f, 0.f, 0.f);
      if (tex) sc = src.col[base + v];
      float x, y, z;
      pose_apply(pR + 9 * s, pT + 3 * s, (float)(bx * TS_B + (v >> 8)) * vs, (float)(by * TS_B + ((v >> 4) & 15)) * vs,
                 (float)(bz * TS_B + (v & 15)) * vs, x, y, z);  // :293-294
      const float gx = x / vs, gy = y / vs, gz = z / vs;
      const int lo0 = (int)floorf(gx), lo1 = (int)floorf(gy), lo2 = (int)floorf(gz);  // :296
#pragma unroll
      for (int c = 1; c < 8; c++) {  // c=0 (di=dj=dk=0) skipped: reference quirk :300
        const int ci = lo0 + ((c >> 2) & 1), cj = lo1 + ((c >> 1) & 1), ck = lo2 + (c & 1);
        const float wt = (1.0f - fabsf((float)ci - gx)) * (1.0f - fabsf((float)cj - gy)) * (1.0f - fabsf((float)ck - gz));  // :303
        if (!ts_in_bounds(dst, ci, cj, ck)) continue;
        const unsigned long long key = ts_pack_key(0, ci >> TS_BSHIFT, cj >> TS_BSHIFT, ck >> TS_BSHIFT);
        if (key != cur_key) {
          cur_key = key;
          cur_blk = ts_get_or_alloc_cached(dst, key);
          if (cur_blk >= 0) ts_mark_dirty(dst, cur_blk);
        }
        if (cur_blk < 0) continue;
        const size_t o = (size_t)cur_blk * TS_B3 + ts_voxel_off(ci, cj, ck);
        const float w = t.y * wt;                    // :307
        red_add_f32x2(&dst.acc[o], w * t.x, w);      // :274-275
        if (tex) {                                   // :276-277: sum w*c here, / sum w at commit
          float* dc = (float*)&dst.col[o];
          atomicAdd(dc, w * sc.x); atomicAdd(dc + 1, w * sc.y); atomicAdd(dc + 2, w * sc.z);
        }
        if (dst.obs[o] == 0) dst.obs[o] = 2;         // :279 observed, value pending (2 -> 1 at commit)
        sat_add_i8(&dst.occ[o], occ);                // :280
      }
    }
  }
}

extern "C" int tslam_tsdf_fuse(tslam_tsdf_t* dst, tslam_tsdf_t* src, void* stream) {
  if (!dst || !src || dst == src) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(src, st);
  if (rc) return rc;
  dst->n_integrate_calls = 0;  // pending updates of dst are discarded by reset() (:312-313)
  rc = tslam_tsdf_reset(dst, stream);
  if (rc) return rc;
  k_fuse<<<dst->sm_count * 8, 256, 0, st>>>(dst->g, src->g, dst->pose_R, dst->pose_T, dst->in.vs);
  TS_LAUNCH_CHECK(dst);
  return ts_launch_commit(dst, st, 0, 1);
}

// multi-GPU building blocks (see tslam_dist.cu): fusion that leaves its sums pending, and the fused commit
extern "C" int tslam_tsdf_fuse_pending(tslam_tsdf_t* dst, tslam_tsdf_t* src, void* stream) {
  if (!dst || !src || dst == src) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(src, st);
  if (rc) return rc;
  dst->n_integrate_calls = 0;
  rc = tslam_tsdf_reset(dst, stream);
  if (rc) return rc;
  k_fuse<<<dst->sm_count * 8, 256, 0, st>>>(dst->g, src->g, dst->pose_R, dst->pose_T, dst->in.vs);
  TS_LAUNCH_CHECK(dst);
  return TSLAM_OK;
}
extern "C" int tslam_tsdf_commit_fused(tslam_tsdf_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  return ts_launch_commit(m, (cudaStream_t)stream, 0, 1);
}

// ---------------------------------------------------------------------------
// stats / sync / profiling
// ---------------------------------------------------------------------------
extern "C" int tslam_tsdf_get_stats(tslam_tsdf_t* m, int64_t* out8, int clear) {
  if (!m || !out8) return TSLAM_E_INVALID;
  TS_CUDA(cudaDeviceSynchronize());
  TsCounters c;
  TS_CUDA(cudaMemcpy(&c, m->counters, sizeof(c), cudaMemcpyDeviceToHost));
  int sc[4];
  TS_CUDA(cudaMemcpy(sc, m->scratch_i, sizeof(sc), cudaMemcpyDeviceToHost));
  out8[0] = (int64_t)c.n_px; out8[1] = (int64_t)c.n_valid; out8[2] = (int64_t)c.n_rays; out8[3] = (int64_t)c.n_updates;
  out8[4] = (int64_t)c.n_oob; out8[5] = sc[0]; out8[6] = sc[2]; out8[7] = m->launches;
  if (clear) TS_CUDA(cudaMemset(m->counters, 0, sizeof(TsCounters)));
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_get_march_stats(tslam_tsdf_t* m, int64_t* out6) {
  if (!m || !out6) return TSLAM_E_INVALID;
  TS_CUDA(cudaDeviceSynchronize());
  TsCounters c;
  TS_CUDA(cudaMemcpy(&c, m->counters, sizeof(c), cudaMemcpyDeviceToHost));
  out6[0] = (int64_t)c.n_segs; out6[1] = (int64_t)c.n_items; out6[2] = (int64_t)c.n_slow; out6[3] = (int64_t)c.n_fallback;
  out6[4] = (int64_t)c.n_generic; out6[5] = (int64_t)c.n_verify_bad;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_get_march_stats2(tslam_tsdf_t* m, int64_t* out7) {
  if (!m || !out7) return TSLAM_E_INVALID;
  int rc = tslam_tsdf_get_march_stats(m, out7);
  if (rc) return rc;
  TsCounters c;
  TS_CUDA(cudaMemcpy(&c, m->counters, sizeof(c), cudaMemcpyDeviceToHost));
  out7[6] = (int64_t)c.n_seg_guard;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_sync(tslam_tsdf_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  TS_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return ts_check_deferred(m);
}

extern "C" int64_t tslam_tsdf_launch_count(tslam_tsdf_t* m) { return m ? m->launches : 0; }

extern "C" int tslam_tsdf_set_profiling(tslam_tsdf_t* m, int on) {
  if (!m) return TSLAM_E_INVALID;
  if (on && !m->ev) {
    m->ev = new cudaEvent_t[TS_PROF_EV * TS_PROF_RING];
    for (int i = 0; i < TS_PROF_EV * TS_PROF_RING; i++) TS_CUDA(cudaEventCreate(&m->ev[i]));
  }
  m->profiling = on;
  m->prof_launches = 0;
  return TSLAM_OK;
}
// ms3[3*i + {0,1,2}] = bucket / ray-march / commit(+reset) kernel time of the i-th most recent
// recorded integrate launch, i < n (n <= TS_PROF_RING).  Returns the number of rows written in *n_out.
// ms7[7*i + ...] = bucket, ray march (all of its kernels), commit, then the parts of the ray march: the interval between
// the bucket kernel and the first march kernel (0: nothing runs there), set-up + segment count + class + scan, segment
// fill, march (with the generic path and the resets).  The last four are 0 for launches of the legacy kernel.
extern "C" int tslam_tsdf_kernel_ms2(tslam_tsdf_t* m, int32_t n, float* ms7, int32_t* n_out) {
  if (!m || !ms7 || !n_out || !m->ev) return TSLAM_E_INVALID;
  TS_CUDA(cudaDeviceSynchronize());
  long long have = m->prof_launches < TS_PROF_RING ? m->prof_launches : TS_PROF_RING;
  if (n > have) n = (int32_t)have;
  for (int i = 0; i < n; i++) {
    cudaEvent_t* pe = m->ev + TS_PROF_EV * ((m->prof_launches - 1 - i) % TS_PROF_RING);
    for (int q = 0; q < 3; q++) TS_CUDA(cudaEventElapsedTime(&ms7[7 * i + q], pe[q], pe[q + 1]));
    for (int q = 0; q < 4; q++) ms7[7 * i + 3 + q] = 0.0f;
    if (m->march_mode && !m->g.cword) {  // pe[4], pe[5]: after the scan and after the scattering walk (ts_march_launch)
      TS_CUDA(cudaEventElapsedTime(&ms7[7 * i + 4], pe[1], pe[4]));
      TS_CUDA(cudaEventElapsedTime(&ms7[7 * i + 5], pe[4], pe[5]));
      TS_CUDA(cudaEventElapsedTime(&ms7[7 * i + 6], pe[5], pe[2]));
    }
  }
  *n_out = n;
  return TSLAM_OK;
}
extern "C" int tslam_tsdf_kernel_ms(tslam_tsdf_t* m, int32_t n, float* ms3, int32_t* n_out) {
  if (!m || !ms3 || !n_out || !m->ev) return TSLAM_E_INVALID;
  TS_CUDA(cudaDeviceSynchronize());
  long long have = m->prof_launches < TS_PROF_RING ? m->prof_launches : TS_PROF_RING;
  if (n > have) n = (int32_t)have;
  for (int i = 0; i < n; i++) {
    cudaEvent_t* pe = m->ev + TS_PROF_EV * ((m->prof_launches - 1 - i) % TS_PROF_RING);
    for (int q = 0; q < 3; q++) TS_CUDA(cudaEventElapsedTime(&ms3[3 * i + q], pe[q], pe[q + 1]));
  }
  *n_out = n;
  return TSLAM_OK;
}
