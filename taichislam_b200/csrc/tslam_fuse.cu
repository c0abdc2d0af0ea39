// libtslam.so - incremental fusion of a submap collection into a TSDF global map (tslam_tsdf_fuse_update).  sm_90a.
//
// Contract (DESIGN.md section 7, "Incremental global fusion").  The global map keeps, per voxel, exact integer sums of
// the terms k_fuse splats (tslam_tsdf.cu): every observed voxel of a non-ghost block of submap s, placed at its fused
// pose by ts_splat_pos / ts_splat_corner (the helpers k_fuse calls), adds to each in-volume corner c = 1 .. 7
//     w = W wt,  w T  and, on textured maps,  w c  per channel   (f32, as k_fuse forms them)
// each quantised to q(f) = llrint((double)f * 2^24).  A source voxel with a term that is not finite or has |f| >= 2^23
// adds nothing to any corner (it is counted as skipped).  Per dst voxel the sums are
//     S_wT, S_w (int64), S_c[3] (int64, textured maps), and  co = count * 2^32 + S_occ  (one int64 word)
// where count is the number of contributions and S_occ the sum of their source occ.  Readout of a voxel:
//     obs = count > 0,  T = (float)((double)S_wT / (double)S_w),  W = (float)((double)S_w * 2^-24),
//     occ = clamp(S_occ, -128, 127),  colour = (float)((double)S_c / (double)S_w)
// (count > 0 with S_w = 0 gives NaN like k_fuse's 0 / 0); count = 0 leaves the voxel as never written (all zero).
//
// Bounds.  A rigid placement puts at most 8 source voxels (points at mutual distance >= 1 voxel) into any closed unit
// cube of the global grid, and a dst voxel takes contributions from the 2 x 2 x 2 cube of cells around it: at most
// 64 per submap, 2^16 for 1024 submaps.  |q| < 2^23 * 2^24 = 2^47 per term, so every final sum is below 2^63 in
// magnitude, count < 2^16 and |S_occ| <= 128 * 2^16 < 2^31 (co decodes as count = (co + 2^31) >> 32).  The sums are
// kept with wrapping int64 additions, which commute: a partial sum that overflows while a moved submap's removal and
// re-addition are both in flight still ends on the exact total.  Because every sum is exact and order-free, dst does
// not depend on the history of updates: any sequence of calls ends bit for bit where one call on a fresh map would.
//
// An update plans on the host (per-submap block counts and radii from k_fz_plan), lists the source blocks of the
// submaps with work (k_fz_list), activates the dst blocks the additions need (k_fz_splat<0>), grows the sum planes
// to the pool blocks in use, splats (k_fz_splat<1>: removals at the old pose, additions at the new one) and reads the
// touched blocks out of the sums (k_fz_commit), stamping them for the incremental mesh and the ESDF.
#include <cmath>
#include <cstring>
#include <vector>
#include "tslam_internal.cuh"

#define FZ_Q 16777216.0             // 2^24: quantum of the sums
#define FZ_FMAX 8388608.0f          // 2^23: terms at or above this magnitude are skipped
#define TS_ERR_FUSE_MISSING 16      // g.err: a removal found no dst block (the sums and the pool disagree)

// full-update reasons (stats8[0]; 0 = incremental)
enum { FZ_INCR = 0, FZ_FIRST = 1, FZ_ASKED = 2, FZ_OTHER_SRC = 3, FZ_DST_WRITTEN = 4, FZ_CONTENT = 5, FZ_COST = 6 };

struct FzJob {        // one placement of one submap: sign +1 adds, -1 removes
  float R[9], T[3];
  int sign, pad;
};
struct FzSums {       // sum planes, [cap blocks * 4096] int64 each
  long long* wt;      // S_wT
  long long* w;       // S_w
  long long* co;      // count << 32 + S_occ
  long long* c;       // textured maps: 3 planes S_c (c + p * stride), else null
  size_t stride;      // elements per plane
};
struct FzDev {        // device scratch of one update (TsFuse::dev)
  int* nblk;          // [max_submaps] non-ghost source blocks per submap (k_fz_plan)
  unsigned* rbits;    // [max_submaps] float bits of the farthest block corner from the submap origin (k_fz_plan)
  int2* job_of;       // [max_submaps] (removal job, addition job), -1 none
  FzJob* jobs;        // [2 * max_submaps]
  int* list;          // [src max_blocks] source blocks with work
  unsigned long long* ctr;  // [0] list length, [1] voxels splatted, [2] voxels skipped, [3] dst ghost blocks, [4] dirty blocks
};

struct FzSub {        // what a submap contributes to dst (TsFuse::sub)
  int fused;          // 1: its voxels are in the sums, at (R, T)
  float R[9], T[3];
  unsigned long long ver;  // src content version at that time
  int nblk;           // its non-ghost source blocks then
};
struct TsFuse {
  int valid;          // the sums describe dst (cleared by a failed update)
  unsigned long long src_serial, gen;  // src handle and dst write generation of the last update
  std::vector<FzSub> sub;
  void* sums;         // sum planes (grown geometrically, never shrunk)
  size_t cap_blocks;
  void* dev;          // FzDev arrays
  size_t dev_bytes;
  int dev_submaps, dev_blocks;
};

static unsigned long long g_serial = 0;  // handle numbers (create is not called concurrently with itself here)

int ts_fuse_init(tslam_tsdf* m) {
  m->serial = __atomic_add_fetch(&g_serial, 1ull, __ATOMIC_RELAXED);
  m->write_gen = 0;
  m->content_ver = new unsigned long long[m->cfg.max_submaps]();
  m->fz = nullptr;
  return TSLAM_OK;
}

void ts_fuse_free(tslam_tsdf* m) {
  delete[] m->content_ver;
  m->content_ver = nullptr;
  if (m->fz) {
    if (m->fz->sums) cudaFree(m->fz->sums);
    if (m->fz->dev) cudaFree(m->fz->dev);
    delete m->fz;
    m->fz = nullptr;
  }
}

void ts_map_written(tslam_tsdf* m, int submap) {
  m->write_gen++;
  if (!m->content_ver) return;
  if (submap < 0) {
    for (int s = 0; s < m->cfg.max_submaps; s++) m->content_ver[s]++;
  } else if (submap < m->cfg.max_submaps) {
    m->content_ver[submap]++;
  }
}

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
// non-ghost blocks and radius per source submap; ghost blocks of dst
__global__ void __launch_bounds__(256) k_fz_plan(TsGrid src, TsGrid dst, float vs, FzDev f) {
  const int nb = min(*src.n_blocks, src.max_blocks);
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    if (src.ghost[b]) continue;
    int s, bx, by, bz;
    ts_unpack_key(src.block_key[b], s, bx, by, bz);
    const float ex = fmaxf(fabsf((float)(bx * TS_B) * vs), fabsf((float)(bx * TS_B + TS_B) * vs));
    const float ey = fmaxf(fabsf((float)(by * TS_B) * vs), fabsf((float)(by * TS_B + TS_B) * vs));
    const float ez = fmaxf(fabsf((float)(bz * TS_B) * vs), fabsf((float)(bz * TS_B + TS_B) * vs));
    atomicAdd(&f.nblk[s], 1);
    atomicMax(&f.rbits[s], __float_as_uint(sqrtf(ex * ex + ey * ey + ez * ez)));  // non-negative floats order as uints
  }
  const int nd = min(*dst.n_blocks, dst.max_blocks);
  unsigned ng = 0;
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nd; b += gridDim.x * blockDim.x) ng += dst.ghost[b] != 0;
  if (ng) atomicAdd(&f.ctr[3], (unsigned long long)ng);
}

// the non-ghost source blocks of submaps with a job
__global__ void __launch_bounds__(256) k_fz_list(TsGrid src, FzDev f) {
  const int nb = min(*src.n_blocks, src.max_blocks);
  const int stride = gridDim.x * blockDim.x;
  const int iters = (nb + stride - 1) / stride;
  for (int it = 0; it < iters; ++it) {
    const int b = it * stride + blockIdx.x * blockDim.x + threadIdx.x;
    bool want = false;
    if (b < nb && !src.ghost[b]) {
      int s, bx, by, bz;
      ts_unpack_key(src.block_key[b], s, bx, by, bz);
      const int2 j = f.job_of[s];
      want = j.x >= 0 || j.y >= 0;
    }
    const long long row = warp_append_u64(want, &f.ctr[0]);
    if (want) f.list[row] = b;
  }
}

__device__ __forceinline__ bool fz_term_ok(float x) { return fabsf(x) < FZ_FMAX; }  // false for NaN and +-inf too
__device__ __forceinline__ long long fz_q(float x) { return __double2ll_rn((double)x * FZ_Q); }

// One CTA per listed source block.  PASS 0 activates the dst blocks of the additions; PASS 1 adds each job's signed
// terms into the sum planes (removals find their blocks, or raise TS_ERR_FUSE_MISSING) and flags the blocks it touched.
template <int PASS>
__global__ void __launch_bounds__(256) k_fz_splat(TsGrid dst, TsGrid src, FzDev f, FzSums S, float vs) {
  const int nl = (int)f.ctr[0];
  const bool tex = dst.col != nullptr && src.col != nullptr;  // (the host refuses maps that differ in it)
  unsigned long long n_splat = 0, n_skip = 0;
  for (int q = blockIdx.x; q < nl; q += gridDim.x) {
    const int b = f.list[q];
    int s, bx, by, bz;
    ts_unpack_key(src.block_key[b], s, bx, by, bz);
    const int2 jj = f.job_of[s];
    for (int r = 0; r < 2; r++) {
      const int job = r == 0 ? jj.x : jj.y;
      if (job < 0) continue;
      const FzJob& J = f.jobs[job];
      const int sign = J.sign;
      if (PASS == 0 && sign < 0) continue;
      const size_t base = (size_t)b * TS_B3;
      unsigned long long cur_key = TS_EMPTY;
      int cur_blk = -1;
      for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
        if (!(src.obs[base + v] > 0)) continue;
        const float2 t = src.tw[base + v];
        const int occ = src.occ[base + v];
        float4 sc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (tex) sc = src.col[base + v];
        const TsSplatPos p = ts_splat_pos(J.R, J.T, (float)(bx * TS_B + (v >> 8)) * vs, (float)(by * TS_B + ((v >> 4) & 15)) * vs,
                                          (float)(bz * TS_B + (v & 15)) * vs, vs);
        bool ok = true;
#pragma unroll
        for (int c = 1; c < 8; c++) {
          int ci, cj, ck;
          float wt;
          if (!ts_splat_corner(dst, p, c, ci, cj, ck, wt)) continue;
          const float w = t.y * wt;
          ok = ok && fz_term_ok(w) && fz_term_ok(w * t.x);
          if (tex) ok = ok && fz_term_ok(w * sc.x) && fz_term_ok(w * sc.y) && fz_term_ok(w * sc.z);
        }
        if (!ok) { n_skip++; continue; }
        n_splat++;
#pragma unroll
        for (int c = 1; c < 8; c++) {
          int ci, cj, ck;
          float wt;
          if (!ts_splat_corner(dst, p, c, ci, cj, ck, wt)) continue;
          const unsigned long long key = ts_pack_key(0, ci >> TS_BSHIFT, cj >> TS_BSHIFT, ck >> TS_BSHIFT);
          if (key != cur_key) {
            cur_key = key;
            if (PASS == 0) {
              cur_blk = ts_get_or_alloc_cached(dst, key);
            } else {
              cur_blk = ts_find(dst, key);
              if (cur_blk >= 0) ts_mark_dirty(dst, cur_blk);
              else if (sign < 0) atomicOr(dst.err, TS_ERR_FUSE_MISSING);
            }
          }
          if (PASS == 0 || cur_blk < 0) continue;
          const size_t o = (size_t)cur_blk * TS_B3 + ts_voxel_off(ci, cj, ck);
          const float w = t.y * wt;
          const long long qw = fz_q(w), qwt = fz_q(w * t.x), qco = (1ll << 32) + (long long)occ;
          red_add_u64((unsigned long long*)&S.wt[o], (unsigned long long)(sign > 0 ? qwt : -qwt));
          red_add_u64((unsigned long long*)&S.w[o], (unsigned long long)(sign > 0 ? qw : -qw));
          red_add_u64((unsigned long long*)&S.co[o], (unsigned long long)(sign > 0 ? qco : -qco));
          if (tex) {
            const long long q0 = fz_q(w * sc.x), q1 = fz_q(w * sc.y), q2 = fz_q(w * sc.z);
            red_add_u64((unsigned long long*)&S.c[o], (unsigned long long)(sign > 0 ? q0 : -q0));
            red_add_u64((unsigned long long*)&S.c[S.stride + o], (unsigned long long)(sign > 0 ? q1 : -q1));
            red_add_u64((unsigned long long*)&S.c[2 * S.stride + o], (unsigned long long)(sign > 0 ? q2 : -q2));
          }
        }
      }
    }
  }
  if (PASS == 1) {
    for (int o = 16; o > 0; o >>= 1) {
      n_splat += __shfl_xor_sync(0xffffffffu, n_splat, o);
      n_skip += __shfl_xor_sync(0xffffffffu, n_skip, o);
    }
    if ((threadIdx.x & 31) == 0) {
      if (n_splat) atomicAdd(&f.ctr[1], n_splat);
      if (n_skip) atomicAdd(&f.ctr[2], n_skip);
    }
  }
}

// read the voxels of the dirty blocks out of the sums; stamp the blocks for the incremental mesh and the ESDF
__global__ void __launch_bounds__(256) k_fz_commit(TsGrid g, FzSums S, unsigned long long* stamp, unsigned long long seq) {
  const int nd = *g.n_dirty;
  for (int q = blockIdx.x; q < nd; q += gridDim.x) {
    const int blk = g.dirty_list[q];
    const size_t base = (size_t)blk * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const size_t o = base + v;
      const long long co = S.co[o];
      const long long cnt = (co + (1ll << 31)) >> 32;
      const long long socc = co - (long long)((unsigned long long)cnt << 32);
      if (cnt == 0) {
        g.tw[o] = make_float2(0.0f, 0.0f);
        g.obs[o] = 0;
        g.occ[o] = 0;
        if (g.col) g.col[o] = make_float4(0.f, 0.f, 0.f, 0.f);
        continue;
      }
      const double sw = (double)S.w[o];
      g.tw[o] = make_float2((float)((double)S.wt[o] / sw), (float)(sw * (1.0 / FZ_Q)));
      g.obs[o] = 1;
      g.occ[o] = (int8_t)(socc > 127 ? 127 : (socc < -128 ? -128 : socc));
      if (g.col && S.c)
        g.col[o] = make_float4((float)((double)S.c[o] / sw), (float)((double)S.c[S.stride + o] / sw), (float)((double)S.c[2 * S.stride + o] / sw), 0.0f);
    }
    if (threadIdx.x == 0) {
      g.dirty_flag[blk] = 0;
      g.esdf_dirty[blk] = 1;
      stamp[blk] = seq;
    }
  }
}

// ---------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------
static int fz_planes(const tslam_tsdf* m) { return m->g.col ? 6 : 3; }

static FzSums fz_sums(const TsFuse* z, int planes) {
  FzSums S;
  const size_t n = z->cap_blocks * TS_B3;
  long long* p = (long long*)z->sums;
  S.stride = n;
  S.wt = p;
  S.w = p + n;
  S.co = p + 2 * n;
  S.c = planes == 6 ? p + 3 * n : nullptr;
  return S;
}

// sum planes for at least `need` pool blocks: grown to max(need, 2 x cap) (at most max_blocks), the old sums kept
static int fz_reserve_sums(tslam_tsdf* m, size_t need, cudaStream_t st) {
  TsFuse* z = m->fz;
  if (need <= z->cap_blocks) return TSLAM_OK;
  size_t cap = std::max(need, 2 * z->cap_blocks);
  if (cap > (size_t)m->g.max_blocks) cap = (size_t)m->g.max_blocks;
  const int planes = fz_planes(m);
  const size_t bytes = cap * TS_B3 * 8 * planes;
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    ts_set_error("fuse_update: cannot allocate %zu bytes of sum planes (%zu pool blocks x %d planes x 32 KiB): %s", bytes, cap, planes,
                 cudaGetErrorString(e));
    return TSLAM_E_CUDA;
  }
  const size_t old_n = z->cap_blocks * TS_B3, n = cap * TS_B3;
  for (int k = 0; k < planes; k++) {
    long long* dstp = (long long*)p + k * n;
    if (old_n) TS_CUDA(cudaMemcpyAsync(dstp, (long long*)z->sums + k * old_n, old_n * 8, cudaMemcpyDeviceToDevice, st));
    TS_CUDA(cudaMemsetAsync(dstp + old_n, 0, (n - old_n) * 8, st));
  }
  if (z->sums) {
    TS_CUDA(cudaStreamSynchronize(st));
    TS_CUDA(cudaFree(z->sums));
  }
  z->sums = p;
  z->cap_blocks = cap;
  return TSLAM_OK;
}

static int fz_reserve_dev(tslam_tsdf* dst, tslam_tsdf* src, FzDev& f) {
  TsFuse* z = dst->fz;
  const int S = dst->cfg.max_submaps, B = src->g.max_blocks;
  if (!z->dev || z->dev_submaps != S || z->dev_blocks < B) {
    if (z->dev) TS_CUDA(cudaFree(z->dev));
    z->dev = nullptr;
    const size_t bytes = (size_t)S * (4 + 4 + 8) + (size_t)2 * S * sizeof(FzJob) + (size_t)B * 4 + 8 * 8 + 256;
    TS_CUDA(cudaMalloc(&z->dev, bytes));
    z->dev_bytes = bytes;
    z->dev_submaps = S;
    z->dev_blocks = B;
  }
  char* p = (char*)z->dev;
  f.ctr = (unsigned long long*)p; p += 8 * 8;
  f.jobs = (FzJob*)p; p += (size_t)2 * S * sizeof(FzJob);
  f.job_of = (int2*)p; p += (size_t)S * 8;
  f.nblk = (int*)p; p += (size_t)S * 4;
  f.rbits = (unsigned*)p; p += (size_t)S * 4;
  f.list = (int*)p;
  return TSLAM_OK;
}

// rotation angle of R0^T R (row-major 3x3), in double
static double fz_angle(const float* R0, const float* R) {
  double tr = 0.0;
  for (int i = 0; i < 3; i++)
    for (int k = 0; k < 3; k++) tr += (double)R0[3 * k + i] * (double)R[3 * k + i];  // trace(R0^T R) = sum R0_ki R_ki
  double c = (tr - 1.0) * 0.5;
  c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
  return std::acos(c);
}

extern "C" int tslam_tsdf_fuse_update(tslam_tsdf_t* dst, tslam_tsdf_t* src, const uint8_t* include, float tolerance, int32_t full,
                                      int64_t* stats8, void* stream) {
  if (!std::isfinite(tolerance) || tolerance < 0.0f) { ts_set_error("fuse_update: tolerance %g must be finite and >= 0", (double)tolerance); return TSLAM_E_INVALID; }
  if (!dst || !src) { ts_set_error("fuse_update: NULL handle"); return TSLAM_E_INVALID; }
  if (dst == src) { ts_set_error("fuse_update: dst == src (a map cannot be fused into itself)"); return TSLAM_E_INVALID; }
  if (!dst->cfg.is_global_map) { ts_set_error("fuse_update: dst is not a global map (is_global_map = 0)"); return TSLAM_E_INVALID; }
  if (dst->cfg.max_submaps != src->cfg.max_submaps || dst->in.vs != src->in.vs || (dst->g.col != nullptr) != (src->g.col != nullptr)) {
    ts_set_error("fuse_update: dst and src differ in max_submaps (%d, %d), voxel size (%g, %g) or texture setting (%d, %d)", dst->cfg.max_submaps,
                 src->cfg.max_submaps, (double)dst->in.vs, (double)src->in.vs, dst->g.col != nullptr, src->g.col != nullptr);
    return TSLAM_E_INVALID;
  }
  if (dst->tile_cuts_set) { ts_set_error("fuse_update: dst is a tiled map (tile cuts set): not supported"); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const int S = dst->cfg.max_submaps;
  int rc = ts_flush_pending(src, st);
  if (rc) return rc;
  rc = ts_flush_pending(dst, st);
  if (rc) return rc;
  if (!dst->fz) {
    dst->fz = new TsFuse();
    dst->fz->valid = 0;
    dst->fz->sums = nullptr;
    dst->fz->cap_blocks = 0;
    dst->fz->dev = nullptr;
    dst->fz->sub.assign(S, FzSub());
  }
  TsFuse* z = dst->fz;
  FzDev f;
  rc = fz_reserve_dev(dst, src, f);
  if (rc) return rc;

  // plan: source blocks and radius per submap, dst ghosts, dst poses
  TS_CUDA(cudaMemsetAsync(f.ctr, 0, 8 * 8, st));
  TS_CUDA(cudaMemsetAsync(f.nblk, 0, (size_t)S * 8, st));  // nblk and rbits
  const int gp = src->sm_count * 4;
  k_fz_plan<<<gp, 256, 0, st>>>(src->g, dst->g, src->in.vs, f);
  TS_LAUNCH_CHECK(dst);
  std::vector<int> nblk(S);
  std::vector<float> rad(S), pR((size_t)S * 9), pT((size_t)S * 3);
  unsigned long long ctr0[8];
  TS_CUDA(cudaMemcpyAsync(nblk.data(), f.nblk, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(rad.data(), f.rbits, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(ctr0, f.ctr, sizeof(ctr0), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(pR.data(), dst->pose_R, (size_t)S * 36, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(pT.data(), dst->pose_T, (size_t)S * 12, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (ctr0[3] > 0) { ts_set_error("fuse_update: dst holds %llu ghost blocks (a tiled map): not supported", ctr0[3]); return TSLAM_E_INVALID; }

  int reason = FZ_INCR;
  if (full) reason = FZ_ASKED;
  else if (!z->valid) reason = FZ_FIRST;
  else if (z->src_serial != src->serial) reason = FZ_OTHER_SRC;
  else if (z->gen != dst->write_gen) reason = FZ_DST_WRITTEN;
  enum { NONE = 0, ADD, REMOVE, MOVE, KEEP };
  std::vector<unsigned char> act(S, NONE);
  long long n_add = 0, n_move = 0, n_remove = 0, n_tol = 0, cost = 0, cost_full = 0;
  for (int s = 0; s < S; s++) {
    const bool want = (!include || include[s]) && nblk[s] > 0;
    if (want) cost_full += nblk[s];
    if (reason != FZ_INCR) continue;
    const FzSub& r = z->sub[s];
    if (!r.fused) {
      if (want) { act[s] = ADD; cost += nblk[s]; }
      continue;
    }
    if (r.ver != src->content_ver[s]) { reason = FZ_CONTENT; continue; }  // its old content is gone: cannot be subtracted
    if (!want) { act[s] = REMOVE; cost += r.nblk; continue; }
    const float* R = &pR[(size_t)9 * s];
    const float* T = &pT[(size_t)3 * s];
    if (!memcmp(R, r.R, 36) && !memcmp(T, r.T, 12)) { act[s] = KEEP; continue; }
    if (tolerance > 0.0f) {
      const double dx = (double)T[0] - r.T[0], dy = (double)T[1] - r.T[1], dz = (double)T[2] - r.T[2];
      const double move = std::sqrt(dx * dx + dy * dy + dz * dz) + fz_angle(r.R, R) * (double)rad[s];
      if (move <= (double)tolerance) { act[s] = KEEP; n_tol++; continue; }
    }
    act[s] = MOVE;
    cost += r.nblk + nblk[s];
  }
  if (reason == FZ_INCR && cost > cost_full) reason = FZ_COST;
  const bool is_full = reason != FZ_INCR;
  if (is_full) {
    n_add = n_move = n_remove = n_tol = 0;
    for (int s = 0; s < S; s++) act[s] = ((!include || include[s]) && nblk[s] > 0) ? ADD : NONE;
  }
  for (int s = 0; s < S; s++) {
    n_add += act[s] == ADD;
    n_move += act[s] == MOVE;
    n_remove += act[s] == REMOVE;
  }

  // jobs
  std::vector<FzJob> jobs;
  std::vector<int2> job_of(S, make_int2(-1, -1));
  for (int s = 0; s < S; s++) {
    if (act[s] == REMOVE || act[s] == MOVE) {
      FzJob j;
      memcpy(j.R, z->sub[s].R, 36); memcpy(j.T, z->sub[s].T, 12);
      j.sign = -1; j.pad = 0;
      job_of[s].x = (int)jobs.size();
      jobs.push_back(j);
    }
    if (act[s] == ADD || act[s] == MOVE) {
      FzJob j;
      memcpy(j.R, &pR[(size_t)9 * s], 36); memcpy(j.T, &pT[(size_t)3 * s], 12);
      j.sign = 1; j.pad = 0;
      job_of[s].y = (int)jobs.size();
      jobs.push_back(j);
    }
  }

  const int planes = fz_planes(dst);
  z->valid = 0;  // until this update completes
  if (is_full) {
    const unsigned long long gen = dst->write_gen;
    rc = tslam_tsdf_reset(dst, stream);  // also compacts the pool: blocks left empty by removals are dropped
    if (rc) return rc;
    dst->write_gen = gen;
    // every plane in full: a reset of dst since the last update left the pool empty but not the sums (at most 2x the
    // blocks in use: the planes grow geometrically)
    if (z->sums) TS_CUDA(cudaMemsetAsync(z->sums, 0, z->cap_blocks * TS_B3 * 8 * planes, st));
  }
  if (!jobs.empty()) {
    TS_CUDA(cudaMemcpyAsync(f.jobs, jobs.data(), jobs.size() * sizeof(FzJob), cudaMemcpyHostToDevice, st));
    TS_CUDA(cudaMemcpyAsync(f.job_of, job_of.data(), (size_t)S * 8, cudaMemcpyHostToDevice, st));
    const int gl = std::max(1, std::min((src->g.max_blocks + 255) / 256, src->sm_count * 4));
    k_fz_list<<<gl, 256, 0, st>>>(src->g, f);
    TS_LAUNCH_CHECK(dst);
    const int gs = dst->sm_count * 8;
    if (n_add + n_move > 0) {
      k_fz_splat<0><<<gs, 256, 0, st>>>(dst->g, src->g, f, FzSums{}, dst->in.vs);
      TS_LAUNCH_CHECK(dst);
    }
    int nb = 0, err = 0;
    TS_CUDA(cudaMemcpyAsync(&nb, dst->g.n_blocks, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaMemcpyAsync(&err, dst->g.err, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
    if (err) return ts_check_deferred(dst);  // pool exhausted: nothing was added; the next update is a full one
    rc = fz_reserve_sums(dst, (size_t)std::min(nb, dst->g.max_blocks), st);
    if (rc) return rc;
    k_fz_splat<1><<<gs, 256, 0, st>>>(dst->g, src->g, f, fz_sums(z, planes), dst->in.vs);
    TS_LAUNCH_CHECK(dst);
  }
  // commit the touched blocks
  rc = ts_collect_dirty(dst, st);
  if (rc) return rc;
  TS_CUDA(cudaMemcpyAsync(&f.ctr[4], dst->g.n_dirty, 4, cudaMemcpyDeviceToDevice, st));
  if (z->sums) {
    const unsigned long long seq = ++dst->commit_seq;  // stamp of every block this update writes (incremental mesh)
    k_fz_commit<<<dst->sm_count * 4, 256, 0, st>>>(dst->g, fz_sums(z, planes), dst->blk_stamp, seq);
    TS_LAUNCH_CHECK(dst);
  }
  TS_CUDA(cudaMemsetAsync(dst->g.n_dirty, 0, 4, st));
  unsigned long long ctr[8];
  int err = 0;
  TS_CUDA(cudaMemcpyAsync(ctr, f.ctr, sizeof(ctr), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(&err, dst->g.err, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (err & TS_ERR_FUSE_MISSING) {
    const int rest = err & ~TS_ERR_FUSE_MISSING;
    TS_CUDA(cudaMemcpy(dst->g.err, &rest, 4, cudaMemcpyHostToDevice));
    ts_set_error("fuse_update: a removal found no block of dst (its sums and pool disagree); the next update is a full one");
    return TSLAM_E_CUDA;
  }
  rc = ts_check_deferred(dst);
  if (rc) return rc;
  // voxels that lose their last contribution become unobserved, which the incremental ESDF does not undo
  if (n_remove + n_move > 0) dst->esdf_full_needed = 1;

  for (int s = 0; s < S; s++) {
    FzSub& r = z->sub[s];
    if (is_full) r.fused = 0;
    if (act[s] == REMOVE) r.fused = 0;
    if (act[s] == ADD || act[s] == MOVE) {
      r.fused = 1;
      memcpy(r.R, &pR[(size_t)9 * s], 36);
      memcpy(r.T, &pT[(size_t)3 * s], 12);
      r.ver = src->content_ver[s];
      r.nblk = nblk[s];
    }
  }
  z->valid = 1;
  z->src_serial = src->serial;
  z->gen = dst->write_gen;
  if (stats8) {
    stats8[0] = reason;
    stats8[1] = n_add;
    stats8[2] = n_move;
    stats8[3] = n_remove;
    stats8[4] = n_tol;
    stats8[5] = (int64_t)ctr[1];
    stats8[6] = (int64_t)ctr[2];
    stats8[7] = (int64_t)(unsigned)ctr[4];
  }
  return TSLAM_OK;
}
