// libtslam.so - incremental fusion of Octomap submaps into an Octomap global map (tslam_octo_fuse_update).  sm_90a.
//
// Contract (include/tslam.h; DESIGN.md section 7, "Incremental Octomap fusion").  After an update, every voxel word
// and colour word of dst is what tslam_octo_fuse gives for the included submaps at their fused poses: every source
// voxel the rule of dst carries over (OcHits: c > min_occupy_thres, OcLogodds: known) is placed by oc_fuse_cell, the
// helper k_octo_fuse calls, and
//   hit counter: dst.cnt = sum of c mod 2^32.  Removals subtract in the cnt plane itself: wrapping u32 arithmetic is
//                exact, so the plane is its own sum.
//   log-odds:    a sum word per voxel, co = count * 2^32 + sum L (int64, wrapping adds), and the readout
//                count > 0 ? lo_word(clamp(sum L, l_min, l_max)) : 0.
//   colour:      max of the source colour words (seq << 24 | rgb).  A max cannot be subtracted: the colour words of
//                every dst block a removal touched are cleared and raised again from the included submaps.
// Bounds.  A rigid placement puts at most 27 source voxels into one dst cell: the voxels are lattice points at mutual
// distance vs, the cell is a cube of side vs (plus f32 rounding, far below 1 %), and its 27 sub-cubes of side
// (1 + eps) vs / 3 have a diameter below vs, so each holds at most one of them.  With at most 1024 submaps a cell takes
// at most 27 * 1024 < 2^15 contributions, and |L| <= Lmax (the source's clamp limits) keeps |sum L| <= 27 * S * Lmax.
// The update refuses maps where that can reach 2^30: then count fits 2^31 and co decodes as count = (co + 2^31) >> 32.
// Why the readout is k_octo_fuse's: k_octo_fuse adds L << 1 per contribution (wrapping u32) and ORs the known bit, then
// k_octo_lo_clamp clamps once.  With |sum L| < 2^30 the u32 sum is 2 sum L exactly as an int32, its low bit is zero,
// so the word is lo_word(sum L) and its clamp is lo_word(clamp(sum L)); a cell without contributions stays 0.
// Every sum is exact and order-free, so dst does not depend on the history of updates.
//
// An update plans on the host (source blocks and radius per submap from k_of_plan, tslam_fuse_plan.cuh's rule), lists
// the source blocks of the submaps with work (k_of_list), activates the dst blocks the additions need (k_of_splat<0>),
// grows the sum words to the pool blocks in use (log-odds), adds the signed terms (k_of_splat<1>), reads the touched
// blocks out of the sums and flags them for the trackers (k_of_commit), and on textured maps recolours the blocks
// removals touched (k_of_list + k_of_recolour).
#include <cmath>
#include <cstring>
#include <type_traits>
#include <vector>
#include "tslam_internal.cuh"
#include "tslam_fuse_plan.cuh"

#define OF_CELL_MAX 27                // source voxels one rigid placement can put into one dst cell
#define OF_SUM_LIMIT (1ll << 30)      // |sum L| of a log-odds cell stays below this
#define OF_TOUCHED 1                  // dflag bits: the update changed the block's words ...
#define OF_RECOLOUR 2                 // ... and a removal touched it (its colour words are recomputed)

struct OfDev {        // device scratch of one update (OcFuse::dev)
  int* nblk;          // [max_submaps] source blocks per submap (k_of_plan)
  unsigned* rbits;    // [max_submaps] float bits of the farthest block corner from the submap origin (k_of_plan)
  int2* job_of;       // [max_submaps] (removal job, addition job), -1 none
  FzJob* jobs;        // [2 * max_submaps]
  int* list;          // [src max_blocks] source blocks with work
  int* dflag;         // [dst max_blocks] OF_TOUCHED | OF_RECOLOUR
  int* dlist;         // [dst max_blocks] touched dst blocks
  unsigned long long* ctr;  // [0] list length, [1] source voxels placed, [2] voxels recoloured, [3] touched dst blocks
};

struct OcFuse {
  int valid;          // dst and its sums are the fusion of the recorded submaps (cleared by a failed update)
  unsigned long long src_serial, gen;  // src handle and dst write generation of the last update
  std::vector<FzSub> sub;
  long long* sums;    // log-odds: [cap_blocks * 512] sum words (grown geometrically, never shrunk)
  size_t cap_blocks;
  void* dev;          // OfDev arrays
  int dev_submaps, dev_src_blocks, dev_dst_blocks;
};

void oc_map_written(tslam_octo* m, int submap) {
  m->write_gen++;
  if (!m->content_ver) return;
  if (submap < 0) {
    for (int s = 0; s < m->cfg.max_submaps; s++) m->content_ver[s]++;
  } else if (submap < m->cfg.max_submaps) {
    m->content_ver[submap]++;
  }
}

void oc_fuse_free(tslam_octo* m) {
  if (!m->ofz) return;
  if (m->ofz->sums) cudaFree(m->ofz->sums);
  if (m->ofz->dev) cudaFree(m->ofz->dev);
  delete m->ofz;
  m->ofz = nullptr;
}

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
// blocks and radius per source submap (8^3 blocks; the corners bound every voxel of the block)
__global__ void __launch_bounds__(256) k_of_plan(OcGrid src, float vs, OfDev f) {
  const int nb = min(*src.n_blocks, src.max_blocks);
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(src.block_key[b], s, bx, by, bz);
    const float ex = fmaxf(fabsf((float)(bx * OC_B) * vs), fabsf((float)(bx * OC_B + OC_B) * vs));
    const float ey = fmaxf(fabsf((float)(by * OC_B) * vs), fabsf((float)(by * OC_B + OC_B) * vs));
    const float ez = fmaxf(fabsf((float)(bz * OC_B) * vs), fabsf((float)(bz * OC_B + OC_B) * vs));
    atomicAdd(&f.nblk[s], 1);
    atomicMax(&f.rbits[s], __float_as_uint(sqrtf(ex * ex + ey * ey + ez * ez)));  // non-negative floats order as uints
  }
}

// the source blocks of submaps with a job
__global__ void __launch_bounds__(256) k_of_list(OcGrid src, OfDev f) {
  const int nb = min(*src.n_blocks, src.max_blocks);
  const int stride = gridDim.x * blockDim.x;
  const int iters = (nb + stride - 1) / stride;
  for (int it = 0; it < iters; ++it) {  // uniform trip count: the warp ballot below needs all lanes
    const int b = it * stride + blockIdx.x * blockDim.x + threadIdx.x;
    bool want = false;
    if (b < nb) {
      int s, bx, by, bz;
      ts_unpack_key(src.block_key[b], s, bx, by, bz);
      const int2 j = f.job_of[s];
      want = j.x >= 0 || j.y >= 0;
    }
    const long long row = warp_append_u64(want, &f.ctr[0]);
    if (want) f.list[row] = b;
  }
}

// first touch of dst block blk by this update (bits: OF_TOUCHED, | OF_RECOLOUR for a removal)
__device__ __forceinline__ void of_flag(const OfDev& f, int blk, int bits) {
  if ((*(volatile int*)&f.dflag[blk] & bits) == bits) return;
  if (atomicOr(&f.dflag[blk], bits) == 0) f.dlist[atomicAdd(&f.ctr[3], 1ull)] = blk;
}

// One CTA per listed source block, 4 voxels per thread.  PASS 0 activates the dst blocks of the additions; PASS 1 adds
// each job's signed terms (hit counter: into cnt; log-odds: into the sum words), raises the colour words of additions,
// and flags the dst blocks it touches (removals find their blocks, or raise OC_ERR_FUSE_MISSING).
template <int PASS, class Rule>
__global__ void __launch_bounds__(128) k_of_splat(OcGrid dst, OcGrid src, OfDev f, long long* sums, Rule rule, float vs) {
  constexpr bool LO = std::is_same<Rule, OcLogodds>::value;
  const int nl = (int)f.ctr[0];
  const bool tex = dst.cw != nullptr && src.cw != nullptr;  // (the host refuses maps that differ in it)
  unsigned long long n_place = 0;
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
      unsigned long long cur_key = TS_EMPTY;
      int cur_blk = -1;
      for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
        const size_t e = (size_t)b * OC_B3 + v;
        const unsigned int c = src.cnt[e];
        if (!rule.fuse_src(c)) continue;
        n_place++;
        int i, j, k;
        oc_fuse_cell(J.R, J.T, bx, by, bz, v, vs, i, j, k);
        if (!ts_in_bounds(dst, i, j, k)) continue;
        const unsigned long long key = ts_pack_key(0, i >> OC_BSHIFT, j >> OC_BSHIFT, k >> OC_BSHIFT);
        if (key != cur_key) {
          cur_key = key;
          if (PASS == 0) {
            cur_blk = ts_get_or_alloc_cached(dst, key);
          } else {
            cur_blk = ts_find(dst, key);
            if (cur_blk >= 0) of_flag(f, cur_blk, sign < 0 ? (OF_TOUCHED | OF_RECOLOUR) : OF_TOUCHED);
            else if (sign < 0) atomicOr(dst.err, OC_ERR_FUSE_MISSING);
          }
        }
        if (PASS == 0 || cur_blk < 0) continue;
        const size_t o = (size_t)cur_blk * OC_B3 + oc_voxel_off(i, j, k);
        if constexpr (LO) {
          const long long t = (1ll << 32) + (long long)lo_val(c);
          red_add_u64((unsigned long long*)&sums[o], (unsigned long long)(sign > 0 ? t : -t));
        } else {
          red_add_u32(&dst.cnt[o], sign > 0 ? c : 0u - c);
        }
        if (tex && sign > 0) {
          const unsigned long long cw = src.cw[e];
          if (cw) ts_red_max_u64(&dst.cw[o], cw);
        }
      }
    }
  }
  if (PASS == 1) {
    for (int o = 16; o > 0; o >>= 1) n_place += __shfl_xor_sync(0xffffffffu, n_place, o);
    if ((threadIdx.x & 31) == 0 && n_place) atomicAdd(&f.ctr[1], n_place);
  }
}

// One CTA per touched dst block: log-odds words from the sums (count > 0 ? lo_word(clamp(sum L)) : 0), the colour
// words of blocks a removal touched cleared for the recolour, and the block flagged for the trackers that exist.
template <bool LO>
__global__ void __launch_bounds__(128) k_of_commit(OcGrid g, OfDev f, const long long* __restrict__ sums, int l_min, int l_max, int* esdf_dirty,
                                                    int* fr_dirty) {
  const int nd = (int)f.ctr[3];
  for (int q = blockIdx.x; q < nd; q += gridDim.x) {
    const int blk = f.dlist[q];
    if (threadIdx.x == 0) {
      if (esdf_dirty) esdf_dirty[blk] = 1;
      if (fr_dirty) fr_dirty[blk] = 1;
    }
    const bool clear = g.cw != nullptr && (f.dflag[blk] & OF_RECOLOUR);
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
      const size_t o = (size_t)blk * OC_B3 + v;
      if constexpr (LO) {
        const long long co = sums[o];
        const long long cnt = (co + (1ll << 31)) >> 32;
        const long long sl = co - (long long)((unsigned long long)cnt << 32);
        g.cnt[o] = cnt > 0 ? lo_word((int)(sl < l_min ? l_min : (sl > l_max ? l_max : sl))) : 0u;
      }
      if (clear) g.cw[o] = 0ull;
    }
  }
}

// Textured maps: one CTA per listed source block of the submaps to recolour (addition jobs at their fused poses):
// raise the colour words of the dst blocks that a removal touched, as k_octo_fuse raises them.
template <class Rule>
__global__ void __launch_bounds__(128) k_of_recolour(OcGrid dst, OcGrid src, OfDev f, Rule rule, float vs) {
  const int nl = (int)f.ctr[0];
  unsigned long long n_col = 0;
  for (int q = blockIdx.x; q < nl; q += gridDim.x) {
    const int b = f.list[q];
    int s, bx, by, bz;
    ts_unpack_key(src.block_key[b], s, bx, by, bz);
    const FzJob& J = f.jobs[f.job_of[s].y];
    unsigned long long cur_key = TS_EMPTY;
    int cur_blk = -1;
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
      const size_t e = (size_t)b * OC_B3 + v;
      const unsigned int c = src.cnt[e];
      if (!rule.fuse_src(c)) continue;
      const unsigned long long cw = src.cw[e];
      if (!cw) continue;
      int i, j, k;
      oc_fuse_cell(J.R, J.T, bx, by, bz, v, vs, i, j, k);
      if (!ts_in_bounds(dst, i, j, k)) continue;
      const unsigned long long key = ts_pack_key(0, i >> OC_BSHIFT, j >> OC_BSHIFT, k >> OC_BSHIFT);
      if (key != cur_key) {
        cur_key = key;
        cur_blk = ts_find(dst, key);
        if (cur_blk >= 0 && !(f.dflag[cur_blk] & OF_RECOLOUR)) cur_blk = -1;
      }
      if (cur_blk < 0) continue;
      ts_red_max_u64(&dst.cw[(size_t)cur_blk * OC_B3 + oc_voxel_off(i, j, k)], cw);
      n_col++;
    }
  }
  for (int o = 16; o > 0; o >>= 1) n_col += __shfl_xor_sync(0xffffffffu, n_col, o);
  if ((threadIdx.x & 31) == 0 && n_col) atomicAdd(&f.ctr[2], n_col);
}

// ---------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------
static int of_check_args(tslam_octo* dst, tslam_octo* src, float tolerance) {
  if (!std::isfinite(tolerance) || tolerance < 0.0f) {
    ts_set_error("octo fuse_update: tolerance %g must be finite and >= 0", (double)tolerance);
    return TSLAM_E_INVALID;
  }
  if (!dst || !src) { ts_set_error("octo fuse_update: NULL handle"); return TSLAM_E_INVALID; }
  if (dst == src) { ts_set_error("octo fuse_update: dst == src (a map cannot be fused into itself)"); return TSLAM_E_INVALID; }
  return TSLAM_OK;
}

static int of_check_maps(tslam_octo* dst, tslam_octo* src) {
  if (dst->logodds != src->logodds) {
    ts_set_error("octo fuse_update: dst is a %s map and src a %s map", dst->logodds ? "log-odds" : "hit-counter", src->logodds ? "log-odds" : "hit-counter");
    return TSLAM_E_INVALID;
  }
  // (N / Nz may differ: placement tests only dst's bounds, as k_octo_fuse does - a 100 m global map of 10 m submaps)
  if (dst->cfg.max_submaps != src->cfg.max_submaps || dst->in.vs != src->in.vs || (dst->g.cw != nullptr) != (src->g.cw != nullptr)) {
    ts_set_error("octo fuse_update: dst and src differ in max_submaps (%d, %d), voxel size (%g, %g) or texture setting (%d, %d)",
                 dst->cfg.max_submaps, src->cfg.max_submaps, (double)dst->in.vs, (double)src->in.vs, dst->g.cw != nullptr, src->g.cw != nullptr);
    return TSLAM_E_INVALID;
  }
  if (src->logodds) {
    const long long lmax = std::max(-(long long)src->lo.l_min, (long long)src->lo.l_max);
    if ((long long)OF_CELL_MAX * src->cfg.max_submaps * lmax >= OF_SUM_LIMIT) {
      ts_set_error("octo fuse_update: %d x max_submaps (%d) x max(|l_min|, l_max) of src (%lld) reaches 2^30: a cell's log-odds sum could "
                   "overflow", OF_CELL_MAX, src->cfg.max_submaps, lmax);
      return TSLAM_E_INVALID;
    }
  }
  return TSLAM_OK;
}

static void of_dev(OcFuse* z, OfDev& f) {
  const size_t S = (size_t)z->dev_submaps;
  char* p = (char*)z->dev;
  f.ctr = (unsigned long long*)p; p += 8 * 8;
  f.jobs = (FzJob*)p; p += 2 * S * sizeof(FzJob);
  f.job_of = (int2*)p; p += S * 8;
  f.nblk = (int*)p; p += S * 4;
  f.rbits = (unsigned*)p; p += S * 4;
  f.dflag = (int*)p; p += (size_t)z->dev_dst_blocks * 4;
  f.dlist = (int*)p; p += (size_t)z->dev_dst_blocks * 4;
  f.list = (int*)p;
}

// dst's fusion state and device scratch for this pair of maps
static int of_open(tslam_octo* dst, tslam_octo* src, OfDev& f) {
  if (!dst->ofz) {
    dst->ofz = new OcFuse();
    OcFuse* z = dst->ofz;
    z->valid = 0;
    z->sums = nullptr;
    z->cap_blocks = 0;
    z->dev = nullptr;
    z->sub.assign(dst->cfg.max_submaps, FzSub());
  }
  OcFuse* z = dst->ofz;
  const int S = dst->cfg.max_submaps, B = src->g.max_blocks, D = dst->g.max_blocks;
  if (!z->dev || z->dev_submaps != S || z->dev_src_blocks < B || z->dev_dst_blocks != D) {
    if (z->dev) TS_CUDA(cudaFree(z->dev));
    z->dev = nullptr;
    const size_t bytes = 8 * 8 + (size_t)2 * S * sizeof(FzJob) + (size_t)S * (8 + 4 + 4) + (size_t)D * 8 + (size_t)B * 4 + 256;
    TS_CUDA(cudaMalloc(&z->dev, bytes));
    z->dev_submaps = S;
    z->dev_src_blocks = B;
    z->dev_dst_blocks = D;
  }
  of_dev(z, f);
  return TSLAM_OK;
}

// log-odds sum words for at least `need` pool blocks: grown to max(need, 2 x cap) (at most max_blocks), the old sums kept
static int of_reserve_sums(tslam_octo* m, size_t need, cudaStream_t st) {
  OcFuse* z = m->ofz;
  if (need <= z->cap_blocks) return TSLAM_OK;
  size_t cap = std::max(need, 2 * z->cap_blocks);
  if (cap > (size_t)m->g.max_blocks) cap = (size_t)m->g.max_blocks;
  long long* p = nullptr;
  const size_t bytes = cap * OC_B3 * 8;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    ts_set_error("octo fuse_update: cannot allocate %zu bytes of sum words (%zu pool blocks x 4 KiB): %s", bytes, cap, cudaGetErrorString(e));
    return TSLAM_E_CUDA;
  }
  const size_t old_n = z->cap_blocks * OC_B3, n = cap * OC_B3;
  if (old_n) TS_CUDA(cudaMemcpyAsync(p, z->sums, old_n * 8, cudaMemcpyDeviceToDevice, st));
  TS_CUDA(cudaMemsetAsync(p + old_n, 0, (n - old_n) * 8, st));
  if (z->sums) {
    TS_CUDA(cudaStreamSynchronize(st));
    TS_CUDA(cudaFree(z->sums));
  }
  z->sums = p;
  z->cap_blocks = cap;
  return TSLAM_OK;
}

// spectral-norm bound of a pose's R (Gershgorin on R^T R): how far R can stretch a vector
static double of_stretch(const float* R) {
  double worst = 0.0;
  for (int a = 0; a < 3; a++) {
    double row = 0.0;
    for (int b = 0; b < 3; b++) {
      double g = 0.0;
      for (int k = 0; k < 3; k++) g += (double)R[3 * k + a] * (double)R[3 * k + b];
      row += std::fabs(g);
    }
    worst = std::max(worst, row);
  }
  return std::sqrt(worst);
}

// upload jobs / job_of and list the source blocks of the submaps with a job
static int of_list(tslam_octo* dst, tslam_octo* src, const OfDev& f, const std::vector<FzJob>& jobs, const std::vector<int2>& job_of,
                   cudaStream_t st) {
  TS_CUDA(cudaMemsetAsync(&f.ctr[0], 0, 8, st));
  TS_CUDA(cudaMemcpyAsync(f.jobs, jobs.data(), jobs.size() * sizeof(FzJob), cudaMemcpyHostToDevice, st));
  TS_CUDA(cudaMemcpyAsync(f.job_of, job_of.data(), job_of.size() * sizeof(int2), cudaMemcpyHostToDevice, st));
  const int gl = std::max(1, std::min((src->g.max_blocks + 255) / 256, src->sm_count * 4));
  k_of_list<<<gl, 256, 0, st>>>(src->g, f);
  TS_LAUNCH_CHECK(dst);
  return TSLAM_OK;
}

static FzJob of_job(const float* R, const float* T, int sign) {
  FzJob j;
  memcpy(j.R, R, 36);
  memcpy(j.T, T, 12);
  j.sign = sign;
  j.pad = 0;
  return j;
}

// the update after its plan: splat, commit, recolour; *ctr: the device counters at the end
static int of_execute(tslam_octo* dst, tslam_octo* src, const OfDev& f, const FzPlan& P, cudaStream_t st, unsigned long long* ctr) {
  OcFuse* z = dst->ofz;
  const int S = dst->cfg.max_submaps;
  std::vector<FzJob> jobs;
  std::vector<int2> job_of(S, make_int2(-1, -1));
  for (int s = 0; s < S; s++) {
    if (P.act[s] == FZ_REMOVE || P.act[s] == FZ_MOVE) {
      job_of[s].x = (int)jobs.size();
      jobs.push_back(of_job(z->sub[s].R, z->sub[s].T, -1));
    }
    if (P.act[s] == FZ_ADD || P.act[s] == FZ_MOVE) {
      job_of[s].y = (int)jobs.size();
      jobs.push_back(of_job(&P.pR[(size_t)9 * s], &P.pT[(size_t)3 * s], 1));
    }
  }
  z->valid = 0;  // until this update completes
  if (P.full) {
    const unsigned long long gen = dst->write_gen;
    int rc = tslam_octo_reset(dst, (void*)st);  // also invalidates every tracker
    if (rc) return rc;
    dst->write_gen = gen;
    if (z->sums) TS_CUDA(cudaMemsetAsync(z->sums, 0, z->cap_blocks * OC_B3 * 8, st));
  }
  TS_CUDA(cudaMemsetAsync(f.ctr, 0, 8 * 8, st));
  TS_CUDA(cudaMemsetAsync(f.dflag, 0, (size_t)dst->g.max_blocks * 4, st));
  if (!jobs.empty()) {
    int rc = of_list(dst, src, f, jobs, job_of, st);
    if (rc) return rc;
    const int gs = dst->sm_count * 8;
    if (P.n_add + P.n_move > 0) {
      oc_with_rule(dst, [&](auto rule) { k_of_splat<0><<<gs, 128, 0, st>>>(dst->g, src->g, f, nullptr, rule, dst->in.vs); });
      TS_LAUNCH_CHECK(dst);
    }
    int nb = 0, err = 0;
    TS_CUDA(cudaMemcpyAsync(&nb, dst->g.n_blocks, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaMemcpyAsync(&err, dst->g.err, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
    if (err & (TS_ERR_POOL_FULL | TS_ERR_TABLE_FULL)) return oc_deferred(dst);  // nothing was added; the next update is full
    if (dst->logodds) {
      rc = of_reserve_sums(dst, (size_t)std::min(nb, dst->g.max_blocks), st);
      if (rc) return rc;
    }
    oc_with_rule(dst, [&](auto rule) { k_of_splat<1><<<gs, 128, 0, st>>>(dst->g, src->g, f, z->sums, rule, dst->in.vs); });
    TS_LAUNCH_CHECK(dst);
    const int gc = dst->sm_count * 8;
    if (dst->logodds)
      k_of_commit<true><<<gc, 128, 0, st>>>(dst->g, f, z->sums, dst->lo.l_min, dst->lo.l_max, dst->esdf_dirty, dst->fr_dirty);
    else
      k_of_commit<false><<<gc, 128, 0, st>>>(dst->g, f, nullptr, 0, 0, dst->esdf_dirty, dst->fr_dirty);
    TS_LAUNCH_CHECK(dst);
  }
  // Recolour: the blocks removals touched lost their colour words; the included submaps whose placed bounding sphere
  // can reach such a block raise them again at their fused poses.  A submap placed at (R, T) with radius r puts its
  // voxels into cells within r |R| + (sqrt 3 / 2) vs of T, and two cells of one 8^3 block are at most 7 sqrt 3 vs apart.
  if (dst->g.cw && P.n_remove + P.n_move > 0) {
    const double vs = (double)dst->in.vs;
    std::vector<double> rc_c, rc_r;  // centre and reach of every removal
    for (int s = 0; s < S; s++)
      if (P.act[s] == FZ_REMOVE || P.act[s] == FZ_MOVE) {
        for (int a = 0; a < 3; a++) rc_c.push_back(z->sub[s].T[a]);
        rc_r.push_back((double)P.rad[s] * of_stretch(z->sub[s].R));
      }
    jobs.clear();
    std::fill(job_of.begin(), job_of.end(), make_int2(-1, -1));
    for (int s = 0; s < S; s++) {
      const float *R = nullptr, *T = nullptr;
      if (P.act[s] == FZ_ADD || P.act[s] == FZ_MOVE) { R = &P.pR[(size_t)9 * s]; T = &P.pT[(size_t)3 * s]; }
      else if (P.act[s] == FZ_KEEP) { R = z->sub[s].R; T = z->sub[s].T; }
      if (!R) continue;
      const double reach = (double)P.rad[s] * of_stretch(R);
      bool near = false;
      for (size_t q = 0; q < rc_r.size() && !near; q++) {
        const double dx = (double)T[0] - rc_c[3 * q], dy = (double)T[1] - rc_c[3 * q + 1], dz = (double)T[2] - rc_c[3 * q + 2];
        const double slack = 1e-5 * (reach + rc_r[q] + std::fabs((double)T[0]) + std::fabs((double)T[1]) + std::fabs((double)T[2]) +
                                     std::fabs(rc_c[3 * q]) + std::fabs(rc_c[3 * q + 1]) + std::fabs(rc_c[3 * q + 2]));
        near = std::sqrt(dx * dx + dy * dy + dz * dz) <= reach + rc_r[q] + 9.0 * std::sqrt(3.0) * vs + slack;
      }
      if (!near) continue;
      job_of[s].y = (int)jobs.size();
      jobs.push_back(of_job(R, T, 1));
    }
    if (!jobs.empty()) {
      int rc = of_list(dst, src, f, jobs, job_of, st);
      if (rc) return rc;
      oc_with_rule(dst, [&](auto rule) { k_of_recolour<<<dst->sm_count * 8, 128, 0, st>>>(dst->g, src->g, f, rule, dst->in.vs); });
      TS_LAUNCH_CHECK(dst);
    }
  }
  TS_CUDA(cudaMemcpyAsync(ctr, f.ctr, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  return TSLAM_OK;
}

extern "C" int tslam_octo_fuse_update(tslam_octo_t* dst, tslam_octo_t* src, const uint8_t* include, float tolerance, int32_t full,
                                      int64_t* stats8, void* stream) {
  int rc = of_check_args(dst, src, tolerance);
  if (rc) return rc;
  rc = of_check_maps(dst, src);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  TS_CUDA(cudaStreamSynchronize(st));
  rc = oc_deferred(dst);  // an error of earlier work on dst is reported before anything is written
  if (rc) return rc;
  OfDev f;
  rc = of_open(dst, src, f);
  if (rc) return rc;
  OcFuse* z = dst->ofz;
  int reason = FZ_INCR;
  if (full) reason = FZ_ASKED;
  else if (!z->valid) reason = FZ_FIRST;
  else if (z->src_serial != src->serial) reason = FZ_OTHER_SRC;
  else if (z->gen != dst->write_gen) reason = FZ_DST_WRITTEN;

  // plan: source blocks and radius per submap, dst's pose table
  const int S = dst->cfg.max_submaps;
  TS_CUDA(cudaMemsetAsync(f.nblk, 0, (size_t)S * 8, st));  // nblk and rbits
  k_of_plan<<<src->sm_count * 4, 256, 0, st>>>(src->g, src->in.vs, f);
  TS_LAUNCH_CHECK(dst);
  FzPlan P;
  P.nblk.assign(S, 0);
  P.rad.assign(S, 0.0f);
  P.pR.assign((size_t)S * 9, 0.0f);
  P.pT.assign((size_t)S * 3, 0.0f);
  P.ghosts = 0;
  TS_CUDA(cudaMemcpyAsync(P.nblk.data(), f.nblk, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(P.rad.data(), f.rbits, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(P.pR.data(), dst->pose_R, (size_t)S * 36, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(P.pT.data(), dst->pose_T, (size_t)S * 12, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  reason = fz_decide(P, z->sub, src->content_ver, include, tolerance, reason);
  fz_settle(P, reason == FZ_INCR && P.cost > P.cost_full ? FZ_COST : reason);

  unsigned long long ctr[8] = {0};
  rc = of_execute(dst, src, f, P, st, ctr);
  if (rc) return rc;
  rc = oc_deferred(dst);  // a removal that found no block (OC_ERR_FUSE_MISSING): the sums stay invalid
  if (rc) return rc;
  fz_record_subs(z->sub, P, src->content_ver);
  z->valid = 1;
  z->src_serial = src->serial;
  z->gen = dst->write_gen;
  if (stats8) {
    stats8[0] = P.reason;
    stats8[1] = P.n_add;
    stats8[2] = P.n_move;
    stats8[3] = P.n_remove;
    stats8[4] = P.n_tol;
    stats8[5] = (int64_t)ctr[1];
    stats8[6] = (int64_t)ctr[2];
    stats8[7] = (int64_t)ctr[3];
  }
  return TSLAM_OK;
}
