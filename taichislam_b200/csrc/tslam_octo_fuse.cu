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
// An update plans and lists the source blocks of the submaps with work as the TSDF's does (tslam_fuse_plan.cuh: the
// plan rule, fusion state, scratch, sum storage, k_fz_plan / k_fz_list and the host steps around them), activates the
// dst blocks the additions need (k_of_splat<0>), grows the sum words to the pool blocks in use (log-odds), adds the
// signed terms (k_of_splat<1>), reads the touched blocks out of the sums and flags them for the trackers
// (k_of_commit), and on textured maps recolours the blocks removals touched (k_fz_list + k_of_recolour).
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

// Device scratch of one update.  ctr: [0] list length, [1] source voxels placed, [2] voxels recoloured, [3] touched dst
// blocks.
struct OfDev : FzDev {
  int* dflag;         // [dst max_blocks] OF_TOUCHED | OF_RECOLOUR
  int* dlist;         // [dst max_blocks] touched dst blocks
  void carve_tail(FzCarve& c, int D) {
    dflag = c.take<int>(D);
    dlist = c.take<int>(D);
  }
};

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
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

// the update after its plan: splat, commit, recolour; *ctr: the device counters at the end
static int of_execute(tslam_octo* dst, tslam_octo* src, const OfDev& f, const FzPlan& P, cudaStream_t st, unsigned long long* ctr) {
  FzState* z = dst->fz;
  const int S = dst->cfg.max_submaps;
  const FzJobs J = fz_jobs(P, z->sub);
  z->valid = 0;  // until this update completes
  if (P.full) {
    const unsigned long long gen = dst->ver.write_gen;
    int rc = tslam_octo_reset(dst, (void*)st);  // also invalidates every tracker
    if (rc) return rc;
    dst->ver.write_gen = gen;
    if (z->sums) TS_CUDA(cudaMemsetAsync(z->sums, 0, z->cap_blocks * OC_B3 * 8, st));
  }
  TS_CUDA(cudaMemsetAsync(f.dflag, 0, (size_t)dst->g.max_blocks * 4, st));
  if (!J.jobs.empty()) {
    int rc = fz_list(dst, src, f, J, st);
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
      rc = fz_reserve_sums(*z, (size_t)std::min(nb, dst->g.max_blocks), (size_t)dst->g.max_blocks, OC_B3, 1, "octo fuse_update", st);
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
    FzJobs RJ(S);
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
      if (near) RJ.add(s, R, T, 1);
    }
    if (!RJ.jobs.empty()) {
      TS_CUDA(cudaMemsetAsync(&f.ctr[0], 0, 8, st));  // (the list of the splat is done with)
      int rc = fz_list(dst, src, f, RJ, st);
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
  int rc = fz_check_args(dst, src, tolerance, "octo fuse_update");
  if (rc) return rc;
  rc = of_check_maps(dst, src);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  TS_CUDA(cudaStreamSynchronize(st));
  rc = oc_deferred(dst);  // an error of earlier work on dst is reported before anything is written
  if (rc) return rc;
  OfDev f;
  rc = fz_open(dst->fz, dst->cfg.max_submaps, src->g.max_blocks, dst->g.max_blocks, f);
  if (rc) return rc;
  FzState* z = dst->fz;
  const int reason = fz_reason(*z, full, FZ_FIRST, src->ver.serial, z->gen != dst->ver.write_gen);
  FzPlan P;
  rc = fz_plan(dst, src, f, include, tolerance, reason, st, P);
  if (rc) return rc;
  fz_settle(P, P.reason == FZ_INCR && P.cost > P.cost_full ? FZ_COST : P.reason);

  unsigned long long ctr[8] = {0};
  rc = of_execute(dst, src, f, P, st, ctr);
  if (rc) return rc;
  rc = oc_deferred(dst);  // a removal that found no block (OC_ERR_FUSE_MISSING): the sums stay invalid
  if (rc) return rc;
  fz_record(*z, P, src->ver);
  z->gen = dst->ver.write_gen;
  fz_stats(P, (int64_t)ctr[1], (int64_t)ctr[2], (int64_t)ctr[3], stats8);
  return TSLAM_OK;
}
