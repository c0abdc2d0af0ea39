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
// An update plans and lists the source blocks of the submaps with work as the Octomap's does (tslam_fuse_plan.cuh: the
// plan rule, fusion state, scratch, sum storage, k_fz_plan / k_fz_list and the host steps around them), activates the
// dst blocks the additions need (k_fz_splat<0>), grows the sum planes to the pool blocks in use, splats
// (k_fz_splat<1>: removals at the old pose, additions at the new one) and reads the touched blocks out of the sums
// (k_fz_commit), stamping them for the incremental mesh and the ESDF.
//
// Tiled global maps (tslam_tsdf_fuse_update_tiled_*, DESIGN.md section 6) run the same plan, splat and commit per rank:
// the sums of a block live on its owner, the other ranks pack the sum rows of their foreign blocks (k_fz_pack) and the
// owner adds them (k_fz_unpack_add).  The terms are the same multiset per voxel, so the bounds above carry over and the
// union of the tiles is bit for bit the single map's.
#include <cmath>
#include <cstring>
#include <vector>
#include "tslam_internal.cuh"
#include "tslam_fuse_plan.cuh"

#define FZ_Q 16777216.0             // 2^24: quantum of the sums
#define FZ_FMAX 8388608.0f          // 2^23: terms at or above this magnitude are skipped
#define TS_ERR_FUSE_MISSING 16      // g.err: a removal found no dst block (the sums and the pool disagree)

struct FzSums {       // sum planes, [cap blocks * 4096] int64 each
  long long* wt;      // S_wT
  long long* w;       // S_w
  long long* co;      // count << 32 + S_occ
  long long* c;       // textured maps: 3 planes S_c (c + p * stride), else null
  size_t stride;      // elements per plane
};
// Device scratch of one update.  ctr: [0] list length, [1] voxels splatted, [2] voxels skipped, [3] dst ghost blocks,
// [4] dirty blocks, [5] voxels whose count decodes as negative (tiled updates).
struct TsDev : FzDev {
  TsTiling* tiling;   // a tiled update's tiling (k_fz_splat indexes its cuts: as a kernel parameter they would be
                      // copied to the stack)
  void carve_tail(FzCarve& c, int) { tiling = c.take<TsTiling>(1); }
};

// (FzState::gen of a tiled update: write_gen - ghost_gen, as ghost imports are not writes of dst's own content)
struct TsFuse : FzState {
  // tiled updates (tslam_tsdf_fuse_update_tiled_*)
  int ever_valid;     // the sums were valid once: invalid sums read "sums not valid", not "first call"
  int tiled;          // the last update was tiled, with this tiling (world 0 for a single-map update)
  TsTiling tiling;
  int phase;          // of the update in progress: 0 none, 1 planned, 2 splatted, 3 packed, 4 unpacked
  FzPlan plan;        // its plan (phase >= 1), source handle and the tiling it packs with
  unsigned long long plan_src;
  TsTiling plan_tiling;
};

static unsigned long long g_serial = 0;  // handle numbers (create is not called concurrently with itself here)

void fz_ver_init(FzVer& v, int max_submaps) {
  v.serial = __atomic_add_fetch(&g_serial, 1ull, __ATOMIC_RELAXED);
  v.write_gen = 0;
  v.content_ver = new unsigned long long[max_submaps]();
  v.n = max_submaps;
}

void fz_ver_free(FzVer& v) {
  delete[] v.content_ver;
  v.content_ver = nullptr;
}

void fz_written(FzVer& v, int submap) {
  v.write_gen++;
  if (!v.content_ver) return;
  if (submap < 0) {
    for (int s = 0; s < v.n; s++) v.content_ver[s]++;
  } else if (submap < v.n) {
    v.content_ver[submap]++;
  }
}

void ts_fuse_free(tslam_tsdf* m) { fz_free(m->fz); }

TsFuseView ts_fuse_view(tslam_tsdf* m) {
  TsFuseView v = {nullptr, 0, m->g.col ? 6 : 3, 0, 0};
  if (m->fz) {
    v.sums = m->fz->sums;
    v.cap_blocks = v.sums ? m->fz->cap_blocks : 0;
    v.valid = m->fz->valid;
    v.phase = m->fz->phase;
  }
  return v;
}

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
__device__ __forceinline__ bool fz_term_ok(float x) { return fabsf(x) < FZ_FMAX; }  // false for NaN and +-inf too
__device__ __forceinline__ long long fz_q(float x) { return __double2ll_rn((double)x * FZ_Q); }

// One CTA per listed source block.  PASS 0 activates the dst blocks of the additions; PASS 1 adds each job's signed
// terms into the sum planes (removals find their blocks, or raise TS_ERR_FUSE_MISSING) and flags the blocks it touched.
// the block of cell (ci, cj, ck) lies in a foreign tile (not inlined: inlined, the cut search costs k_fz_splat<0> spills)
__device__ __noinline__ bool fz_foreign(const TsTiling* tl, int ci, int cj, int ck) {
  return tile_owner(*tl, ci >> TS_BSHIFT, cj >> TS_BSHIFT, ck >> TS_BSHIFT) != tl->rank;
}
// On a tiled map (tl: its tiling, in device memory; null otherwise) PASS 0 also activates the foreign blocks of removals: their negative terms travel to the
// owner as deltas.  A removal never activates a block of this rank's own tile, which must already hold it.
template <int PASS>
__global__ void __launch_bounds__(256) k_fz_splat(TsGrid dst, TsGrid src, FzDev f, FzSums S, float vs, const TsTiling* tl) {
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
      if (PASS == 0 && sign < 0 && !tl) continue;
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
              if (sign > 0 || fz_foreign(tl, ci, cj, ck)) cur_blk = ts_get_or_alloc_cached(dst, key);
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

// ---- tiled updates: the sums of foreign blocks travel to their owner as deltas --------------------------------------
// One CTA per pool block: a dirty block of a foreign tile (ghost or not) copies its sum rows into the slot group of its
// owner (row = key, then planes x 4096 int64 in plane order S_wT, S_w, co, S_c[3]), zeroes them and drops its flag.
__global__ void __launch_bounds__(256) k_fz_pack(TsGrid g, TsTiling t, FzSums S, int planes, const int* offsets, int* cursor, long long cap,
                                                  long long* rows) {
  __shared__ long long s_slot;
  const int nb = min(*g.n_blocks, g.max_blocks);
  const long long rl = 1 + (long long)planes * TS_B3;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (!g.dirty_flag[b]) continue;  // uniform per CTA
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    const int o = tile_owner(t, bx, by, bz);
    if (o == t.rank) continue;
    __syncthreads();
    if (threadIdx.x == 0) {
      s_slot = (long long)offsets[o] + atomicAdd(&cursor[o], 1);
      if (s_slot < cap) rows[s_slot * rl] = (long long)g.block_key[b];
      g.dirty_flag[b] = 0;  // not ours: never committed here
    }
    __syncthreads();
    const long long slot = s_slot;
    for (int p = 0; p < planes; p++) {
      long long* sp = S.wt + (size_t)p * S.stride + (size_t)b * TS_B3;
      for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
        if (slot < cap) rows[slot * rl + 1 + (long long)p * TS_B3 + v] = sp[v];
        sp[v] = 0;
      }
    }
  }
}

// the owner activates the received blocks (one thread per row) ...
__global__ void __launch_bounds__(256) k_fz_unpack_alloc(TsGrid g, long long n, long long rl, const long long* rows) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x)
    ts_get_or_alloc(g, (unsigned long long)rows[q * rl]);
}

// ... and, once its sum planes cover them, adds the rows with wrapping int64 adds (several ranks may send the same block)
// and flags the blocks for the commit.  One CTA per row.
__global__ void __launch_bounds__(256) k_fz_unpack_add(TsGrid g, FzSums S, int planes, long long n, const long long* rows) {
  const long long rl = 1 + (long long)planes * TS_B3;
  for (long long q = blockIdx.x; q < n; q += gridDim.x) {
    const long long* row = rows + q * rl;
    const int blk = ts_find(g, (unsigned long long)row[0]);
    if (blk < 0) continue;  // (not activated: the pool ran out, which the allocation pass reported)
    if (threadIdx.x == 0) ts_mark_dirty(g, blk);
    for (int p = 0; p < planes; p++) {
      unsigned long long* sp = (unsigned long long*)(S.wt + (size_t)p * S.stride + (size_t)blk * TS_B3);
      for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
        const long long x = row[1 + (long long)p * TS_B3 + v];
        if (x) red_add_u64(sp + v, (unsigned long long)x);
      }
    }
  }
}

// voxels of the dirty blocks whose contribution count decodes as negative: the sums of the ranks disagree
__global__ void __launch_bounds__(256) k_fz_negative(TsGrid g, FzSums S, unsigned long long* bad) {
  const int nd = *g.n_dirty;
  unsigned long long n = 0;
  for (int q = blockIdx.x; q < nd; q += gridDim.x) {
    const long long* co = S.co + (size_t)g.dirty_list[q] * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) n += ((co[v] + (1ll << 31)) >> 32) < 0;
  }
  if (n) atomicAdd(bad, n);
}

// ---------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------
static int fz_planes(const tslam_tsdf* m) { return m->g.col ? 6 : 3; }

static FzSums fz_sums(const TsFuse* z, int planes) {
  FzSums S;
  const size_t n = z->cap_blocks * TS_B3;
  long long* p = z->sums;
  S.stride = n;
  S.wt = p;
  S.w = p + n;
  S.co = p + 2 * n;
  S.c = planes == 6 ? p + 3 * n : nullptr;
  return S;
}

// sum planes for at least `need` pool blocks (fz_reserve_sums)
static int fz_reserve_planes(tslam_tsdf* m, size_t need, cudaStream_t st) {
  return fz_reserve_sums(*m->fz, need, (size_t)m->g.max_blocks, TS_B3, fz_planes(m), "fuse_update", st);
}

static int fz_check_maps(tslam_tsdf* dst, tslam_tsdf* src) {
  if (!dst->cfg.is_global_map) { ts_set_error("fuse_update: dst is not a global map (is_global_map = 0)"); return TSLAM_E_INVALID; }
  if (dst->cfg.max_submaps != src->cfg.max_submaps || dst->in.vs != src->in.vs || (dst->g.col != nullptr) != (src->g.col != nullptr)) {
    ts_set_error("fuse_update: dst and src differ in max_submaps (%d, %d), voxel size (%g, %g) or texture setting (%d, %d)", dst->cfg.max_submaps,
                 src->cfg.max_submaps, (double)dst->in.vs, (double)src->in.vs, dst->g.col != nullptr, src->g.col != nullptr);
    return TSLAM_E_INVALID;
  }
  return TSLAM_OK;
}

// flush both maps' pending work, then dst's fusion state and device scratch (fz_open)
static int fz_begin(tslam_tsdf* dst, tslam_tsdf* src, cudaStream_t st, TsDev& f) {
  int rc = ts_flush_pending(src, st);
  if (rc) return rc;
  rc = ts_flush_pending(dst, st);
  if (rc) return rc;
  return fz_open(dst->fz, dst->cfg.max_submaps, src->g.max_blocks, 0, f);
}

// Splat the plan into the sums: a full update resets dst and zeroes the sums first.  Tiled (t: the tiling, else null):
// removals also activate their foreign blocks.  Invalidates the sums until the update is recorded.
static int fz_execute(tslam_tsdf* dst, tslam_tsdf* src, const TsDev& f, const FzPlan& P, const TsTiling* t, cudaStream_t st) {
  TsFuse* z = dst->fz;
  const FzJobs J = fz_jobs(P, z->sub);
  const int planes = fz_planes(dst);
  z->valid = 0;  // until this update completes
  if (P.full) {
    const unsigned long long gen = dst->ver.write_gen;
    int rc = tslam_tsdf_reset(dst, (void*)st);  // also compacts the pool: blocks left empty by removals are dropped
    if (rc) return rc;
    dst->ver.write_gen = gen;
    // every plane in full: a reset of dst since the last update left the pool empty but not the sums (at most 2x the
    // blocks in use: the planes grow geometrically)
    if (z->sums) TS_CUDA(cudaMemsetAsync(z->sums, 0, z->cap_blocks * TS_B3 * 8 * planes, st));
  }
  if (!J.jobs.empty()) {
    int rc = fz_list(dst, src, f, J, st);
    if (rc) return rc;
    const int gs = dst->sm_count * 8;
    if (P.n_add + P.n_move > 0 || (t && P.n_remove > 0)) {
      TsTiling* td = nullptr;
      if (t) {
        td = f.tiling;
        TS_CUDA(cudaMemcpyAsync(td, t, sizeof(TsTiling), cudaMemcpyHostToDevice, st));
      }
      k_fz_splat<0><<<gs, 256, 0, st>>>(dst->g, src->g, f, FzSums{}, dst->in.vs, td);
      TS_LAUNCH_CHECK(dst);
    }
    int nb = 0, err = 0;
    TS_CUDA(cudaMemcpyAsync(&nb, dst->g.n_blocks, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaMemcpyAsync(&err, dst->g.err, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
    if (err) return ts_check_deferred(dst);  // pool exhausted: nothing was added; the next update is a full one
    rc = fz_reserve_planes(dst, (size_t)std::min(nb, dst->g.max_blocks), st);
    if (rc) return rc;
    k_fz_splat<1><<<gs, 256, 0, st>>>(dst->g, src->g, f, fz_sums(z, planes), dst->in.vs, nullptr);
    TS_LAUNCH_CHECK(dst);
  }
  return TSLAM_OK;
}

// Read the dirty blocks out of the sums (ctr[4] = their number); tiled updates first count the voxels whose count
// decodes as negative (ctr[5]).  Then the error words: a removal that found no block, inconsistent sums, device flags.
static int fz_commit(tslam_tsdf* dst, const FzDev& f, bool check_negative, cudaStream_t st, unsigned long long* ctr) {
  TsFuse* z = dst->fz;
  const int planes = fz_planes(dst);
  int rc = ts_collect_dirty(dst, st);
  if (rc) return rc;
  TS_CUDA(cudaMemcpyAsync(&f.ctr[4], dst->g.n_dirty, 4, cudaMemcpyDeviceToDevice, st));
  if (z->sums) {
    if (check_negative) {
      k_fz_negative<<<dst->sm_count * 4, 256, 0, st>>>(dst->g, fz_sums(z, planes), &f.ctr[5]);
      TS_LAUNCH_CHECK(dst);
    }
    const unsigned long long seq = ++dst->commit_seq;  // stamp of every block this update writes (incremental mesh)
    k_fz_commit<<<dst->sm_count * 4, 256, 0, st>>>(dst->g, fz_sums(z, planes), dst->blk_stamp, seq);
    TS_LAUNCH_CHECK(dst);
  }
  TS_CUDA(cudaMemsetAsync(dst->g.n_dirty, 0, 4, st));
  int err = 0;
  TS_CUDA(cudaMemcpyAsync(ctr, f.ctr, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(&err, dst->g.err, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (err & TS_ERR_FUSE_MISSING) {
    const int rest = err & ~TS_ERR_FUSE_MISSING;
    TS_CUDA(cudaMemcpy(dst->g.err, &rest, 4, cudaMemcpyHostToDevice));
    ts_set_error("fuse_update: a removal found no block of dst (its sums and pool disagree); the next update is a full one");
    return TSLAM_E_CUDA;
  }
  if (ctr[5]) {
    ts_set_error("fuse_update: %llu voxels of dst decode a negative contribution count (the ranks' sums disagree); the next update is a full "
                 "one", ctr[5]);
    return TSLAM_E_CUDA;
  }
  return ts_check_deferred(dst);
}

// the submaps' new state after a successful update
static void ts_fz_record(tslam_tsdf* dst, tslam_tsdf* src, const FzPlan& P) {
  fz_record(*dst->fz, P, src->ver);
  // voxels that lose their last contribution become unobserved, which the incremental ESDF does not undo
  if (P.n_remove + P.n_move > 0) dst->esdf_full_needed = 1;
  dst->fz->ever_valid = 1;
}

// stats8 of a completed update: voxels splatted, skipped, blocks committed
static void ts_fz_stats(const FzPlan& P, const unsigned long long* ctr, int64_t* stats8) {
  fz_stats(P, (int64_t)ctr[1], (int64_t)ctr[2], (int64_t)(unsigned)ctr[4], stats8);
}

extern "C" int tslam_tsdf_fuse_update(tslam_tsdf_t* dst, tslam_tsdf_t* src, const uint8_t* include, float tolerance, int32_t full,
                                      int64_t* stats8, void* stream) {
  int rc = fz_check_args(dst, src, tolerance, "fuse_update");
  if (rc) return rc;
  rc = fz_check_maps(dst, src);
  if (rc) return rc;
  if (dst->tile_cuts_set) { ts_set_error("fuse_update: dst is a tiled map (tile cuts set): not supported"); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  TsDev f;
  rc = fz_begin(dst, src, st, f);
  if (rc) return rc;
  TsFuse* z = dst->fz;
  // (the sums of a tiled update hold one tile)
  const int reason = fz_reason(*z, full, FZ_FIRST, src->ver.serial, z->gen != dst->ver.write_gen || z->tiled);
  FzPlan P;
  rc = fz_plan(dst, src, f, include, tolerance, reason, st, P);
  if (rc) return rc;
  if (P.ghosts > 0) { ts_set_error("fuse_update: dst holds %llu ghost blocks (a tiled map): not supported", P.ghosts); return TSLAM_E_INVALID; }
  fz_settle(P, P.reason == FZ_INCR && P.cost > P.cost_full ? FZ_COST : P.reason);
  rc = fz_execute(dst, src, f, P, nullptr, st);
  if (rc) return rc;
  unsigned long long ctr[8];
  rc = fz_commit(dst, f, false, st, ctr);
  if (rc) return rc;
  ts_fz_record(dst, src, P);
  z->gen = dst->ver.write_gen;
  z->tiled = 0;
  ts_fz_stats(P, ctr, stats8);
  return TSLAM_OK;
}

// ---------------------------------------------------------------------------
// tiled updates (DESIGN.md section 6, "Incremental tiled fusion"; include/tslam.h)
// ---------------------------------------------------------------------------
static const char* const FZ_PHASE[] = {"none", "plan", "splat", "pack", "unpack"};

static int fz_phase(tslam_tsdf* dst, int want, const char* what) {
  const int ph = dst->fz ? dst->fz->phase : 0;
  if (ph != want) {
    ts_set_error("%s: called out of order (the last phase of this update was '%s', this call follows '%s')", what, FZ_PHASE[ph], FZ_PHASE[want]);
    return TSLAM_E_INVALID;
  }
  return TSLAM_OK;
}

// tiles3 / rank / world checks that need no handle (fill_tiling repeats them with the map's cuts)
static int fz_check_tiles(const int32_t* tiles3, int32_t rank, int32_t world) {
  if (!tiles3 || world < 1 || world > 24 || rank < 0 || rank >= world || tiles3[0] < 1 || tiles3[1] < 1 || tiles3[2] < 1 ||
      tiles3[0] > TS_MAX_TILES_AXIS || tiles3[1] > TS_MAX_TILES_AXIS || tiles3[2] > TS_MAX_TILES_AXIS || tiles3[0] * tiles3[1] * tiles3[2] != world) {
    ts_set_error("fuse_update_tiled: bad tiling %d x %d x %d for rank %d of world %d (1 <= world <= 24)", tiles3 ? tiles3[0] : -1, tiles3 ? tiles3[1] : -1,
                 tiles3 ? tiles3[2] : -1, rank, world);
    return TSLAM_E_INVALID;
  }
  return TSLAM_OK;
}

static int fz_tiling(tslam_tsdf* m, const int32_t* tiles3, int32_t rank, int32_t world, TsTiling* t) {
  memset(t, 0, sizeof(*t));  // (the tiling is compared bytewise)
  return fill_tiling(m, tiles3, rank, world, t);
}

extern "C" int tslam_tsdf_fuse_update_tiled_plan(tslam_tsdf_t* dst, tslam_tsdf_t* src, const int32_t* tiles3, int32_t rank, int32_t world,
                                                 const uint8_t* include, float tolerance, int32_t full, int64_t* plan3, uint8_t* present,
                                                 void* stream) {
  int rc = fz_check_args(dst, src, tolerance, "fuse_update");
  if (rc) return rc;
  if (!plan3 || !present) { ts_set_error("fuse_update_tiled_plan: NULL plan3 or present"); return TSLAM_E_INVALID; }
  rc = fz_check_tiles(tiles3, rank, world);
  if (rc) return rc;
  rc = fz_check_maps(dst, src);
  if (rc) return rc;
  TsTiling t;
  rc = fz_tiling(dst, tiles3, rank, world, &t);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  TsDev f;
  rc = fz_begin(dst, src, st, f);
  if (rc) return rc;
  TsFuse* z = dst->fz;
  if (z->phase >= 2) z->valid = 0;  // an update abandoned after its splat left the sums part-way
  z->phase = 0;
  // owned content written; ghost imports are not
  int reason = fz_reason(*z, full, z->ever_valid ? FZ_INVALID : FZ_FIRST, src->ver.serial, z->gen != dst->ver.write_gen - dst->ghost_gen);
  if (reason == FZ_INCR && (!z->tiled || memcmp(&z->tiling, &t, sizeof(t)))) reason = FZ_CUTS;
  rc = fz_plan(dst, src, f, include, tolerance, reason, st, z->plan);
  if (rc) return rc;
  const FzPlan& P = z->plan;
  for (int s = 0; s < dst->cfg.max_submaps; s++) present[s] = P.nblk[s] > 0;
  plan3[0] = P.reason;
  plan3[1] = P.cost;
  plan3[2] = P.cost_full;
  z->plan_src = src->ver.serial;
  z->plan_tiling = t;
  z->phase = 1;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_fuse_update_tiled_splat(tslam_tsdf_t* dst, tslam_tsdf_t* src, int32_t reason, void* stream) {
  if (!dst || !src) { ts_set_error("fuse_update_tiled_splat: NULL handle"); return TSLAM_E_INVALID; }
  if (reason < FZ_INCR || reason > FZ_INVALID) { ts_set_error("fuse_update_tiled_splat: reason %d outside [0, 8]", reason); return TSLAM_E_INVALID; }
  int rc = fz_phase(dst, 1, "fuse_update_tiled_splat");
  if (rc) return rc;
  TsFuse* z = dst->fz;
  if (src->ver.serial != z->plan_src) { ts_set_error("fuse_update_tiled_splat: src is not the map the update was planned with"); return TSLAM_E_INVALID; }
  if (reason == FZ_INCR && z->plan.reason != FZ_INCR) {
    ts_set_error("fuse_update_tiled_splat: an incremental update where this rank's plan is full (reason %d)", z->plan.reason);
    return TSLAM_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  TsDev f;
  fz_dev(*z, f);  // (the plan sized it for src)
  fz_settle(z->plan, reason);
  z->phase = 2;  // (from here on a failure leaves the sums invalid)
  return fz_execute(dst, src, f, z->plan, &z->plan_tiling, st);
}

extern "C" int tslam_tsdf_fuse_update_tiled_pack(tslam_tsdf_t* dst, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts,
                                                 int64_t cap, int64_t* rows, void* stream) {
  if (!dst || !counts || cap < 0 || (cap && !rows)) { ts_set_error("fuse_update_tiled_pack: NULL handle, counts or rows, or cap < 0"); return TSLAM_E_INVALID; }
  int rc = fz_check_tiles(tiles3, rank, world);
  if (rc) return rc;
  rc = fz_phase(dst, 2, "fuse_update_tiled_pack");
  if (rc) return rc;
  TsFuse* z = dst->fz;
  TsTiling t;
  rc = fz_tiling(dst, tiles3, rank, world, &t);
  if (rc) return rc;
  if (!z->plan.full && memcmp(&t, &z->plan_tiling, sizeof(t))) {
    ts_set_error("fuse_update_tiled_pack: the tiling changed during an incremental update (only a full update may move the cuts)");
    return TSLAM_E_INVALID;
  }
  int h_off[24];
  long long tot = 0;
  for (int r = 0; r < world; r++) {
    h_off[r] = (int)tot;
    tot += counts[r] < 0 ? 0 : counts[r];
  }
  if (tot > cap) { ts_set_error("fuse_update_tiled_pack: %lld blocks to send, capacity %lld", tot, (long long)cap); return TSLAM_E_CAPACITY; }
  cudaStream_t st = (cudaStream_t)stream;
  if (z->sums) {
    int* d_off = dst->scratch_i + 16;
    int* d_cur = dst->scratch_i + 40;
    TS_CUDA(cudaMemcpyAsync(d_off, h_off, world * sizeof(int), cudaMemcpyHostToDevice, st));
    TS_CUDA(cudaMemsetAsync(d_cur, 0, 24 * sizeof(int), st));
    const int planes = fz_planes(dst);
    k_fz_pack<<<dst->sm_count * 4, 256, 0, st>>>(dst->g, t, fz_sums(z, planes), planes, d_off, d_cur, cap, (long long*)rows);
    TS_LAUNCH_CHECK(dst);
    TS_CUDA(cudaStreamSynchronize(st));  // h_off is on the stack
  }
  z->plan_tiling = t;
  z->phase = 3;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_fuse_update_tiled_unpack(tslam_tsdf_t* dst, int64_t n, const int64_t* rows, void* stream) {
  if (!dst || n < 0 || (n && !rows)) { ts_set_error("fuse_update_tiled_unpack: NULL handle or rows, or n < 0"); return TSLAM_E_INVALID; }
  int rc = fz_phase(dst, 3, "fuse_update_tiled_unpack");
  if (rc) return rc;
  TsFuse* z = dst->fz;
  cudaStream_t st = (cudaStream_t)stream;
  TsDev f;
  fz_dev(*z, f);
  const int planes = fz_planes(dst);
  if (n > 0) {
    const long long rl = 1 + (long long)planes * TS_B3;
    k_fz_unpack_alloc<<<(int)std::min<long long>((n + 255) / 256, dst->sm_count * 4), 256, 0, st>>>(dst->g, n, rl, (const long long*)rows);
    TS_LAUNCH_CHECK(dst);
    int nb = 0, err = 0;
    TS_CUDA(cudaMemcpyAsync(&nb, dst->g.n_blocks, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaMemcpyAsync(&err, dst->g.err, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
    if (err & ~TS_ERR_FUSE_MISSING) return ts_check_deferred(dst);  // pool exhausted on the owner
    rc = fz_reserve_planes(dst, (size_t)std::min(nb, dst->g.max_blocks), st);
    if (rc) return rc;
    k_fz_unpack_add<<<(int)std::min<long long>(n, dst->sm_count * 4), 256, 0, st>>>(dst->g, fz_sums(z, planes), planes, n, (const long long*)rows);
    TS_LAUNCH_CHECK(dst);
  }
  unsigned long long ctr[8];
  rc = fz_commit(dst, f, true, st, ctr);
  if (rc) return rc;
  z->phase = 4;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_fuse_update_tiled_finish(tslam_tsdf_t* dst, tslam_tsdf_t* src, int32_t ok, int64_t* stats8, void* stream) {
  if (!dst || !src) { ts_set_error("fuse_update_tiled_finish: NULL handle"); return TSLAM_E_INVALID; }
  TsFuse* z = dst->fz;
  if (!z || z->phase == 0) { ts_set_error("fuse_update_tiled_finish: no tiled update is in progress"); return TSLAM_E_INVALID; }
  if (!ok) {  // the update failed on some rank: a plan alone wrote nothing, anything later leaves the sums invalid
    if (z->phase >= 2) z->valid = 0;
    z->phase = 0;
    return TSLAM_OK;
  }
  int rc = fz_phase(dst, 4, "fuse_update_tiled_finish");
  if (rc) return rc;
  if (src->ver.serial != z->plan_src) { ts_set_error("fuse_update_tiled_finish: src is not the map the update was planned with"); return TSLAM_E_INVALID; }
  TsDev f;
  fz_dev(*z, f);
  unsigned long long ctr[8];
  TS_CUDA(cudaMemcpyAsync(ctr, f.ctr, sizeof(ctr), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  TS_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  ts_fz_record(dst, src, z->plan);
  z->gen = dst->ver.write_gen - dst->ghost_gen;
  z->tiled = 1;
  z->tiling = z->plan_tiling;
  z->phase = 0;
  ts_fz_stats(z->plan, ctr, stats8);
  return TSLAM_OK;
}
