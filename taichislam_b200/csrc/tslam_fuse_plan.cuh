// libtslam.so - what the incremental global fusions share: tslam_tsdf_fuse_update (tslam_fuse.cu, single and tiled
// maps) and tslam_octo_fuse_update (tslam_octo_fuse.cu).  The plan rule (what an update does with each submap), so
// that `include`, `tolerance` and the full-update reasons mean the same thing for both map types; the fusion state of a
// destination, its device scratch and sum storage; the plan and list kernels; and the host steps around them.  What
// differs - the splat and readout of each map's voxels - stays in the two .cu files.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <type_traits>
#include <vector>
#include "tslam_internal.cuh"

// full-update reasons (stats8[0]; 0 = incremental)
// 7, 8: tiled updates only (tslam_tsdf_fuse_update_tiled_*)
enum { FZ_INCR = 0, FZ_FIRST = 1, FZ_ASKED = 2, FZ_OTHER_SRC = 3, FZ_DST_WRITTEN = 4, FZ_CONTENT = 5, FZ_COST = 6, FZ_CUTS = 7,
       FZ_INVALID = 8 };
enum { FZ_NONE = 0, FZ_ADD, FZ_REMOVE, FZ_MOVE, FZ_KEEP };  // what an update does with a submap

struct FzJob {        // one placement of one submap: sign +1 adds, -1 removes
  float R[9], T[3];
  int sign, pad;
};
struct FzSub {        // what a submap contributes to dst
  int fused;          // 1: its voxels are in dst, at (R, T)
  float R[9], T[3];
  unsigned long long ver;  // src content version at that time
  int nblk;           // its source blocks then
};
struct FzPlan {        // one update, from its plan to its record
  int reason;         // FZ_*
  bool full;
  std::vector<unsigned char> want, act;  // per submap: included with source blocks; FZ_NONE .. FZ_KEEP
  std::vector<int> nblk;
  std::vector<float> rad, pR, pT;        // radius, dst pose table
  long long n_add, n_move, n_remove, n_tol, cost, cost_full;  // cost: source blocks an incremental update splats
  unsigned long long ghosts;             // dst ghost blocks (TSDF)
};

// The state of a map as a fusion destination, created by its first update (the TSDF's TsFuse adds the tiled fields).
struct FzState {
  int valid = 0;      // dst (and its sums) are the fusion of the recorded submaps (cleared by a failed update)
  unsigned long long src_serial = 0, gen = 0;  // src handle and dst write generation of the last update
  std::vector<FzSub> sub;
  long long* sums = nullptr;  // sum storage (fz_reserve_sums: grown geometrically, never shrunk)
  size_t cap_blocks = 0;      // pool blocks it covers
  void* dev = nullptr;        // device scratch (fz_open)
  int dev_submaps = 0, dev_src_blocks = 0, dev_dst_blocks = 0;  // what it was sized for
};

template <class Z>
static void fz_free(Z*& z) {
  if (!z) return;
  if (z->sums) cudaFree(z->sums);
  if (z->dev) cudaFree(z->dev);
  delete z;
  z = nullptr;
}

// rotation angle of R0^T R (row-major 3x3), in double
static inline double fz_angle(const float* R0, const float* R) {
  double tr = 0.0;
  for (int i = 0; i < 3; i++)
    for (int k = 0; k < 3; k++) tr += (double)R0[3 * k + i] * (double)R[3 * k + i];  // trace(R0^T R) = sum R0_ki R_ki
  double c = (tr - 1.0) * 0.5;
  c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
  return std::acos(c);
}

// The full-update reason the handles give: asked (full), no valid state (`first`: the reason to report then), another
// source than last time, dst written since (`dst_written`); FZ_INCR when none applies.
static inline int fz_reason(const FzState& z, int full, int first, unsigned long long src_serial, bool dst_written) {
  if (full) return FZ_ASKED;
  if (!z.valid) return first;
  if (z.src_serial != src_serial) return FZ_OTHER_SRC;
  if (dst_written) return FZ_DST_WRITTEN;
  return FZ_INCR;
}

// The per-submap decisions of an update, from P.nblk (source blocks per submap), P.rad (radius of each submap's blocks
// about its origin), P.pR / P.pT (dst's pose table), the records `sub` of the last update and src's content versions.
// `reason` is the full-update reason found from the handles; when it is FZ_INCR the actions of an incremental update
// are planned: unchanged or moved within tolerance (|T - T0| + angle(R0^T R) r_s <= tolerance; 0: iff the pose bits
// are equal) -> KEEP, newly included -> ADD, excluded or now empty -> REMOVE, moved -> MOVE.  A fused submap whose
// content changed makes the update full (FZ_CONTENT).  Returns the reason; the cost rule is the caller's (fz_settle).
static inline int fz_decide(FzPlan& P, const std::vector<FzSub>& sub, const unsigned long long* content_ver, const uint8_t* include,
                            float tolerance, int reason) {
  const int S = (int)P.nblk.size();
  P.want.assign(S, 0);
  P.act.assign(S, FZ_NONE);
  P.n_add = P.n_move = P.n_remove = P.n_tol = P.cost = P.cost_full = 0;
  const std::vector<int>& nblk = P.nblk;
  for (int s = 0; s < S; s++) {
    const bool want = (!include || include[s]) && nblk[s] > 0;
    P.want[s] = want;
    if (want) P.cost_full += nblk[s];
    if (reason != FZ_INCR) continue;
    const FzSub& r = sub[s];
    if (!r.fused) {
      if (want) { P.act[s] = FZ_ADD; P.cost += nblk[s]; }
      continue;
    }
    if (r.ver != content_ver[s]) { reason = FZ_CONTENT; continue; }  // its old content is gone: cannot be subtracted
    if (!want) { P.act[s] = FZ_REMOVE; P.cost += r.nblk; continue; }
    const float* R = &P.pR[(size_t)9 * s];
    const float* T = &P.pT[(size_t)3 * s];
    if (!memcmp(R, r.R, 36) && !memcmp(T, r.T, 12)) { P.act[s] = FZ_KEEP; continue; }
    if (tolerance > 0.0f) {
      const double dx = (double)T[0] - r.T[0], dy = (double)T[1] - r.T[1], dz = (double)T[2] - r.T[2];
      const double move = std::sqrt(dx * dx + dy * dy + dz * dz) + fz_angle(r.R, R) * (double)P.rad[s];
      if (move <= (double)tolerance) { P.act[s] = FZ_KEEP; P.n_tol++; continue; }
    }
    P.act[s] = FZ_MOVE;
    P.cost += r.nblk + nblk[s];
  }
  P.reason = reason;
  return reason;
}

// the update's final reason: a full update adds every included submap
static inline void fz_settle(FzPlan& P, int reason) {
  P.reason = reason;
  P.full = reason != FZ_INCR;
  if (P.full) {
    P.n_tol = 0;
    for (size_t s = 0; s < P.act.size(); s++) P.act[s] = P.want[s] ? FZ_ADD : FZ_NONE;
  }
  P.n_add = P.n_move = P.n_remove = 0;
  for (size_t s = 0; s < P.act.size(); s++) {
    P.n_add += P.act[s] == FZ_ADD;
    P.n_move += P.act[s] == FZ_MOVE;
    P.n_remove += P.act[s] == FZ_REMOVE;
  }
}

// the record of a successful update: the submaps' records (act / pose table / nblk of P, content versions of src),
// and z valid for src; the write generation it saw is the caller's
static inline void fz_record(FzState& z, const FzPlan& P, const FzVer& src) {
  for (size_t s = 0; s < z.sub.size(); s++) {
    FzSub& r = z.sub[s];
    if (P.full) r.fused = 0;
    if (P.act[s] == FZ_REMOVE) r.fused = 0;
    if (P.act[s] == FZ_ADD || P.act[s] == FZ_MOVE) {
      r.fused = 1;
      memcpy(r.R, &P.pR[(size_t)9 * s], 36);
      memcpy(r.T, &P.pT[(size_t)3 * s], 12);
      r.ver = src.content_ver[s];
      r.nblk = P.nblk[s];
    }
  }
  z.valid = 1;
  z.src_serial = src.serial;
}

// ---------------------------------------------------------------------------
// device scratch of one update
// ---------------------------------------------------------------------------
struct FzDev {        // the arrays both maps use; each map's Dev adds its own after them (carve_tail)
  int* nblk;          // [max_submaps] source blocks per submap (k_fz_plan)
  unsigned* rbits;    // [max_submaps] float bits of the farthest block corner from the submap origin (k_fz_plan)
  int2* job_of;       // [max_submaps] (removal job, addition job), -1 none
  FzJob* jobs;        // [2 * max_submaps]
  int* list;          // [src max_blocks] source blocks with work (k_fz_list)
  unsigned long long* ctr;  // [8] [0] list length; the rest is each map's
};

// consecutive arrays in one buffer, each at its type's alignment; with a null base it only counts the bytes
struct FzCarve {
  char* base;
  size_t bytes;
  template <class T>
  T* take(size_t n) {
    bytes = (bytes + alignof(T) - 1) / alignof(T) * alignof(T);
    T* p = base ? (T*)(base + bytes) : nullptr;
    bytes += n * sizeof(T);
    return p;
  }
};

// The scratch of S submaps, B source blocks and D dst blocks laid out from base: the common arrays, then the map's
// (f.carve_tail).  Returns its size, so that the allocation and the layout come from the same code.
template <class Dev>
static size_t fz_carve(char* base, int S, int B, int D, Dev& f) {
  FzCarve c{base, 0};
  f.ctr = c.take<unsigned long long>(8);
  f.jobs = c.take<FzJob>((size_t)2 * S);
  f.job_of = c.take<int2>(S);
  f.nblk = c.take<int>(S);
  f.rbits = c.take<unsigned>(S);  // (right after nblk: fz_plan clears both at once)
  f.list = c.take<int>(B);
  f.carve_tail(c, D);
  return c.bytes;
}

// the scratch of z as fz_open last sized it
template <class Dev>
static void fz_dev(const FzState& z, Dev& f) {
  fz_carve((char*)z.dev, z.dev_submaps, z.dev_src_blocks, z.dev_dst_blocks, f);
}

// dst's fusion state z (the first update creates it) and its device scratch: reallocated when the submap count S or the
// dst pool size D that the map's own arrays take (0: none) changed, or the source pool size B grew
template <class Z, class Dev>
static int fz_open(Z*& z, int S, int B, int D, Dev& f) {
  if (!z) {
    z = new Z();
    z->sub.assign(S, FzSub());
  }
  if (!z->dev || z->dev_submaps != S || z->dev_src_blocks < B || z->dev_dst_blocks != D) {
    if (z->dev) TS_CUDA(cudaFree(z->dev));
    z->dev = nullptr;
    TS_CUDA(cudaMalloc(&z->dev, fz_carve(nullptr, S, B, D, f)));
    z->dev_submaps = S;
    z->dev_src_blocks = B;
    z->dev_dst_blocks = D;
  }
  fz_dev(*z, f);
  return TSLAM_OK;
}

// Sum storage for at least `need` pool blocks: `planes` planes of `words` int64 per block, plane after plane, grown to
// max(need, 2 x cap) blocks (at most max_blocks) with the old sums kept and the new ones zero.  `what` prefixes the error.
static inline int fz_reserve_sums(FzState& z, size_t need, size_t max_blocks, size_t words, int planes, const char* what, cudaStream_t st) {
  if (need <= z.cap_blocks) return TSLAM_OK;
  size_t cap = std::max(need, 2 * z.cap_blocks);
  if (cap > max_blocks) cap = max_blocks;
  const size_t bytes = cap * words * 8 * planes;
  long long* p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    if (planes > 1)
      ts_set_error("%s: cannot allocate %zu bytes of sum planes (%zu pool blocks x %d planes x %zu KiB): %s", what, bytes, cap, planes, words / 128,
                   cudaGetErrorString(e));
    else
      ts_set_error("%s: cannot allocate %zu bytes of sum words (%zu pool blocks x %zu KiB): %s", what, bytes, cap, words / 128, cudaGetErrorString(e));
    return TSLAM_E_CUDA;
  }
  const size_t old_n = z.cap_blocks * words, n = cap * words;
  for (int k = 0; k < planes; k++) {
    long long* dstp = p + k * n;
    if (old_n) TS_CUDA(cudaMemcpyAsync(dstp, z.sums + k * old_n, old_n * 8, cudaMemcpyDeviceToDevice, st));
    TS_CUDA(cudaMemsetAsync(dstp + old_n, 0, (n - old_n) * 8, st));
  }
  if (z.sums) {
    TS_CUDA(cudaStreamSynchronize(st));
    TS_CUDA(cudaFree(z.sums));
  }
  z.sums = p;
  z.cap_blocks = cap;
  return TSLAM_OK;
}

// ---------------------------------------------------------------------------
// kernels, over the grid of either map (TsGrid: 16^3 blocks, ghost blocks of tiled maps skipped; OcGrid: 8^3 blocks)
// ---------------------------------------------------------------------------
__device__ __forceinline__ bool fz_ghost(const TsGrid& g, int b) { return g.ghost[b] != 0; }
__device__ __forceinline__ bool fz_ghost(const OcGrid&, int) { return false; }

// blocks and radius per source submap (the corners bound every voxel of the block); TsGrid: ghost blocks of dst (ctr[3])
template <class G>
__global__ void __launch_bounds__(256) k_fz_plan(G src, G dst, float vs, FzDev f) {
  constexpr int E = std::is_same<G, TsGrid>::value ? TS_B : OC_B;
  const int nb = min(*src.n_blocks, src.max_blocks);
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    if (fz_ghost(src, b)) continue;
    int s, bx, by, bz;
    ts_unpack_key(src.block_key[b], s, bx, by, bz);
    const float ex = fmaxf(fabsf((float)(bx * E) * vs), fabsf((float)(bx * E + E) * vs));
    const float ey = fmaxf(fabsf((float)(by * E) * vs), fabsf((float)(by * E + E) * vs));
    const float ez = fmaxf(fabsf((float)(bz * E) * vs), fabsf((float)(bz * E + E) * vs));
    atomicAdd(&f.nblk[s], 1);
    atomicMax(&f.rbits[s], __float_as_uint(sqrtf(ex * ex + ey * ey + ez * ez)));  // non-negative floats order as uints
  }
  if constexpr (std::is_same<G, TsGrid>::value) {
    const int nd = min(*dst.n_blocks, dst.max_blocks);
    unsigned ng = 0;
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nd; b += gridDim.x * blockDim.x) ng += fz_ghost(dst, b);
    if (ng) atomicAdd(&f.ctr[3], (unsigned long long)ng);
  }
}

// the (non-ghost) source blocks of submaps with a job
template <class G>
__global__ void __launch_bounds__(256) k_fz_list(G src, FzDev f) {
  const int nb = min(*src.n_blocks, src.max_blocks);
  const int stride = gridDim.x * blockDim.x;
  const int iters = (nb + stride - 1) / stride;
  for (int it = 0; it < iters; ++it) {  // uniform trip count: the warp ballot below needs all lanes
    const int b = it * stride + blockIdx.x * blockDim.x + threadIdx.x;
    bool want = false;
    if (b < nb && !fz_ghost(src, b)) {
      int s, bx, by, bz;
      ts_unpack_key(src.block_key[b], s, bx, by, bz);
      const int2 j = f.job_of[s];
      want = j.x >= 0 || j.y >= 0;
    }
    const long long row = warp_append_u64(want, &f.ctr[0]);
    if (want) f.list[row] = b;
  }
}

// ---------------------------------------------------------------------------
// host steps (M: tslam_tsdf or tslam_octo)
// ---------------------------------------------------------------------------
// Refusals that need no handle contents (TSLAM_E_INVALID, nothing written); `what` prefixes the error
static inline int fz_check_args(const void* dst, const void* src, float tolerance, const char* what) {
  if (!std::isfinite(tolerance) || tolerance < 0.0f) {
    ts_set_error("%s: tolerance %g must be finite and >= 0", what, (double)tolerance);
    return TSLAM_E_INVALID;
  }
  if (!dst || !src) { ts_set_error("%s: NULL handle", what); return TSLAM_E_INVALID; }
  if (dst == src) { ts_set_error("%s: dst == src (a map cannot be fused into itself)", what); return TSLAM_E_INVALID; }
  return TSLAM_OK;
}

// The plan of an update (k_fz_plan: source blocks and radius per submap, dst ghosts; dst's pose table), after clearing
// the counters.  `reason` is the full-update reason found from the host state; when it is FZ_INCR the per-submap actions
// of an incremental update are planned, which may still find a fused submap whose content changed (FZ_CONTENT).  The
// cost rule and the switch to a full update's actions are the caller's (fz_settle), as a tiled update decides them over
// all ranks.
template <class M>
static int fz_plan(M* dst, M* src, const FzDev& f, const uint8_t* include, float tolerance, int reason, cudaStream_t st, FzPlan& P) {
  const int S = dst->cfg.max_submaps;
  TS_CUDA(cudaMemsetAsync(f.ctr, 0, 8 * 8, st));
  TS_CUDA(cudaMemsetAsync(f.nblk, 0, (size_t)S * 8, st));  // nblk and rbits
  k_fz_plan<<<src->sm_count * 4, 256, 0, st>>>(src->g, dst->g, src->in.vs, f);
  TS_LAUNCH_CHECK(dst);
  P.nblk.assign(S, 0);
  P.rad.assign(S, 0.0f);
  P.pR.assign((size_t)S * 9, 0.0f);
  P.pT.assign((size_t)S * 3, 0.0f);
  unsigned long long ctr0[8] = {0};
  TS_CUDA(cudaMemcpyAsync(P.nblk.data(), f.nblk, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(P.rad.data(), f.rbits, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
  // (each copy to pageable memory is a round trip: only a grid with ghost blocks reads the counters)
  if constexpr (std::is_same<decltype(dst->g), TsGrid>::value) TS_CUDA(cudaMemcpyAsync(ctr0, f.ctr, sizeof(ctr0), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(P.pR.data(), dst->pose_R, (size_t)S * 36, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(P.pT.data(), dst->pose_T, (size_t)S * 12, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  P.ghosts = ctr0[3];
  fz_decide(P, dst->fz->sub, src->ver.content_ver, include, tolerance, reason);
  return TSLAM_OK;
}

// the jobs of an update (host copies of f.jobs / f.job_of)
struct FzJobs {
  std::vector<FzJob> jobs;
  std::vector<int2> of;  // per submap: (removal job, addition job), -1 none
  explicit FzJobs(int S) : of(S, make_int2(-1, -1)) {}
  void add(int s, const float* R, const float* T, int sign) {  // submap s at (R, T): sign -1 removes, +1 adds
    FzJob j;
    memcpy(j.R, R, 36);
    memcpy(j.T, T, 12);
    j.sign = sign;
    j.pad = 0;
    (sign < 0 ? of[s].x : of[s].y) = (int)jobs.size();
    jobs.push_back(j);
  }
};

// the jobs of a plan: removals at the recorded poses (REMOVE, MOVE), additions at dst's pose table (ADD, MOVE)
static inline FzJobs fz_jobs(const FzPlan& P, const std::vector<FzSub>& sub) {
  FzJobs J((int)sub.size());
  for (size_t s = 0; s < sub.size(); s++) {
    if (P.act[s] == FZ_REMOVE || P.act[s] == FZ_MOVE) J.add((int)s, sub[s].R, sub[s].T, -1);
    if (P.act[s] == FZ_ADD || P.act[s] == FZ_MOVE) J.add((int)s, &P.pR[(size_t)9 * s], &P.pT[(size_t)3 * s], 1);
  }
  return J;
}

// upload the jobs and list the source blocks of the submaps with one (f.list, f.ctr[0], which must be zero)
template <class M>
static int fz_list(M* dst, M* src, const FzDev& f, const FzJobs& J, cudaStream_t st) {
  TS_CUDA(cudaMemcpyAsync(f.jobs, J.jobs.data(), J.jobs.size() * sizeof(FzJob), cudaMemcpyHostToDevice, st));
  TS_CUDA(cudaMemcpyAsync(f.job_of, J.of.data(), J.of.size() * sizeof(int2), cudaMemcpyHostToDevice, st));
  const int gl = std::max(1, std::min((src->g.max_blocks + 255) / 256, src->sm_count * 4));
  k_fz_list<<<gl, 256, 0, st>>>(src->g, f);
  TS_LAUNCH_CHECK(dst);
  return TSLAM_OK;
}

// stats8 of an update: the plan's reason and counts, then the three counters the map reports
static inline void fz_stats(const FzPlan& P, int64_t c5, int64_t c6, int64_t c7, int64_t* stats8) {
  if (!stats8) return;
  stats8[0] = P.reason;
  stats8[1] = P.n_add;
  stats8[2] = P.n_move;
  stats8[3] = P.n_remove;
  stats8[4] = P.n_tol;
  stats8[5] = c5;
  stats8[6] = c6;
  stats8[7] = c7;
}
