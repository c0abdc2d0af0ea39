// libtslam.so - ESDF: converged 26-neighbour signed-distance wavefront over the
// observed voxels of one submap.
//
// Semantic source: DenseSDF.propogate_esdf and its raise/lower queues
// (dense_esdf.py:228-333).  That code is dead at HEAD (not exported, stale ctor and
// indices) and its lower queue never re-inserts improved voxels (:292,:298 commented
// out), so there is no runnable reference behaviour: PARITY UNPINNED.  We implement
// the converged fixed point the code describes (DESIGN.md "ESDF"):
//   fixed band |TSDF| < gamma = voxel_scale (is_fixed :228-230): ESDF = TSDF (:315-320)
//   other observed voxels start at sign(TSDF)*max_ray_length (:324,:328) and relax
//     positive side: E(v) = min(E(v), E(h) + |dir|*vs)   h in fixed U positive   (:286-291)
//     negative side: E(v) = max(E(v), E(h) - |dir|*vs)   h in fixed U negative   (:294-298)
//   to convergence.  f32 min/+ is monotone, so the least fixed point is unique and
//   equals the oracle's multi-source Dijkstra bit-for-bit.
// The wavefront - full and incremental update, raise and lower waves, queries - is the one both ESDFs share
// (tslam_esdf_common.cuh), on 16^3 blocks (18^3 tiles, 256 threads, 4 CTAs per SM).  This ESDF's rules (EsTsdf):
//   classes     UNOBS, FIXED (|t| < gamma), POS, NEG, INERT (t NaN), from the live obs / tw planes; the field is g.esdf
//   seeds       FIXED: t; other observed voxels: sgn(t) * max_ray_length; unobserved: 0
//   targets     POS (min side) and NEG (max side); sources of a target: FIXED voxels and voxels of its own side, each
//               offering E(h) +- c
//   detect      (blocks committed since the last update) a voxel whose class changed, that became observed, or whose
//               fixed-band value moved -> CHANGED
//   raise test  a target whose value is EXACTLY E(h) +- c of any flagged neighbour h
//   queries     a corner has a value when it was FIXED, POS or NEG; ghost blocks are read only after a completed tiled
//               ESDF
//   extras      init clears esdf_dirty; tiled (TILED): the sweep skips ghosts and marks changed owned blocks in xmark
// Unflagged voxels keep values that are still attainable (their support chain avoids every changed voxel), i.e. upper
// bounds; min/+ relaxation from there converges to the SAME least fixed point as a full recompute - tested
// bit-for-bit (tests/test_gpu_mc_octo_esdf.py::test_esdf_incremental_equals_full_512).  The reference seeds its wave
// from the voxels the frame just touched (dense_esdf.py:309-330) and has a raise and a lower queue (:260-299).
#include <cstring>
#include "tslam_esdf_common.cuh"
#include "tslam_traj.cuh"

enum { ES_UNOBS = 0, ES_FIXED = 1, ES_POS = 2, ES_NEG = 3, ES_INERT = 4 };  // INERT: observed, TSDF is NaN

struct EsAux {
  int* nbr;      // [max_blocks*27] neighbour block indices (-1 = absent)
  int* epoch;    // [max_blocks] last sweep in which the block changed
  int* changed;  // [ES_MAX_SWEEPS+2] changed[k] != 0 <=> sweep k changed something
  unsigned char* cls;  // [max_blocks*4096] class of the voxel at the last update (+ flags during an update)
  int* repoch;   // [max_blocks] raise wave: last raise sweep in which the block gained suspects
  int* rchanged; // [ES_MAX_SWEEPS+2]
  int* counts;   // [4] changed voxels, suspect voxels, re-initialised blocks, (spare)
  int* nb_seen;  // [1] blocks in the pool when the last update ran (blocks are bump-allocated: higher indices are newer)
  int* xmark;    // [max_blocks] tiled ESDF: owned block changed since last packed / ghost block unpacked since last relax
};
__device__ __forceinline__ unsigned char es_class(bool obs, float t, float gamma) {
  if (!obs) return ES_UNOBS;
  return (fabsf(t) < gamma) ? ES_FIXED : (t > 0.0f ? ES_POS : (t < 0.0f ? ES_NEG : ES_INERT));
}
__device__ __forceinline__ float es_sgn(float v) { return (float)((0.0f < v) - (v < 0.0f)); }

// The TSDF ESDF's rules for the shared wavefront (tslam_esdf_common.cuh).  Classes come from the live obs / tw planes;
// the field is g.esdf.
struct EsTsdf {
  static constexpr int SHIFT = TS_BSHIFT, THREADS = 256, GRID = 4;
  static constexpr int COUNTS_CLEARED = 8;  // nb_seen too (set again by init / prepare)
  static constexpr bool GHOSTS = true;
  static constexpr unsigned char NONE = ES_UNOBS, MIN_SIDE = ES_POS, MAX_SIDE = ES_NEG;
  TsGrid g;
  EsAux a;
  int submap;
  float gamma, far_v, vs;  // fixed band |TSDF| < gamma, seeds +-far_v, voxel size
  bool ghosts;             // queries: ghost blocks hold their owners' final values (a completed tiled ESDF)
  __device__ float* field() const { return g.esdf; }
  __device__ int* dirty() const { return g.esdf_dirty; }
  __device__ float seed(size_t off, unsigned char& c) const {
    const bool ob = g.obs[off] != 0;
    const float t = g.tw[off].x;
    c = es_class(ob, t, gamma);
    float e = 0.0f;
    if (ob) e = (c == ES_FIXED) ? t : es_sgn(t) * far_v;
    return e;
  }
  // a class change, a newly observed voxel, or a fixed-band value that moved
  __device__ bool moved(size_t off, unsigned char oc) const {
    const float t = g.tw[off].x;
    const unsigned char nc = es_class(g.obs[off] != 0, t, gamma);
    return (nc != oc) || (nc == ES_FIXED && g.esdf[off] != t);
  }
  __device__ void stage(size_t off, float& e, unsigned char& c) const {
    if (g.obs[off]) {
      const float t = g.tw[off].x;
      c = (fabsf(t) < gamma) ? ES_FIXED : (t > 0.0f ? ES_POS : (t < 0.0f ? ES_NEG : ES_INERT));
      e = *(volatile float*)&g.esdf[off];
    }
  }
  __device__ static bool target(unsigned char c) { return c == ES_POS || c == ES_NEG; }
  __device__ static bool source(unsigned char c, unsigned char h) { return h == ES_FIXED || h == c; }
  __device__ static bool raise_source(unsigned char) { return true; }
  __device__ static float cand_min(unsigned char, float he, float d) { return he + d; }
  __device__ static float cand_max(unsigned char, float he, float d) { return he - d; }
  __device__ static bool valid(unsigned char c) { return c == ES_FIXED || c == ES_POS || c == ES_NEG; }
  __device__ void init_done(int b) const { g.esdf_dirty[b] = 0; }
  __device__ void prepare_block(int, int) const {}
};

// ---- tiled ESDF (tslam_esdf_tiled_*) ----------------------------------------------------------------------------
// Start of a relax: only the ghosts unpacked since the last relax are wave sources (epoch 0); every other block of the
// submap waits for the wave (epoch -1).  The marks of owned blocks (changed since last packed) are kept.
__global__ void __launch_bounds__(256) k_esdf_rearm(TsGrid g, EsAux aux) {
  const int nb = min(*aux.nb_seen, g.max_blocks);
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    if (aux.epoch[b] < -1) continue;  // block of another submap
    const bool src = g.ghost[b] && aux.xmark[b];
    aux.epoch[b] = src ? 0 : -1;
    if (g.ghost[b]) aux.xmark[b] = 0;
  }
}

// One CTA per received block: overwrite the ESDF plane of an existing ghost block of the submap and mark it as a
// source of the next relax.  A key that is absent, owned, of another submap or newer than the update is counted in
// *bad and nothing is written for it.
__global__ void __launch_bounds__(256) k_esdf_ghost_unpack(TsGrid g, EsAux aux, long long n, const long long* keys, const float4* esdf_in,
                                                            int* bad) {
  __shared__ int s_blk;
  const int nb_seen = *aux.nb_seen;
  for (long long q = blockIdx.x; q < n; q += gridDim.x) {
    __syncthreads();
    if (threadIdx.x == 0) {
      int b = ts_find(g, (unsigned long long)keys[q]);
      if (b >= nb_seen || (b >= 0 && (!g.ghost[b] || aux.epoch[b] < -1))) b = -1;
      if (b < 0) atomicAdd(bad, 1);
      s_blk = b;
    }
    __syncthreads();
    const int blk = s_blk;
    if (blk < 0) continue;
    float4* dst = reinterpret_cast<float4*>(g.esdf + (size_t)blk * TS_B3);
    for (int v = threadIdx.x; v < TS_B3 / 4; v += blockDim.x) dst[v] = esdf_in[q * (TS_B3 / 4) + v];
    if (threadIdx.x == 0) aux.xmark[blk] = 1;
  }
}

__global__ void __launch_bounds__(256) k_esdf_gather(TsGrid g, int submap, long long cap, int32_t* idx, float* esdf,
                                                      unsigned long long* counter) {
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
        esdf[row] = g.esdf[base + v];
      }
    }
  }
}

static int es_alloc(tslam_tsdf* m) {
  if (m->g.esdf) return TSLAM_OK;
  const size_t nb = (size_t)m->g.max_blocks;
  TS_CUDA(cudaMalloc(&m->g.esdf, nb * TS_B3 * 4));
  TS_CUDA(cudaMemset(m->g.esdf, 0, nb * TS_B3 * 4));
  TS_CUDA(cudaMalloc(&m->esdf_aux, (nb * 30 + 2 * (ES_MAX_SWEEPS + 2) + 8) * 4 + nb * TS_B3));
  TS_CUDA(cudaMemset(m->esdf_aux, 0, (nb * 30 + 2 * (ES_MAX_SWEEPS + 2) + 8) * 4 + nb * TS_B3));
  m->esdf_full_needed = 1;
  return TSLAM_OK;
}
static EsAux es_aux(tslam_tsdf* m) {
  EsAux aux;
  const size_t nb = (size_t)m->g.max_blocks;
  aux.nbr = (int*)m->esdf_aux;
  aux.epoch = aux.nbr + nb * 27;
  aux.repoch = aux.epoch + nb;
  aux.changed = aux.repoch + nb;
  aux.rchanged = aux.changed + (ES_MAX_SWEEPS + 2);
  aux.counts = aux.rchanged + (ES_MAX_SWEEPS + 2);
  aux.nb_seen = aux.counts + 4;  // (inside the 8-int counts area; cleared with it at the start of every update)
  aux.cls = (unsigned char*)(aux.counts + 8);
  aux.xmark = (int*)(aux.cls + nb * TS_B3);
  return aux;
}
int* ts_esdf_xmark(tslam_tsdf* m) { return m->esdf_aux ? es_aux(m).xmark : nullptr; }
static EsTsdf es_rules(tslam_tsdf* m, int submap) {
  // dense_esdf.py:40 (fixed band), :324 (seed distance)
  return EsTsdf{m->g, es_aux(m), submap, (float)m->cfg.voxel_scale, (float)m->cfg.max_ray_length, m->in.vs, m->esdf_tiled == 2};
}

// mode 0 = incremental when the state allows it (same submap as the last update, no reset / bulk load in between),
// 1 = full recompute.  stats4 (HOST, may be NULL): lower sweeps, raise sweeps, changed voxels, suspect voxels.
extern "C" int tslam_esdf_update2(tslam_tsdf_t* m, int32_t submap, int32_t mode, int32_t* stats4, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  rc = es_alloc(m);
  if (rc) return rc;
  // (the state a tiled ESDF leaves - ghosts holding their owners' values - is no base for an incremental update)
  const bool full = mode == 1 || m->esdf_full_needed || m->esdf_submap != submap || m->esdf_tiled != 0;
  m->esdf_tiled = 0;
  rc = es_update(m, es_rules(m, submap), full, st, stats4);
  if (rc) return rc;
  m->esdf_full_needed = 0;
  m->esdf_submap = submap;
  return TSLAM_OK;
}

extern "C" int tslam_esdf_update(tslam_tsdf_t* m, int32_t submap, int32_t* n_sweeps_out, void* stream) {
  int32_t st4[4] = {0, 0, 0, 0};
  int rc = tslam_esdf_update2(m, submap, 0, st4, stream);
  if (n_sweeps_out) *n_sweeps_out = st4[0];
  return rc;
}

// ---- tiled ESDF: begin -> (ESDF halo pack -> exchange -> ghost unpack -> relax)* -> end --------------------------
// The exchange loop between begin and end is driven by the host layer (taichislam_b200/distributed.py); the ESDF halo
// pack lives with the other halo code in tslam_dist.cu.  Every value is an attainable upper bound at every step, so
// the loop ends at the single map's least fixed point (DESIGN.md section 6).
static int es_tiled_open(tslam_tsdf* m, const char* what) {
  if (!m->g.esdf || m->esdf_tiled != 1 || m->esdf_full_needed) {
    ts_set_error("%s: no tiled ESDF is in progress (tslam_esdf_tiled_begin, then no reset, load, fusion or ghost import)", what);
    return TSLAM_E_INVALID;
  }
  return TSLAM_OK;
}

extern "C" int tslam_esdf_tiled_begin(tslam_tsdf_t* m, int32_t submap, int32_t* n_sweeps_out, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  rc = es_alloc(m);
  if (rc) return rc;
  int32_t st4[4];
  m->esdf_tiled = 1;
  rc = es_update<true>(m, es_rules(m, submap), true, st, st4);
  if (rc) return rc;
  m->esdf_full_needed = 0;
  m->esdf_submap = submap;
  if (n_sweeps_out) *n_sweeps_out = st4[0];
  return TSLAM_OK;
}

extern "C" int tslam_esdf_ghost_unpack(tslam_tsdf_t* m, int64_t n, const int64_t* keys, const float* esdf, void* stream) {
  if (!m || n < 0 || (n && (!keys || !esdf))) return TSLAM_E_INVALID;
  int rc = es_tiled_open(m, "tslam_esdf_ghost_unpack");
  if (rc || n == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int* bad = m->scratch_i + 12;
  TS_CUDA(cudaMemsetAsync(bad, 0, 4, st));
  k_esdf_ghost_unpack<<<(int)(n < m->sm_count * 4 ? n : m->sm_count * 4), 256, 0, st>>>(m->g, es_aux(m), n, (const long long*)keys,
                                                                                         (const float4*)esdf, bad);
  TS_LAUNCH_CHECK(m);
  int h_bad = 0;
  TS_CUDA(cudaMemcpyAsync(&h_bad, bad, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (h_bad) {
    ts_set_error("tslam_esdf_ghost_unpack: %d of %lld keys are not ghost blocks of submap %d (nothing written for them)", h_bad, (long long)n,
                 m->esdf_submap);
    return TSLAM_E_INVALID;
  }
  return TSLAM_OK;
}

extern "C" int tslam_esdf_tiled_relax(tslam_tsdf_t* m, int32_t* n_sweeps_out, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  int rc = es_tiled_open(m, "tslam_esdf_tiled_relax");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const EsTsdf p = es_rules(m, m->esdf_submap);
  int n_lower = 0;
  TS_CUDA(cudaMemsetAsync(p.a.changed, 0, (ES_MAX_SWEEPS + 2) * 4, st));
  k_esdf_rearm<<<m->sm_count * 2, 256, 0, st>>>(m->g, p.a);
  TS_LAUNCH_CHECK(m);
  rc = es_wave(m, st, p.a.changed, 4, [&](int k) { es_k_wave<EsTsdf, false, true><<<m->sm_count * EsTsdf::GRID, EsTsdf::THREADS, 0, st>>>(p, k); }, &n_lower);
  if (rc) return rc;
  if (n_sweeps_out) *n_sweeps_out = n_lower;
  return TSLAM_OK;
}

extern "C" int tslam_esdf_tiled_end(tslam_tsdf_t* m) {
  if (!m) return TSLAM_E_INVALID;
  int rc = es_tiled_open(m, "tslam_esdf_tiled_end");
  if (rc) return rc;
  m->esdf_tiled = 2;
  return TSLAM_OK;
}

extern "C" int tslam_esdf_gather(tslam_tsdf_t* m, int32_t submap, int64_t cap, int32_t* idx, float* esdf, int64_t* n_out,
                                 void* stream) {
  if (!m || !n_out) return TSLAM_E_INVALID;
  if (!m->g.esdf) { ts_set_error("tslam_esdf_update has not run"); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* ctr = (unsigned long long*)(m->scratch_i + 8);
  TS_CUDA(cudaMemsetAsync(ctr, 0, 8, st));
  k_esdf_gather<<<m->sm_count * 4, 256, 0, st>>>(m->g, submap, cap, idx, esdf, ctr);
  TS_LAUNCH_CHECK(m);
  unsigned long long v = 0;
  TS_CUDA(cudaMemcpyAsync(&v, ctr, 8, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  *n_out = (int64_t)v;
  if ((int64_t)v > cap) { ts_set_error("esdf gather: capacity"); return TSLAM_E_CAPACITY; }
  return TSLAM_OK;
}

// ---- reading the field: batched queries and the slice export ----------------------------------------------------
// Both answer from the field as of the last update of the submap: the class byte that update left (not the live obs
// plane) and only the blocks the update saw.  A block allocated later has a pool index >= *nb_seen (bump allocation;
// a reset, which recycles the pool, forces the next update to be a full one and refuses queries until then).
// Ghost blocks count only after a completed tiled ESDF: they then hold their owners' final values.  A query corner has a
// value when it was FIXED, POS or NEG at the last update.
__global__ void __launch_bounds__(256) k_esdf_query(TsGrid g, EsAux aux, int submap, bool ghosts, long long n, const float* __restrict__ xyz,
                                                     float vs, float* __restrict__ dist, float* __restrict__ grad,
                                                     uint8_t* __restrict__ valid) {
  es_query(EsTsdf{g, aux, submap, 0.0f, 0.0f, vs, ghosts}, n, xyz, dist, grad, valid);
}

// cvt_ESDF_to_voxels_slice (dense_esdf.py:498-509): the voxels known at the last update whose uncentred index k + Nz/2
// lies strictly between _index - 0.5 and _index + 0.5 (bounds from the host), with ESDF value and position.  The
// reference's struct-for also visits the unobserved cells of active blocks (ESDF 0): those are not exported here.
__global__ void __launch_bounds__(256) k_esdf_extract_slice(TsGrid g, EsAux aux, int submap, int global_map, const float* pR,
                                                             const float* pT, float vs, float k_lo, float k_hi, long long cap,
                                                             float* xyz, float* val, int* counter) {
  const int nb = min(*aux.nb_seen, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap || g.ghost[b]) continue;  // (uniform per CTA)
    const size_t base = (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const int k = bz * TS_B + (v & 15);
      const float ku = (float)(k + g.hNz);
      const bool want = (aux.cls[base + v] & ES_CLS) != ES_UNOBS && k_lo < ku && ku < k_hi;
      const int row = warp_append_i32(want, counter);
      if (want && row < cap) {
        float x, y, z;
        voxel_xyz(g, global_map, pR, pT, s, bx * TS_B + (v >> 8), by * TS_B + ((v >> 4) & 15), k, vs, x, y, z);
        xyz[3 * (size_t)row] = x; xyz[3 * (size_t)row + 1] = y; xyz[3 * (size_t)row + 2] = z;
        val[row] = g.esdf[base + v];
      }
    }
  }
}

// the field of `submap` can be read: an update has completed, for that submap, and nothing has invalidated its state
static int es_readable(tslam_tsdf* m, int32_t submap, const char* what) {
  if (!m->g.esdf) { ts_set_error("%s: no ESDF has been computed (tslam_esdf_update has not run)", what); return TSLAM_E_INVALID; }
  if (m->esdf_full_needed) {
    ts_set_error("%s: the map was reset, bulk-loaded or fused since the last completed tslam_esdf_update", what);
    return TSLAM_E_INVALID;
  }
  if (m->esdf_submap != submap) {
    ts_set_error("%s: the last tslam_esdf_update was for submap %d, not %d", what, m->esdf_submap, submap);
    return TSLAM_E_INVALID;
  }
  if (m->esdf_tiled == 1) {
    ts_set_error("%s: a tiled ESDF is in progress (tslam_esdf_tiled_begin without tslam_esdf_tiled_end)", what);
    return TSLAM_E_INVALID;
  }
  return TSLAM_OK;
}

extern "C" int tslam_esdf_query(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* xyz, float* dist, float* grad,
                                uint8_t* valid, void* stream) {
  if (!m || n < 0 || (n && (!xyz || !dist || !grad || !valid))) return TSLAM_E_INVALID;
  int rc = es_readable(m, submap, "tslam_esdf_query");
  if (rc || n == 0) return rc;
  long long blocks = (n + 255) / 256;
  if (blocks > (long long)m->sm_count * 16) blocks = (long long)m->sm_count * 16;
  k_esdf_query<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(m->g, es_aux(m), submap, m->esdf_tiled == 2, n, xyz, m->in.vs, dist,
                                                               grad, valid);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

extern "C" int tslam_esdf_extract_slice(tslam_tsdf_t* m, int32_t submap, float z, int64_t cap, float* xyz, float* val,
                                        int32_t* count_dev, void* stream) {
  if (!m || cap < 0 || !xyz || !val || !count_dev) return TSLAM_E_INVALID;
  int rc = es_readable(m, submap, "tslam_esdf_extract_slice");
  if (rc) return rc;
  // _index = (z + map_size_z/2) / voxel_scale in f32 (dense_esdf.py:504), map_size_z = voxel_scale * Nz
  const float msz = (float)(m->cfg.voxel_scale * (double)m->cfg.Nz);
  const float index = (z + msz / 2.0f) / m->in.vs;
  k_esdf_extract_slice<<<m->sm_count * 4, 256, 0, (cudaStream_t)stream>>>(m->g, es_aux(m), submap, m->cfg.is_global_map, m->pose_R,
                                                                          m->pose_T, m->in.vs, index - 0.5f, index + 0.5f, cap, xyz,
                                                                          val, count_dev);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

// Trajectories against this ESDF (tslam_traj.cuh), read as tslam_esdf_query reads it
extern "C" int tslam_esdf_trajectory(tslam_tsdf_t* m, int32_t submap, int32_t T, const int32_t* n_ctrl, const double* ctrl_in,
                                     const tslam_traj_params_t* params, double* ctrl_out, double* cost, int32_t* info, void* stream) {
  const char* what = "tslam_esdf_trajectory";
  long long sum_n = 0;
  int rc = tj_check_args(what, T, n_ctrl, ctrl_in, params, ctrl_out, cost, info, &sum_n);
  if (rc) return rc;
  if (!m) { ts_set_error("%s: NULL handle", what); return TSLAM_E_INVALID; }
  rc = es_readable(m, submap, what);
  if (rc) return rc;
  if (params->clearance > m->cfg.max_ray_length) {
    ts_set_error("%s: clearance %g above the ESDF's far value max_ray_length %g", what, params->clearance, m->cfg.max_ray_length);
    return TSLAM_E_INVALID;
  }
  const EsTsdf p{m->g, es_aux(m), submap, 0.0f, 0.0f, m->in.vs, m->esdf_tiled == 2};
  return tj_run(m, p, m->in.vs, what, &m->traj_mem, &m->traj_mem_bytes, T, n_ctrl, sum_n, ctrl_in, params, ctrl_out, cost, info,
                (cudaStream_t)stream);
}
