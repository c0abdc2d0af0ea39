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
// Implementation: block-parallel wavefront with a block-level WORK QUEUE.
//   * a CTA stages its block plus a one-voxel halo (18^3) in shared memory, relaxes to
//     LOCAL convergence (ballot-voted iterations), writes back and stamps the block
//     with the sweep number when anything changed;
//   * sweep k only runs the blocks that have a neighbour (26 + self) stamped >= k-1 -
//     the wave front; every block's 27 neighbour indices are resolved once per update;
//   * sweeps are enqueued in groups; a sweep whose predecessor changed nothing returns
//     at once, so the host only synchronises once per group to test for convergence.
//
// INCREMENTAL update (round 2; the reference seeds its wave from the voxels the frame just touched,
// dense_esdf.py:309-330, and has a raise and a lower queue, :260-299).  State kept between updates: the field and a
// class byte per voxel.  An update after new commits:
//   1. detect   (blocks committed since the last update): voxels whose class changed, that became observed, or whose
//               fixed-band value moved are flagged CHANGED;
//   2. raise    wave: a non-fixed voxel whose value is EXACTLY a flagged neighbour's old value +- the edge cost may
//               have been derived from it -> flagged SUSPECT, and so on to closure (f32 equality is exact: at a
//               fixed point every relaxed value IS some neighbour's value +- cost);
//   3. re-init  changed voxels take their new class / seed, suspects go back to +-max_ray_length;
//   4. lower    the sweep kernel above, started from the re-initialised blocks only.
// Unflagged voxels keep values that are still attainable (their support chain avoids every changed voxel), i.e. upper
// bounds; min/+ relaxation from there converges to the SAME least fixed point as a full recompute - tested
// bit-for-bit (tests/test_gpu_mc_octo_esdf.py::test_esdf_incremental_equals_full_512).
#include <cstring>
#include "tslam_esdf_common.cuh"

#define ES_T 18
#define ES_T3 (ES_T * ES_T * ES_T)

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

__device__ __forceinline__ int es_tidx(int lx, int ly, int lz) { return ((lx + 1) * ES_T + (ly + 1)) * ES_T + (lz + 1); }
__device__ __forceinline__ float es_sgn(float v) { return (float)((0.0f < v) - (v < 0.0f)); }

// TILED (tslam_esdf_tiled_begin): ghost blocks are seeded like owned ones, and every owned block of the submap is
// marked for the first ESDF halo pack.
template <bool TILED>
__global__ void __launch_bounds__(256) k_esdf_init(TsGrid g, EsAux aux, int submap, float gamma, float far_v) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  if (blockIdx.x == 0 && threadIdx.x == 0) *aux.nb_seen = nb;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (threadIdx.x == 0) aux.epoch[b] = (s == submap) ? 0 : -1000000;
    if (TILED && threadIdx.x == 0) aux.xmark[b] = (s == submap && !g.ghost[b]) ? 1 : 0;
    if (s != submap) continue;
    if (threadIdx.x < 27) {
      const int dx = threadIdx.x / 9 - 1, dy = (threadIdx.x / 3) % 3 - 1, dz = threadIdx.x % 3 - 1;
      aux.nbr[b * 27 + threadIdx.x] = ts_find(g, ts_pack_key(s, bx + dx, by + dy, bz + dz));
    }
    const size_t base = (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      float e = 0.0f;
      const bool ob = g.obs[base + v] != 0;
      const float t = g.tw[base + v].x;
      if (ob) e = (fabsf(t) < gamma) ? t : es_sgn(t) * far_v;
      g.esdf[base + v] = e;
      aux.cls[base + v] = es_class(ob, t, gamma);
    }
    if (threadIdx.x == 0) g.esdf_dirty[b] = 0;
  }
}

// ---- incremental update ------------------------------------------------------------------------------------------
// neighbour table of every block of the submap + epochs reset; the voxel state is left alone
__global__ void __launch_bounds__(256) k_esdf_prepare(TsGrid g, EsAux aux, int submap) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  if (blockIdx.x == 0 && threadIdx.x == 0) *aux.nb_seen = nb;
  const int w = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31, nw = (gridDim.x * 256) >> 5;
  for (int b = w; b < nb; b += nw) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (lane == 0) { aux.epoch[b] = (s == submap) ? -1 : -1000000; aux.repoch[b] = -1; }
    if (s != submap) continue;
    if (lane < 27) {
      const int dx = lane / 9 - 1, dy = (lane / 3) % 3 - 1, dz = lane % 3 - 1;
      aux.nbr[b * 27 + lane] = ts_find(g, ts_pack_key(s, bx + dx, by + dy, bz + dz));
    }
  }
}

// 1. detect: blocks committed since the last update
__global__ void __launch_bounds__(256) k_esdf_detect(TsGrid g, EsAux aux, int submap, float gamma) {
  __shared__ int s_any;
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (!g.esdf_dirty[b] || aux.epoch[b] < -1) continue;  // (uniform per CTA)
    __syncthreads();
    if (threadIdx.x == 0) s_any = 0;
    __syncthreads();
    const size_t base = (size_t)b * TS_B3;
    int mine = 0;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const unsigned char oc = aux.cls[base + v] & ES_CLS;
      const float t = g.tw[base + v].x;
      const unsigned char nc = es_class(g.obs[base + v] != 0, t, gamma);
      const bool ch = (nc != oc) || (nc == ES_FIXED && g.esdf[base + v] != t);
      if (ch) { aux.cls[base + v] = oc | ES_CH; mine++; }
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) { atomicAdd(&s_any, mine); }
    __syncthreads();
    if (threadIdx.x == 0) {
      g.esdf_dirty[b] = 0;
      if (s_any) { aux.repoch[b] = 0; atomicAdd(&aux.counts[0], s_any); }
    }
  }
}

struct EsRTile {
  float e[ES_T3];
  unsigned char cls[ES_T3];
  int nbr[27];
  int active, changed, any_write;
};

// 2. raise wave: flag the voxels that may have been derived from a flagged neighbour
__global__ void __launch_bounds__(256) k_esdf_raise(TsGrid g, EsAux aux, int sweep, float vs) {
  __shared__ EsRTile tile;
  if (sweep > 1 && aux.rchanged[sweep - 1] == 0) return;
  const int nb = min(*g.n_blocks, g.max_blocks);
  const float d1 = vs, d2 = sqrtf(2.0f) * vs, d3 = sqrtf(3.0f) * vs;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    __syncthreads();
    if (threadIdx.x == 0) { tile.active = 0; tile.any_write = 0; }
    __syncthreads();
    if (aux.epoch[b] < -1) continue;
    if (threadIdx.x < 27) {
      const int n = aux.nbr[b * 27 + threadIdx.x];
      tile.nbr[threadIdx.x] = n;
      if (n >= 0 && *(volatile int*)&aux.repoch[n] >= sweep - 1) tile.active = 1;
    }
    __syncthreads();
    if (!tile.active) continue;
    for (int c = threadIdx.x; c < ES_T3; c += blockDim.x) {
      const int lz = c % ES_T - 1, ly = (c / ES_T) % ES_T - 1, lx = c / (ES_T * ES_T) - 1;
      const int nbk = tile.nbr[((((lx + 16) >> 4) * 3 + ((ly + 16) >> 4)) * 3) + ((lz + 16) >> 4)];
      float ev = 0.0f;
      unsigned char cl = ES_UNOBS;
      if (nbk >= 0) {
        const size_t off = (size_t)nbk * TS_B3 + ((((lx & 15) << 4) | (ly & 15)) << 4 | (lz & 15));
        cl = *(volatile unsigned char*)&aux.cls[off];
        ev = g.esdf[off];  // old values: nothing writes the field during the raise wave
      }
      tile.e[c] = ev;
      tile.cls[c] = cl;
    }
    __syncthreads();
    for (int iter = 0; iter < 64; ++iter) {
      if (threadIdx.x == 0) tile.changed = 0;
      __syncthreads();
      bool mine = false;
      for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
        const int c0 = es_tidx(v >> 8, (v >> 4) & 15, v & 15);
        const unsigned char cl = tile.cls[c0];
        if (cl != ES_POS && cl != ES_NEG) continue;  // flagged, fixed, unobserved: nothing to decide
        const float cur = tile.e[c0];
        bool hit = false;
#pragma unroll
        for (int dx = -1; dx <= 1; dx++)
#pragma unroll
          for (int dy = -1; dy <= 1; dy++)
#pragma unroll
            for (int dz = -1; dz <= 1; dz++) {
              const int nz_ = (dx != 0) + (dy != 0) + (dz != 0);
              if (nz_ == 0) continue;
              const int cn = c0 + (dx * ES_T + dy) * ES_T + dz;
              if (!(tile.cls[cn] & (ES_CH | ES_SU))) continue;
              const float dis = nz_ == 1 ? d1 : (nz_ == 2 ? d2 : d3);
              const float he = tile.e[cn];
              hit |= (cl == ES_POS) ? (he + dis == cur) : (he - dis == cur);
            }
        if (hit) { tile.cls[c0] = cl | ES_SU; mine = true; }
      }
      if (__any_sync(0xffffffffu, mine) && (threadIdx.x & 31) == 0) tile.changed = 1;
      __syncthreads();
      const int ch = tile.changed;
      if (ch && threadIdx.x == 0) tile.any_write = 1;
      __syncthreads();
      if (!ch) break;
    }
    if (tile.any_write) {
      const size_t base = (size_t)b * TS_B3;
      for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
        const unsigned char cl = tile.cls[es_tidx(v >> 8, (v >> 4) & 15, v & 15)];
        if (cl & ES_SU) aux.cls[base + v] = cl;
      }
      if (threadIdx.x == 0) {
        __threadfence();
        aux.repoch[b] = sweep;
        aux.rchanged[sweep] = 1;
      }
    }
  }
}

// 3. re-initialise flagged voxels; their blocks start the lower wave (epoch 0)
__global__ void __launch_bounds__(256) k_esdf_reinit(TsGrid g, EsAux aux, float gamma, float far_v) {
  __shared__ int s_n[2];
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (aux.repoch[b] < 0) continue;  // no flagged voxel in this block (uniform per CTA)
    __syncthreads();
    if (threadIdx.x == 0) { s_n[0] = 0; s_n[1] = 0; }
    __syncthreads();
    const size_t base = (size_t)b * TS_B3;
    int nsu = 0;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const unsigned char c = aux.cls[base + v];
      if (!(c & (ES_CH | ES_SU))) continue;
      const float t = g.tw[base + v].x;
      const bool ob = g.obs[base + v] != 0;
      const unsigned char nc = es_class(ob, t, gamma);
      float e = 0.0f;
      if (ob) e = (nc == ES_FIXED) ? t : es_sgn(t) * far_v;
      g.esdf[base + v] = e;
      aux.cls[base + v] = nc;
      nsu += (c & ES_SU) ? 1 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) nsu += __shfl_xor_sync(0xffffffffu, nsu, o);
    if ((threadIdx.x & 31) == 0 && nsu) atomicAdd(&s_n[0], nsu);
    __syncthreads();
    if (threadIdx.x == 0) {
      aux.epoch[b] = 0;
      if (s_n[0]) atomicAdd(&aux.counts[1], s_n[0]);
      atomicAdd(&aux.counts[2], 1);
    }
  }
}

struct EsTile {
  float e[ES_T3];
  unsigned char cls[ES_T3];
  int nbr[27];
  int active;
  int changed;
  int any_write;
};


// TILED: ghost blocks are read-only sources - never relaxed, but their epochs wake their owned neighbours - and an
// owned block that changes is marked for the next ESDF halo pack.  Otherwise every block of the submap is relaxed.
template <bool TILED>
__global__ void __launch_bounds__(256) k_esdf_sweep(TsGrid g, EsAux aux, int submap, int sweep, float gamma, float vs) {
  __shared__ EsTile tile;
  if (sweep > 1 && aux.changed[sweep - 1] == 0) return;  // already converged: nothing to do
  const int nb = min(*g.n_blocks, g.max_blocks);
  const float d1 = vs, d2 = sqrtf(2.0f) * vs, d3 = sqrtf(3.0f) * vs;  // dir.norm()*voxel_scale (dense_esdf.py:285)
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    __syncthreads();
    if (threadIdx.x == 0) { tile.active = 0; tile.any_write = 0; }
    __syncthreads();
    if (aux.epoch[b] < -1) continue;  // block of another submap (uniform per CTA)
    if (TILED && g.ghost[b]) continue;  // the owner's values: a source only
    if (threadIdx.x < 27) {
      const int n = aux.nbr[b * 27 + threadIdx.x];
      tile.nbr[threadIdx.x] = n;
      if (n >= 0 && *(volatile int*)&aux.epoch[n] >= sweep - 1) tile.active = 1;  // the wave front reaches this block
    }
    __syncthreads();
    if (!tile.active) continue;
    for (int c = threadIdx.x; c < ES_T3; c += blockDim.x) {
      const int lz = c % ES_T - 1, ly = (c / ES_T) % ES_T - 1, lx = c / (ES_T * ES_T) - 1;
      const int nx = (lx + 16) >> 4, ny = (ly + 16) >> 4, nz = (lz + 16) >> 4;
      const int nbk = tile.nbr[(nx * 3 + ny) * 3 + nz];
      float ev = 0.0f;
      unsigned char cl = ES_UNOBS;
      if (nbk >= 0) {
        const size_t off = (size_t)nbk * TS_B3 + ((((lx & 15) << 4) | (ly & 15)) << 4 | (lz & 15));
        if (g.obs[off]) {
          const float t = g.tw[off].x;
          cl = (fabsf(t) < gamma) ? ES_FIXED : (t > 0.0f ? ES_POS : (t < 0.0f ? ES_NEG : ES_INERT));
          ev = *(volatile float*)&g.esdf[off];
        }
      }
      tile.e[c] = ev;
      tile.cls[c] = cl;
    }
    __syncthreads();
    // relax to local convergence (values only move monotonically, so in-place racy updates are safe)
    for (int iter = 0; iter < 64; ++iter) {
      if (threadIdx.x == 0) tile.changed = 0;
      __syncthreads();
      bool mine = false;
      for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
        const int lx = v >> 8, ly = (v >> 4) & 15, lz = v & 15;
        const int c0 = es_tidx(lx, ly, lz);
        const unsigned char cl = tile.cls[c0];
        if (cl != ES_POS && cl != ES_NEG) continue;
        float best = tile.e[c0];
        const float cur = best;
#pragma unroll
        for (int dx = -1; dx <= 1; dx++)
#pragma unroll
          for (int dy = -1; dy <= 1; dy++)
#pragma unroll
            for (int dz = -1; dz <= 1; dz++) {
              const int nz_ = (dx != 0) + (dy != 0) + (dz != 0);
              if (nz_ == 0) continue;
              const int cn = c0 + (dx * ES_T + dy) * ES_T + dz;
              const unsigned char hc = tile.cls[cn];
              if (!(hc == ES_FIXED || hc == cl)) continue;
              const float dis = nz_ == 1 ? d1 : (nz_ == 2 ? d2 : d3);
              const float he = tile.e[cn];
              if (cl == ES_POS) best = fminf(best, he + dis); else best = fmaxf(best, he - dis);
            }
        if (best != cur) {
          tile.e[c0] = best;
          mine = true;
        }
      }
      if (__any_sync(0xffffffffu, mine) && (threadIdx.x & 31) == 0) tile.changed = 1;
      __syncthreads();
      const int ch = tile.changed;
      if (ch && threadIdx.x == 0) tile.any_write = 1;
      __syncthreads();
      if (!ch) break;
    }
    if (tile.any_write) {
      const size_t base = (size_t)b * TS_B3;
      for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) g.esdf[base + v] = tile.e[es_tidx(v >> 8, (v >> 4) & 15, v & 15)];
      if (threadIdx.x == 0) {
        __threadfence();
        aux.epoch[b] = sweep;
        aux.changed[sweep] = 1;
        if (TILED) aux.xmark[b] = 1;
      }
    }
  }
}

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
      const unsigned m = __ballot_sync(0xffffffffu, want);
      if (!m) continue;
      const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
      unsigned long long rb = 0;
      if (lane == leader) rb = atomicAdd(counter, (unsigned long long)__popc(m));
      rb = __shfl_sync(0xffffffffu, rb, leader);
      const long long row = (long long)(rb + __popc(m & ((1u << lane) - 1)));
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

// mode 0 = incremental when the state allows it (same submap as the last update, no reset / bulk load in between),
// 1 = full recompute.  stats4 (HOST, may be NULL): lower sweeps, raise sweeps, changed voxels, suspect voxels.
extern "C" int tslam_esdf_update2(tslam_tsdf_t* m, int32_t submap, int32_t mode, int32_t* stats4, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  rc = es_alloc(m);
  if (rc) return rc;
  EsAux aux = es_aux(m);
  const float gamma = (float)m->cfg.voxel_scale;     // dense_esdf.py:40
  const float far_v = (float)m->cfg.max_ray_length;  // dense_esdf.py:324
  // (the state a tiled ESDF leaves - ghosts holding their owners' values - is no base for an incremental update)
  const bool full = mode == 1 || m->esdf_full_needed || m->esdf_submap != submap || m->esdf_tiled != 0;
  int h_counts[4] = {0, 0, 0, 0}, n_lower = 0, n_raise = 0;
  m->esdf_tiled = 0;
  TS_CUDA(cudaMemsetAsync(aux.changed, 0, (2 * (ES_MAX_SWEEPS + 2) + 8) * 4, st));  // changed, rchanged, counts
  if (full) {
    k_esdf_init<false><<<m->sm_count * 4, 256, 0, st>>>(m->g, aux, submap, gamma, far_v);
    TS_LAUNCH_CHECK(m);
    rc = es_wave(m, st, aux.changed, ES_GROUP, [&](int k) { k_esdf_sweep<false><<<m->sm_count * 4, 256, 0, st>>>(m->g, aux, submap, k, gamma, m->in.vs); }, &n_lower);
    if (rc) return rc;
  } else {
    k_esdf_prepare<<<m->sm_count * 2, 256, 0, st>>>(m->g, aux, submap);
    TS_LAUNCH_CHECK(m);
    k_esdf_detect<<<m->sm_count * 4, 256, 0, st>>>(m->g, aux, submap, gamma);
    TS_LAUNCH_CHECK(m);
    rc = es_wave(m, st, aux.rchanged, 4, [&](int k) { k_esdf_raise<<<m->sm_count * 4, 256, 0, st>>>(m->g, aux, k, m->in.vs); }, &n_raise);
    if (rc) return rc;
    k_esdf_reinit<<<m->sm_count * 4, 256, 0, st>>>(m->g, aux, gamma, far_v);
    TS_LAUNCH_CHECK(m);
    rc = es_wave(m, st, aux.changed, 4, [&](int k) { k_esdf_sweep<false><<<m->sm_count * 4, 256, 0, st>>>(m->g, aux, submap, k, gamma, m->in.vs); }, &n_lower);
    if (rc) return rc;
    TS_CUDA(cudaMemcpy(h_counts, aux.counts, 16, cudaMemcpyDeviceToHost));
  }
  m->esdf_full_needed = 0;
  m->esdf_submap = submap;
  if (stats4) { stats4[0] = n_lower; stats4[1] = full ? -1 : n_raise; stats4[2] = h_counts[0]; stats4[3] = h_counts[1]; }
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
  EsAux aux = es_aux(m);
  const float gamma = (float)m->cfg.voxel_scale, far_v = (float)m->cfg.max_ray_length;
  int n_lower = 0;
  m->esdf_tiled = 1;
  TS_CUDA(cudaMemsetAsync(aux.changed, 0, (2 * (ES_MAX_SWEEPS + 2) + 8) * 4, st));
  k_esdf_init<true><<<m->sm_count * 4, 256, 0, st>>>(m->g, aux, submap, gamma, far_v);
  TS_LAUNCH_CHECK(m);
  rc = es_wave(m, st, aux.changed, ES_GROUP, [&](int k) { k_esdf_sweep<true><<<m->sm_count * 4, 256, 0, st>>>(m->g, aux, submap, k, gamma, m->in.vs); }, &n_lower);
  if (rc) return rc;
  m->esdf_full_needed = 0;
  m->esdf_submap = submap;
  if (n_sweeps_out) *n_sweeps_out = n_lower;
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
  EsAux aux = es_aux(m);
  const int submap = m->esdf_submap;
  const float gamma = (float)m->cfg.voxel_scale;
  int n_lower = 0;
  TS_CUDA(cudaMemsetAsync(aux.changed, 0, (ES_MAX_SWEEPS + 2) * 4, st));
  k_esdf_rearm<<<m->sm_count * 2, 256, 0, st>>>(m->g, aux);
  TS_LAUNCH_CHECK(m);
  rc = es_wave(m, st, aux.changed, 4, [&](int k) { k_esdf_sweep<true><<<m->sm_count * 4, 256, 0, st>>>(m->g, aux, submap, k, gamma, m->in.vs); }, &n_lower);
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
// (ghost blocks count only after a completed tiled ESDF: they then hold their owners' final values)
__device__ __forceinline__ int esq_block(const TsGrid& g, int submap, int nb_seen, bool ghosts, int bx, int by, int bz) {
  const int b = ts_find(g, ts_pack_key(submap, bx, by, bz));
  return (b >= 0 && b < nb_seen && (ghosts || !g.ghost[b])) ? b : -1;
}
// Trilinear interpolation of the ESDF over the 8 voxels around each point (voxel i centred at i*vs, submap-local frame)
// and the exact partial derivatives of that interpolant.  One thread per point; each distinct corner block is looked
// up once (the corner cube spans 2, 4 or 8 blocks only where i0 & 15 == 15 on some axis).  Invalid (NaN, valid = 0):
// a non-finite coordinate, a corner outside the volume, a corner in an absent / newer block, a corner in a ghost block
// (unless `ghosts`: the field is a completed tiled ESDF), a corner that was unobserved or INERT at the last update.
__global__ void __launch_bounds__(256) k_esdf_query(TsGrid g, EsAux aux, int submap, bool ghosts, long long n, const float* __restrict__ xyz,
                                                     float vs, float* __restrict__ dist, float* __restrict__ grad,
                                                     uint8_t* __restrict__ valid) {
  const int nb_seen = *aux.nb_seen;
  const float qnan = __int_as_float(0x7fc00000);
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    // both corners i0, i0 + 1 inside the volume: the low corner and i0 < N - hN - 1 per axis
    float u[3];
    int c0[3];
    bool ok = esq_low_corner(g, vs, xyz + 3 * q, u, c0) && c0[0] < g.N - g.hN - 1 && c0[1] < g.N - g.hN - 1 && c0[2] < g.Nz - g.hNz - 1;
    float d = qnan, gx = qnan, gy = qnan, gz = qnan;
    if (ok) {
      const int i0 = c0[0], j0 = c0[1], k0 = c0[2];
      const float fx = __fsub_rn(u[0], (float)i0), fy = __fsub_rn(u[1], (float)j0), fz = __fsub_rn(u[2], (float)k0);
      const bool sx = (i0 & TS_BMASK) == TS_BMASK, sy = (j0 & TS_BMASK) == TS_BMASK, sz = (k0 & TS_BMASK) == TS_BMASK;
      const int x0 = i0 >> TS_BSHIFT, y0 = j0 >> TS_BSHIFT, z0 = k0 >> TS_BSHIFT;
      // b[dx*4 + dy*2 + dz]: block of corner (i0+dx, j0+dy, k0+dz); a corner that shares its block with a lower one reuses it
      int b[8];
      b[0] = esq_block(g, submap, nb_seen, ghosts, x0, y0, z0);
      b[1] = sz ? esq_block(g, submap, nb_seen, ghosts, x0, y0, z0 + 1) : b[0];
      b[2] = sy ? esq_block(g, submap, nb_seen, ghosts, x0, y0 + 1, z0) : b[0];
      b[3] = sy ? (sz ? esq_block(g, submap, nb_seen, ghosts, x0, y0 + 1, z0 + 1) : b[2]) : b[1];
      b[4] = sx ? esq_block(g, submap, nb_seen, ghosts, x0 + 1, y0, z0) : b[0];
      b[5] = sx ? (sz ? esq_block(g, submap, nb_seen, ghosts, x0 + 1, y0, z0 + 1) : b[4]) : b[1];
      b[6] = sx ? (sy ? esq_block(g, submap, nb_seen, ghosts, x0 + 1, y0 + 1, z0) : b[4]) : b[2];
      b[7] = sx ? (sy ? (sz ? esq_block(g, submap, nb_seen, ghosts, x0 + 1, y0 + 1, z0 + 1) : b[6]) : b[5]) : b[3];
      float e[8];
#pragma unroll
      for (int c = 0; c < 8; c++) {
        ok &= b[c] >= 0;
        e[c] = 0.0f;
      }
      if (ok) {
#pragma unroll
        for (int c = 0; c < 8; c++) {
          const size_t off = (size_t)b[c] * TS_B3 + ts_voxel_off(i0 + (c >> 2), j0 + ((c >> 1) & 1), k0 + (c & 1));
          const unsigned char cl = aux.cls[off] & ES_CLS;
          ok &= cl == ES_FIXED || cl == ES_POS || cl == ES_NEG;
          e[c] = g.esdf[off];
        }
      }
      if (ok) {
        esq_interp(e, fx, fy, fz, vs, d, gx, gy, gz);
      } else {
        d = gx = gy = gz = qnan;
      }
    }
    dist[q] = d;
    grad[3 * q] = gx; grad[3 * q + 1] = gy; grad[3 * q + 2] = gz;
    valid[q] = ok ? 1 : 0;
  }
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
