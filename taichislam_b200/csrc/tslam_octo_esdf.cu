// libtslam.so - occupancy ESDF of a log-odds Octomap (DESIGN.md section 7, "Occupancy ESDF"), kept incrementally.
//
// Per submap, as of one update.  Classes come from the cnt plane: OCC = known and L > l_occ, FREE = known and
// L <= l_occ, UNKNOWN = not known.  A FREE voxel starts at +D, an OCC voxel at -D; UNKNOWN voxels are neither sources
// nor targets.  Relaxation over the known 26-neighbours h of v (edge cost c = vs * {1, sqrt 2, sqrt 3}):
//   FREE v: E(v) = min(E(v), h OCC  ?  c : E(h) + c)
//   OCC  v: E(v) = max(E(v), h FREE ? -c : E(h) - c)
// to the fixed point (f32 min/+ is monotone: unique, independent of the schedule).
//
// The scheme is the TSDF ESDF's (tslam_esdf.cu) on 8^3 blocks: a CTA stages its block plus a one-voxel halo (10^3) in
// shared memory and relaxes it to local convergence; sweep k runs the blocks with a neighbour stamped >= k-1.  An
// incremental update runs
//   1. detect  (blocks k_octo_lo_apply updated since the last update): voxels whose class changed -> CHANGED;
//   2. raise   a voxel whose value EQUALS the candidate a flagged neighbour offered it at the old fixed point (old
//              class, old value; the cross-class candidates are the constants +-c) may have been derived from it ->
//              SUSPECT, to closure;
//   3. re-init flagged voxels take their new class and seed;
//   4. lower   the sweep, from the re-initialised blocks.
// Unflagged values stay attainable upper bounds, so the lower wave ends at the full recompute's fixed point, bit for
// bit (DESIGN.md section 7 gives the argument).
#include <cmath>
#include <cstring>
#include "tslam_esdf_common.cuh"

#define OE_T 10
#define OE_T3 (OE_T * OE_T * OE_T)
#define OE_THREADS 128

struct OeAux {
  float* e;            // [max_blocks*512] the field
  unsigned char* cls;  // [max_blocks*512] class at the last update (+ flags during an update)
  int* nbr;            // [max_blocks*27] neighbour block indices (-1 = absent)
  int* epoch;          // [max_blocks] lower wave: last sweep in which the block changed (< -1: block of another submap)
  int* repoch;         // [max_blocks] raise wave: last raise sweep in which the block gained flags (-1: none)
  int* changed;        // [ES_MAX_SWEEPS+2] changed[k] != 0 <=> lower sweep k changed something
  int* rchanged;       // [ES_MAX_SWEEPS+2]
  int* counts;         // [8] changed voxels, suspect voxels, re-initialised blocks, (spare), nb_seen, nb_prev
  int* nb_seen;        // blocks in the pool when the last update ran (bump allocation: higher indices are newer)
  int* nb_prev;        // nb_seen of the update before (incremental update: blocks >= it are new)
};

__device__ __forceinline__ float oe_seed(unsigned char c, float D) { return c == OC_FREE ? D : (c == OC_OCC ? -D : 0.0f); }
__device__ __forceinline__ int oe_tidx(int lx, int ly, int lz) { return ((lx + 1) * OE_T + (ly + 1)) * OE_T + (lz + 1); }

// full update: every block of the submap seeded, neighbour table built, epoch 0 (a wave source)
__global__ void __launch_bounds__(OE_THREADS) k_octo_esdf_init(OcGrid g, OeAux a, int submap, int l_occ, float D) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.nb_seen = nb;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (threadIdx.x == 0) a.epoch[b] = (s == submap) ? 0 : -1000000;
    if (s != submap) continue;
    if (threadIdx.x < 27) {
      const int dx = threadIdx.x / 9 - 1, dy = (threadIdx.x / 3) % 3 - 1, dz = threadIdx.x % 3 - 1;
      a.nbr[b * 27 + threadIdx.x] = ts_find(g, ts_pack_key(s, bx + dx, by + dy, bz + dz));
    }
    const size_t base = (size_t)b * OC_B3;
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
      const unsigned char c = oc_class(g.cnt[base + v], l_occ);
      a.e[base + v] = oe_seed(c, D);
      a.cls[base + v] = c;
    }
  }
}

// incremental update: neighbour table of every block of the submap, epochs reset; a block allocated since the last
// update starts UNKNOWN (whatever its pool slot held before a reset), so detect sees each of its known voxels change
__global__ void __launch_bounds__(256) k_octo_esdf_prepare(OcGrid g, OeAux a, int submap) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  const int nb_prev = *a.nb_prev;
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.nb_seen = nb;
  const int w = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31, nw = (gridDim.x * 256) >> 5;
  for (int b = w; b < nb; b += nw) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (lane == 0) { a.epoch[b] = (s == submap) ? -1 : -1000000; a.repoch[b] = -1; }
    if (s != submap) continue;
    if (lane < 27) {
      const int dx = lane / 9 - 1, dy = (lane / 3) % 3 - 1, dz = lane % 3 - 1;
      a.nbr[b * 27 + lane] = ts_find(g, ts_pack_key(s, bx + dx, by + dy, bz + dz));
    }
    if (b >= nb_prev) {
      const size_t base = (size_t)b * OC_B3;
      for (int v = lane; v < OC_B3; v += 32) { a.cls[base + v] = OC_UNK; a.e[base + v] = 0.0f; }
    }
  }
}

// 1. detect: blocks updated since the last update
__global__ void __launch_bounds__(OE_THREADS) k_octo_esdf_detect(OcGrid g, OeAux a, int* dirty, int l_occ) {
  __shared__ int s_any;
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (!dirty[b] || a.epoch[b] < -1) continue;  // (uniform per CTA)
    __syncthreads();
    if (threadIdx.x == 0) s_any = 0;
    __syncthreads();
    const size_t base = (size_t)b * OC_B3;
    int mine = 0;
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
      const unsigned char oc = a.cls[base + v] & ES_CLS;
      if (oc_class(g.cnt[base + v], l_occ) != oc) { a.cls[base + v] = oc | ES_CH; mine++; }
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_any, mine);
    __syncthreads();
    if (threadIdx.x == 0) {
      dirty[b] = 0;
      if (s_any) { a.repoch[b] = 0; atomicAdd(&a.counts[0], s_any); }
    }
  }
}

struct OeTile {
  float e[OE_T3];
  unsigned char cls[OE_T3];
  int nbr[27];
  int active, changed, any_write;
};

// block + one-voxel halo into shared memory (absent neighbour blocks read UNKNOWN)
__device__ __forceinline__ void oe_stage(const OeAux& a, OeTile& tile) {
  for (int c = threadIdx.x; c < OE_T3; c += blockDim.x) {
    const int lz = c % OE_T - 1, ly = (c / OE_T) % OE_T - 1, lx = c / (OE_T * OE_T) - 1;
    const int nbk = tile.nbr[(((lx + 8) >> 3) * 3 + ((ly + 8) >> 3)) * 3 + ((lz + 8) >> 3)];
    float ev = 0.0f;
    unsigned char cl = OC_UNK;
    if (nbk >= 0) {
      const size_t off = (size_t)nbk * OC_B3 + oc_voxel_off(lx, ly, lz);
      cl = *(volatile unsigned char*)&a.cls[off];
      ev = *(volatile float*)&a.e[off];
    }
    tile.e[c] = ev;
    tile.cls[c] = cl;
  }
}

// 2. raise wave: flag the voxels that may have been derived from a flagged neighbour
__global__ void __launch_bounds__(OE_THREADS) k_octo_esdf_raise(OcGrid g, OeAux a, int sweep, float vs) {
  __shared__ OeTile tile;
  if (sweep > 1 && a.rchanged[sweep - 1] == 0) return;
  const int nb = min(*g.n_blocks, g.max_blocks);
  const float d1 = vs, d2 = sqrtf(2.0f) * vs, d3 = sqrtf(3.0f) * vs;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    __syncthreads();
    if (threadIdx.x == 0) { tile.active = 0; tile.any_write = 0; }
    __syncthreads();
    if (a.epoch[b] < -1) continue;
    if (threadIdx.x < 27) {
      const int n = a.nbr[b * 27 + threadIdx.x];
      tile.nbr[threadIdx.x] = n;
      if (n >= 0 && *(volatile int*)&a.repoch[n] >= sweep - 1) tile.active = 1;
    }
    __syncthreads();
    if (!tile.active) continue;
    oe_stage(a, tile);  // old values: nothing writes the field during the raise wave
    __syncthreads();
    for (int iter = 0; iter < 64; ++iter) {
      if (threadIdx.x == 0) tile.changed = 0;
      __syncthreads();
      bool mine = false;
      for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
        const int c0 = oe_tidx(v >> 6, (v >> 3) & 7, v & 7);
        const unsigned char cl = tile.cls[c0];
        if (cl != OC_FREE && cl != OC_OCC) continue;  // flagged or unknown: nothing to decide
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
              const int cn = c0 + (dx * OE_T + dy) * OE_T + dz;
              const unsigned char hf = tile.cls[cn];
              const unsigned char hc = hf & ES_CLS;  // the neighbour's class at the last update
              if (!(hf & (ES_CH | ES_SU)) || hc == OC_UNK) continue;
              const float dis = nz_ == 1 ? d1 : (nz_ == 2 ? d2 : d3);
              const float he = tile.e[cn];
              const float cand = (cl == OC_FREE) ? (hc == OC_OCC ? dis : he + dis) : (hc == OC_FREE ? -dis : he - dis);
              hit |= cand == cur;
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
      const size_t base = (size_t)b * OC_B3;
      for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
        const unsigned char cl = tile.cls[oe_tidx(v >> 6, (v >> 3) & 7, v & 7)];
        if (cl & ES_SU) a.cls[base + v] = cl;
      }
      if (threadIdx.x == 0) {
        __threadfence();
        a.repoch[b] = sweep;
        a.rchanged[sweep] = 1;
      }
    }
  }
}

// 3. re-initialise flagged voxels; their blocks start the lower wave (epoch 0)
__global__ void __launch_bounds__(OE_THREADS) k_octo_esdf_reinit(OcGrid g, OeAux a, int l_occ, float D) {
  __shared__ int s_n;
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (a.repoch[b] < 0) continue;  // no flagged voxel in this block (uniform per CTA)
    __syncthreads();
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const size_t base = (size_t)b * OC_B3;
    int nsu = 0;
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
      const unsigned char c = a.cls[base + v];
      if (!(c & (ES_CH | ES_SU))) continue;
      const unsigned char nc = oc_class(g.cnt[base + v], l_occ);
      a.e[base + v] = oe_seed(nc, D);
      a.cls[base + v] = nc;
      nsu += (c & ES_SU) ? 1 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) nsu += __shfl_xor_sync(0xffffffffu, nsu, o);
    if ((threadIdx.x & 31) == 0 && nsu) atomicAdd(&s_n, nsu);
    __syncthreads();
    if (threadIdx.x == 0) {
      a.epoch[b] = 0;
      if (s_n) atomicAdd(&a.counts[1], s_n);
      atomicAdd(&a.counts[2], 1);
    }
  }
}

// 4. lower wave (and the whole of a full update): relax the blocks the wave front reaches to local convergence
__global__ void __launch_bounds__(OE_THREADS) k_octo_esdf_sweep(OcGrid g, OeAux a, int sweep, float vs) {
  __shared__ OeTile tile;
  if (sweep > 1 && a.changed[sweep - 1] == 0) return;  // already converged: nothing to do
  const int nb = min(*g.n_blocks, g.max_blocks);
  const float d1 = vs, d2 = sqrtf(2.0f) * vs, d3 = sqrtf(3.0f) * vs;  // the edge costs of k_esdf_sweep
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    __syncthreads();
    if (threadIdx.x == 0) { tile.active = 0; tile.any_write = 0; }
    __syncthreads();
    if (a.epoch[b] < -1) continue;  // block of another submap (uniform per CTA)
    if (threadIdx.x < 27) {
      const int n = a.nbr[b * 27 + threadIdx.x];
      tile.nbr[threadIdx.x] = n;
      if (n >= 0 && *(volatile int*)&a.epoch[n] >= sweep - 1) tile.active = 1;  // the wave front reaches this block
    }
    __syncthreads();
    if (!tile.active) continue;
    oe_stage(a, tile);
    __syncthreads();
    // relax to local convergence (values only move monotonically, so in-place racy updates are safe)
    for (int iter = 0; iter < 64; ++iter) {
      if (threadIdx.x == 0) tile.changed = 0;
      __syncthreads();
      bool mine = false;
      for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
        const int c0 = oe_tidx(v >> 6, (v >> 3) & 7, v & 7);
        const unsigned char cl = tile.cls[c0];
        if (cl == OC_UNK) continue;
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
              const int cn = c0 + (dx * OE_T + dy) * OE_T + dz;
              const unsigned char hc = tile.cls[cn];
              if (hc == OC_UNK) continue;
              const float dis = nz_ == 1 ? d1 : (nz_ == 2 ? d2 : d3);
              const float he = tile.e[cn];
              if (cl == OC_FREE) best = fminf(best, hc == OC_OCC ? dis : he + dis);
              else best = fmaxf(best, hc == OC_FREE ? -dis : he - dis);
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
      const size_t base = (size_t)b * OC_B3;
      for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) a.e[base + v] = tile.e[oe_tidx(v >> 6, (v >> 3) & 7, v & 7)];
      if (threadIdx.x == 0) {
        __threadfence();
        a.epoch[b] = sweep;
        a.changed[sweep] = 1;
      }
    }
  }
}

// (ijk, E) of every voxel known at the last update, in the blocks that update saw
__global__ void __launch_bounds__(OE_THREADS) k_octo_esdf_gather(OcGrid g, OeAux a, int submap, long long cap, int32_t* idx, float* esdf,
                                                                 unsigned long long* counter) {
  const int nb = min(*a.nb_seen, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap) continue;  // (uniform per CTA)
    const size_t base = (size_t)b * OC_B3;
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
      const bool want = (a.cls[base + v] & ES_CLS) != OC_UNK;
      const long long row = oc_warp_append(want, counter);
      if (want && row < cap) {
        idx[3 * row] = bx * OC_B + (v >> 6);
        idx[3 * row + 1] = by * OC_B + ((v >> 3) & 7);
        idx[3 * row + 2] = bz * OC_B + (v & 7);
        esdf[row] = a.e[base + v];
      }
    }
  }
}

__device__ __forceinline__ int oeq_block(const OcGrid& g, int submap, int nb_seen, int bx, int by, int bz) {
  const int b = ts_find(g, ts_pack_key(submap, bx, by, bz));
  return (b >= 0 && b < nb_seen) ? b : -1;
}

// Trilinear interpolation over the 8 voxels around each point and the exact gradient of that interpolant, as
// k_esdf_query.  Invalid (NaN, valid = 0): a non-finite coordinate, a corner outside the volume, a corner in an absent or
// newer block, a corner that was UNKNOWN at the last update.
__global__ void __launch_bounds__(256) k_octo_esdf_query(OcGrid g, OeAux a, int submap, long long n, const float* __restrict__ xyz,
                                                         float vs, float* __restrict__ dist, float* __restrict__ grad,
                                                         uint8_t* __restrict__ valid) {
  const int nb_seen = *a.nb_seen;
  const float qnan = __int_as_float(0x7fc00000);
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    float u[3];
    int c0[3];
    bool ok = esq_low_corner(g, vs, xyz + 3 * q, u, c0) && c0[0] < g.N - g.hN - 1 && c0[1] < g.N - g.hN - 1 && c0[2] < g.Nz - g.hNz - 1;
    float d = qnan, gx = qnan, gy = qnan, gz = qnan;
    if (ok) {
      const int i0 = c0[0], j0 = c0[1], k0 = c0[2];
      const float fx = __fsub_rn(u[0], (float)i0), fy = __fsub_rn(u[1], (float)j0), fz = __fsub_rn(u[2], (float)k0);
      const bool sx = (i0 & OC_BMASK) == OC_BMASK, sy = (j0 & OC_BMASK) == OC_BMASK, sz = (k0 & OC_BMASK) == OC_BMASK;
      const int x0 = i0 >> OC_BSHIFT, y0 = j0 >> OC_BSHIFT, z0 = k0 >> OC_BSHIFT;
      // b[dx*4 + dy*2 + dz]: block of corner (i0+dx, j0+dy, k0+dz); a corner that shares its block with a lower one reuses it
      int b[8];
      b[0] = oeq_block(g, submap, nb_seen, x0, y0, z0);
      b[1] = sz ? oeq_block(g, submap, nb_seen, x0, y0, z0 + 1) : b[0];
      b[2] = sy ? oeq_block(g, submap, nb_seen, x0, y0 + 1, z0) : b[0];
      b[3] = sy ? (sz ? oeq_block(g, submap, nb_seen, x0, y0 + 1, z0 + 1) : b[2]) : b[1];
      b[4] = sx ? oeq_block(g, submap, nb_seen, x0 + 1, y0, z0) : b[0];
      b[5] = sx ? (sz ? oeq_block(g, submap, nb_seen, x0 + 1, y0, z0 + 1) : b[4]) : b[1];
      b[6] = sx ? (sy ? oeq_block(g, submap, nb_seen, x0 + 1, y0 + 1, z0) : b[4]) : b[2];
      b[7] = sx ? (sy ? (sz ? oeq_block(g, submap, nb_seen, x0 + 1, y0 + 1, z0 + 1) : b[6]) : b[5]) : b[3];
      float e[8];
#pragma unroll
      for (int c = 0; c < 8; c++) {
        ok &= b[c] >= 0;
        e[c] = 0.0f;
      }
      if (ok) {
#pragma unroll
        for (int c = 0; c < 8; c++) {
          const size_t off = (size_t)b[c] * OC_B3 + oc_voxel_off(i0 + (c >> 2), j0 + ((c >> 1) & 1), k0 + (c & 1));
          ok &= (a.cls[off] & ES_CLS) != OC_UNK;
          e[c] = a.e[off];
        }
      }
      if (ok) esq_interp(e, fx, fy, fz, vs, d, gx, gy, gz);
      else d = gx = gy = gz = qnan;
    }
    dist[q] = d;
    grad[3 * q] = gx; grad[3 * q + 1] = gy; grad[3 * q + 2] = gz;
    valid[q] = ok ? 1 : 0;
  }
}

// ---- host side -----------------------------------------------------------------------------------------------------
// bytes per pool block: field 2048 + class 512 + neighbour table 108 + epoch, raise epoch, dirty flag 12 = 2680
static size_t oe_bytes(size_t nb) { return nb * (OC_B3 * 5 + 30 * 4) + (2 * (ES_MAX_SWEEPS + 2) + 8) * 4; }

static OeAux oe_aux(tslam_octo* m) {
  const size_t nb = (size_t)m->g.max_blocks;
  OeAux a;
  a.e = (float*)m->esdf_mem;
  a.nbr = (int*)(a.e + nb * OC_B3);
  a.epoch = a.nbr + nb * 27;
  a.repoch = a.epoch + nb;
  // (esdf_dirty = a.repoch + nb)
  a.changed = a.repoch + 2 * nb;
  a.rchanged = a.changed + (ES_MAX_SWEEPS + 2);
  a.counts = a.rchanged + (ES_MAX_SWEEPS + 2);
  a.nb_seen = a.counts + 4;
  a.nb_prev = a.counts + 5;
  a.cls = (unsigned char*)(a.counts + 8);
  return a;
}

static int oe_alloc(tslam_octo* m) {
  if (m->esdf_mem) return TSLAM_OK;
  const size_t bytes = oe_bytes((size_t)m->g.max_blocks);
  TS_CUDA(cudaMalloc(&m->esdf_mem, bytes));
  TS_CUDA(cudaMemset(m->esdf_mem, 0, bytes));
  m->esdf_dirty = oe_aux(m).repoch + m->g.max_blocks;
  return TSLAM_OK;
}

int oc_esdf_free(tslam_octo* m) {
  if (m->esdf_mem) cudaFree(m->esdf_mem);
  m->esdf_mem = nullptr;
  m->esdf_dirty = nullptr;
  return TSLAM_OK;
}

int oc_esdf_field(tslam_octo* m, int32_t submap, const char* what, OcEsdfField* f) {
  int rc = oc_track_readable(m, m->esdf_track, submap, what, "tslam_octo_esdf_update");
  if (rc) return rc;
  const OeAux a = oe_aux(m);
  f->e = a.e;
  f->cls = a.cls;
  f->nb_seen = a.nb_seen;
  f->D = m->esdf_D;
  f->free_cls = OC_FREE;
  f->cls_mask = ES_CLS;
  return TSLAM_OK;
}

// mode 0 = incremental when the state allows it (same submap and D as the last update, no reset / fusion in between),
// 1 = full recompute.  stats4 (HOST, may be NULL): lower sweeps, raise sweeps (-1 = full), changed voxels, suspect voxels.
extern "C" int tslam_octo_esdf_update(tslam_octo_t* m, int32_t submap, float max_dist, int32_t mode, int32_t* stats4, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  int rc = oc_logodds_submap(m, submap, "tslam_octo_esdf_update", "the occupancy ESDF");
  if (rc) return rc;
  if (!(std::isfinite(max_dist) && max_dist > 0.0f)) {
    ts_set_error("tslam_octo_esdf_update: max_dist must be finite and > 0 (got %g)", (double)max_dist);
    return TSLAM_E_INVALID;
  }
  if (mode != 0 && mode != 1) { ts_set_error("tslam_octo_esdf_update: mode must be 0 (incremental) or 1 (full)"); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  rc = oe_alloc(m);
  if (rc) return rc;
  OeAux a = oe_aux(m);
  const int l_occ = m->lo.l_occ;
  const float vs = m->in.vs;
  const bool full = mode == 1 || !m->esdf_track.ready || m->esdf_track.submap != submap ||
                    memcmp(&m->esdf_D, &max_dist, sizeof(float)) != 0;
  int h_counts[4] = {0, 0, 0, 0}, n_lower = 0, n_raise = 0;
  m->esdf_track.ready = 0;  // until this update has completed
  TS_CUDA(cudaMemsetAsync(a.changed, 0, (2 * (ES_MAX_SWEEPS + 2) + 4) * 4, st));  // changed, rchanged, counts[0..3]
  const int grid = m->sm_count * 8;
  if (full) {
    TS_CUDA(cudaMemsetAsync(m->esdf_dirty, 0, (size_t)m->g.max_blocks * 4, st));
    k_octo_esdf_init<<<grid, OE_THREADS, 0, st>>>(m->g, a, submap, l_occ, max_dist);
    TS_LAUNCH_CHECK(m);
    rc = es_wave(m, st, a.changed, ES_GROUP, [&](int k) { k_octo_esdf_sweep<<<grid, OE_THREADS, 0, st>>>(m->g, a, k, vs); }, &n_lower);
    if (rc) return rc;
  } else {
    TS_CUDA(cudaMemcpyAsync(a.nb_prev, a.nb_seen, 4, cudaMemcpyDeviceToDevice, st));
    k_octo_esdf_prepare<<<m->sm_count * 2, 256, 0, st>>>(m->g, a, submap);
    TS_LAUNCH_CHECK(m);
    k_octo_esdf_detect<<<grid, OE_THREADS, 0, st>>>(m->g, a, m->esdf_dirty, l_occ);
    TS_LAUNCH_CHECK(m);
    rc = es_wave(m, st, a.rchanged, 4, [&](int k) { k_octo_esdf_raise<<<grid, OE_THREADS, 0, st>>>(m->g, a, k, vs); }, &n_raise);
    if (rc) return rc;
    k_octo_esdf_reinit<<<grid, OE_THREADS, 0, st>>>(m->g, a, l_occ, max_dist);
    TS_LAUNCH_CHECK(m);
    rc = es_wave(m, st, a.changed, 4, [&](int k) { k_octo_esdf_sweep<<<grid, OE_THREADS, 0, st>>>(m->g, a, k, vs); }, &n_lower);
    if (rc) return rc;
    TS_CUDA(cudaMemcpy(h_counts, a.counts, 16, cudaMemcpyDeviceToHost));
  }
  m->esdf_track = OcTrack{1, submap};
  m->esdf_D = max_dist;
  if (stats4) { stats4[0] = n_lower; stats4[1] = full ? -1 : n_raise; stats4[2] = h_counts[0]; stats4[3] = h_counts[1]; }
  return TSLAM_OK;
}

extern "C" int tslam_octo_esdf_gather(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, float* esdf, int64_t* n_out,
                                      void* stream) {
  if (!m || !n_out || cap < 0 || (cap > 0 && (!idx || !esdf))) return TSLAM_E_INVALID;
  const char* what = "tslam_octo_esdf_gather";
  int rc = oc_track_readable(m, m->esdf_track, submap, what, "tslam_octo_esdf_update");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return oc_counted_gather(m, st, [&](unsigned long long* ctr) {
    k_octo_esdf_gather<<<m->sm_count * 8, OE_THREADS, 0, st>>>(m->g, oe_aux(m), submap, cap, idx, esdf, ctr);
  }, cap, n_out, what);
}

extern "C" int tslam_octo_esdf_query(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, float* dist, float* grad,
                                     uint8_t* valid, void* stream) {
  if (!m || n < 0 || (n && (!xyz || !dist || !grad || !valid))) return TSLAM_E_INVALID;
  int rc = oc_track_readable(m, m->esdf_track, submap, "tslam_octo_esdf_query", "tslam_octo_esdf_update");
  if (rc || n == 0) return rc;
  k_octo_esdf_query<<<oc_grid(n, 256, m->sm_count * 16), 256, 0, (cudaStream_t)stream>>>(m->g, oe_aux(m), submap, n, xyz, m->in.vs, dist,
                                                                                         grad, valid);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
