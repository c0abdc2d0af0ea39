// The block wavefront shared by the two ESDFs of libtslam.so: the TSDF ESDF (tslam_esdf.cu, 16^3 blocks) and the
// occupancy ESDF of the log-odds Octomap (tslam_octo_esdf.cu, 8^3 blocks).  Both keep a field and a class byte per voxel
// and run the same scheme, written here once:
//   full update  every block of the submap seeded and made a wave source, then the lower wave;
//   incremental  detect (voxels of dirty blocks whose class changed -> CHANGED), raise wave (a target voxel whose value
//                EQUALS the candidate a flagged neighbour offered it at the old fixed point may have been derived from
//                it -> SUSPECT, to closure; f32 equality is exact), re-init of the flagged voxels, then the lower wave
//                from the re-initialised blocks;
//   a wave       sweeps over the blocks; sweep k runs the blocks with a neighbour (26 + self) stamped >= k-1: a CTA
//                stages its block plus a one-voxel halo in shared memory, iterates to local convergence (ballot-voted,
//                at most 64 iterations), writes back and stamps the block with k when anything changed.
// Voxels of one of the two target classes relax over their 26 neighbours (edge cost c = vs * {1, sqrt 2, sqrt 3}): a
// MIN_SIDE voxel takes the least candidate, a MAX_SIDE voxel the greatest.  f32 min/+ is monotone, so the fixed point
// is unique; unflagged values stay attainable upper bounds, so an incremental update ends at the full recompute's field.
//
// What differs between the two ESDFs is a rule type P, a small struct passed to the kernels by value: the grid `g`, the
// state `a` (cls, nbr, epoch, repoch, changed, rchanged, counts, nb_seen), the update's parameters, and
//   SHIFT, THREADS, GRID    block edge 1 << SHIFT; threads per CTA and CTAs per SM of the per-block kernels
//   COUNTS_CLEARED          words of a.counts cleared by every update
//   NONE, MIN_SIDE, MAX_SIDE  class of a voxel of an absent block; the two target classes
//   field(), dirty()        the field plane; the per-block flags "written since the last update"
//   seed(off, c)            class c of voxel off now, and its seed value (init, re-init)
//   moved(off, oc)          detect: voxel off must be re-initialised (its class at the last update is oc)
//   stage(off, e, c)        lower wave: value and class of a voxel of a present block
//   target(c), source(c, h) lower wave: a voxel of class c relaxes; a neighbour of class h offers it a candidate
//   raise_source(h)         raise wave: a flagged neighbour of old class h offered a candidate
//   cand_min / cand_max(h, e, c)  candidate of a neighbour (class h, value e) at edge cost c to a MIN_SIDE / MAX_SIDE voxel
//   GHOSTS, valid(c)        queries: the ghost rule of the TSDF's tiled map applies; a corner of class c has a value
//   init_done(b), prepare_block(b, lane)  extras of one ESDF at the end of a block in init / prepare
#pragma once
#include "tslam_internal.cuh"

#define ES_GROUP 6       // sweeps enqueued per host synchronisation (full update)
#define ES_MAX_SWEEPS 4096
#define ES_CH 0x40   // class-byte flags of an incremental update: CHANGED (detect) / SUSPECT (raise wave)
#define ES_SU 0x80
#define ES_CLS 0x0F

// One wave (raise or lower) to convergence: sweeps are enqueued in groups, a sweep whose predecessor changed nothing
// returns at once; the host reads ONE flag per group.  Returns the number of sweeps that did something + 1 in *n_out.
// M = tslam_tsdf or tslam_octo (anything with a launch counter).
template <class M, class Launch>
static int es_wave(M* m, cudaStream_t st, int* flags, int group, Launch launch, int* n_out) {
  int sweeps = 0;
  for (;;) {
    for (int q = 0; q < group && sweeps < ES_MAX_SWEEPS; q++) { sweeps++; launch(sweeps); TS_LAUNCH_CHECK(m); }
    int changed = 0;
    TS_CUDA(cudaMemcpyAsync(&changed, flags + sweeps, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
    if (!changed || sweeps >= ES_MAX_SWEEPS) break;
  }
  if (n_out) {
    static int h_changed[ES_MAX_SWEEPS + 2];
    TS_CUDA(cudaMemcpy(h_changed, flags, (size_t)(sweeps + 1) * 4, cudaMemcpyDeviceToHost));
    int k = 1;
    while (k <= sweeps && h_changed[k]) k++;
    *n_out = k;
  }
  return TSLAM_OK;
}

// lerp(a, b, t) = a + t*(b - a), rounded step by step (never contracted to an FMA): tests/esdf_query_reference.py
__device__ __forceinline__ float esq_lerp(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a))); }

// Trilinear interpolant of the 8 corner values e[dx*4 + dy*2 + dz] at fractions (fx, fy, fz) of the cell: along x, then
// y, then z
__device__ __forceinline__ float esq_value(const float e[8], float fx, float fy, float fz) {
  const float c00 = esq_lerp(e[0], e[4], fx), c01 = esq_lerp(e[1], e[5], fx);
  const float c10 = esq_lerp(e[2], e[6], fx), c11 = esq_lerp(e[3], e[7], fx);
  return esq_lerp(esq_lerp(c00, c10, fy), esq_lerp(c01, c11, fy), fz);
}

// esq_value and the interpolant's exact partial derivatives (tests/esdf_query_reference.py states the same arithmetic
// operation by operation).
__device__ __forceinline__ void esq_interp(const float e[8], float fx, float fy, float fz, float vs, float& d, float& gx, float& gy,
                                           float& gz) {
  d = esq_value(e, fx, fy, fz);
  // d/dx: the four x-differences along y, then z
  const float ax00 = __fsub_rn(e[4], e[0]), ax01 = __fsub_rn(e[5], e[1]), ax10 = __fsub_rn(e[6], e[2]), ax11 = __fsub_rn(e[7], e[3]);
  gx = __fdiv_rn(esq_lerp(esq_lerp(ax00, ax10, fy), esq_lerp(ax01, ax11, fy), fz), vs);
  // d/dy: the four y-differences along x, then z
  const float ay00 = __fsub_rn(e[2], e[0]), ay01 = __fsub_rn(e[3], e[1]), ay10 = __fsub_rn(e[6], e[4]), ay11 = __fsub_rn(e[7], e[5]);
  gy = __fdiv_rn(esq_lerp(esq_lerp(ay00, ay10, fx), esq_lerp(ay01, ay11, fx), fz), vs);
  // d/dz: the four z-differences along x, then y
  const float az00 = __fsub_rn(e[1], e[0]), az01 = __fsub_rn(e[3], e[2]), az10 = __fsub_rn(e[5], e[4]), az11 = __fsub_rn(e[7], e[6]);
  gz = __fdiv_rn(esq_lerp(esq_lerp(az00, az10, fx), esq_lerp(az01, az11, fx), fy), vs);
}

// voxel (i, j, k) within its block of edge 1 << S
template <int S>
__device__ __forceinline__ int es_voff(int i, int j, int k) {
  constexpr int M = (1 << S) - 1;
  return (((i & M) << S) | (j & M)) << S | (k & M);
}
// voxel v of the block -> its cell in the (B+2)^3 tile
template <int S>
__device__ __forceinline__ int es_tidx(int v) {
  constexpr int M = (1 << S) - 1, T = (1 << S) + 2;
  return (((v >> 2 * S) + 1) * T + (((v >> S) & M) + 1)) * T + ((v & M) + 1);
}
// f(tile cell, edge cost) for the 26 neighbours of tile cell c0
template <int T, class F>
__device__ __forceinline__ void es_for_26(int c0, float d1, float d2, float d3, F f) {
#pragma unroll
  for (int dx = -1; dx <= 1; dx++)
#pragma unroll
    for (int dy = -1; dy <= 1; dy++)
#pragma unroll
      for (int dz = -1; dz <= 1; dz++) {
        const int nz_ = (dx != 0) + (dy != 0) + (dz != 0);
        if (nz_ == 0) continue;
        f(c0 + (dx * T + dy) * T + dz, nz_ == 1 ? d1 : (nz_ == 2 ? d2 : d3));
      }
}
// neighbour t (0..26, dx-major) of block (bx, by, bz) of submap s: its pool index or -1
template <class G>
__device__ __forceinline__ int es_nbr(const G& g, int s, int bx, int by, int bz, int t) {
  const int dx = t / 9 - 1, dy = (t / 3) % 3 - 1, dz = t % 3 - 1;
  return ts_find(g, ts_pack_key(s, bx + dx, by + dy, bz + dz));
}
// add every thread's n into *s_sum (shared), one atomic per warp
__device__ __forceinline__ void es_cta_add(int n, int* s_sum) {
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(s_sum, n);
}

// full update: every block of the submap seeded, neighbour table built, epoch 0 (a wave source).  TILED (the TSDF's
// tslam_esdf_tiled_begin): every owned block of the submap is marked for the first ESDF halo pack.
template <class P, bool TILED>
__global__ void __launch_bounds__(P::THREADS) es_k_init(P p) {
  constexpr int B3 = 1 << 3 * P::SHIFT;
  const int nb = min(*p.g.n_blocks, p.g.max_blocks);
  if (blockIdx.x == 0 && threadIdx.x == 0) *p.a.nb_seen = nb;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(p.g.block_key[b], s, bx, by, bz);
    if (threadIdx.x == 0) p.a.epoch[b] = (s == p.submap) ? 0 : -1000000;
    if constexpr (TILED) {
      if (threadIdx.x == 0) p.a.xmark[b] = (s == p.submap && !p.g.ghost[b]) ? 1 : 0;
    }
    if (s != p.submap) continue;
    if (threadIdx.x < 27) p.a.nbr[b * 27 + threadIdx.x] = es_nbr(p.g, s, bx, by, bz, threadIdx.x);
    const size_t base = (size_t)b * B3;
    for (int v = threadIdx.x; v < B3; v += blockDim.x) {
      unsigned char c;
      p.field()[base + v] = p.seed(base + v, c);
      p.a.cls[base + v] = c;
    }
    if (threadIdx.x == 0) p.init_done(b);
  }
}

// incremental update: neighbour table of every block of the submap, epochs reset; the voxel state is left alone
template <class P>
__global__ void __launch_bounds__(256) es_k_prepare(P p) {
  const int nb = min(*p.g.n_blocks, p.g.max_blocks);
  if (blockIdx.x == 0 && threadIdx.x == 0) *p.a.nb_seen = nb;
  const int w = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31, nw = (gridDim.x * 256) >> 5;
  for (int b = w; b < nb; b += nw) {
    int s, bx, by, bz;
    ts_unpack_key(p.g.block_key[b], s, bx, by, bz);
    if (lane == 0) { p.a.epoch[b] = (s == p.submap) ? -1 : -1000000; p.a.repoch[b] = -1; }
    if (s != p.submap) continue;
    if (lane < 27) p.a.nbr[b * 27 + lane] = es_nbr(p.g, s, bx, by, bz, lane);
    p.prepare_block(b, lane);
  }
}

// 1. detect: the voxels of the blocks written since the last update that must be re-initialised -> CHANGED
template <class P>
__global__ void __launch_bounds__(P::THREADS) es_k_detect(P p) {
  constexpr int B3 = 1 << 3 * P::SHIFT;
  __shared__ int s_any;
  int* const dirty = p.dirty();
  const int nb = min(*p.g.n_blocks, p.g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (!dirty[b] || p.a.epoch[b] < -1) continue;  // (uniform per CTA)
    __syncthreads();
    if (threadIdx.x == 0) s_any = 0;
    __syncthreads();
    const size_t base = (size_t)b * B3;
    int mine = 0;
    for (int v = threadIdx.x; v < B3; v += blockDim.x) {
      const unsigned char oc = p.a.cls[base + v] & ES_CLS;
      if (p.moved(base + v, oc)) { p.a.cls[base + v] = oc | ES_CH; mine++; }
    }
    es_cta_add(mine, &s_any);
    __syncthreads();
    if (threadIdx.x == 0) {
      dirty[b] = 0;
      if (s_any) { p.a.repoch[b] = 0; atomicAdd(&p.a.counts[0], s_any); }
    }
  }
}

// 3. re-initialise flagged voxels; their blocks start the lower wave (epoch 0)
template <class P>
__global__ void __launch_bounds__(P::THREADS) es_k_reinit(P p) {
  constexpr int B3 = 1 << 3 * P::SHIFT;
  __shared__ int s_n;
  const int nb = min(*p.g.n_blocks, p.g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (p.a.repoch[b] < 0) continue;  // no flagged voxel in this block (uniform per CTA)
    __syncthreads();
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const size_t base = (size_t)b * B3;
    int nsu = 0;
    for (int v = threadIdx.x; v < B3; v += blockDim.x) {
      const unsigned char c = p.a.cls[base + v];
      if (!(c & (ES_CH | ES_SU))) continue;
      unsigned char nc;
      p.field()[base + v] = p.seed(base + v, nc);
      p.a.cls[base + v] = nc;
      nsu += (c & ES_SU) ? 1 : 0;
    }
    es_cta_add(nsu, &s_n);
    __syncthreads();
    if (threadIdx.x == 0) {
      p.a.epoch[b] = 0;
      if (s_n) atomicAdd(&p.a.counts[1], s_n);
      atomicAdd(&p.a.counts[2], 1);
    }
  }
}

template <int T>
struct EsTile {
  float e[T * T * T];
  unsigned char cls[T * T * T];
  int nbr[27];
  int active, changed, any_write;
};

// One sweep of a wave over the blocks of the submap it reaches: 2. the raise wave (RAISE: flag the target voxels that
// may have been derived from a flagged neighbour; epochs in repoch) or 4. the lower wave (relax; epochs in epoch).
// TILED (the TSDF's tiled ESDF): ghost blocks are read-only sources - never relaxed, but their epochs wake their owned
// neighbours - and an owned block that changes is marked for the next ESDF halo pack.
template <class P, bool RAISE, bool TILED>
__global__ void __launch_bounds__(P::THREADS) es_k_wave(P p, int sweep) {
  constexpr int S = P::SHIFT, B = 1 << S, B3 = B * B * B, T = B + 2;
  __shared__ EsTile<T> tile;
  int* const epoch = RAISE ? p.a.repoch : p.a.epoch;
  int* const changed = RAISE ? p.a.rchanged : p.a.changed;
  if (sweep > 1 && changed[sweep - 1] == 0) return;  // already converged: nothing to do
  const int nb = min(*p.g.n_blocks, p.g.max_blocks);
  const float d1 = p.vs, d2 = sqrtf(2.0f) * p.vs, d3 = sqrtf(3.0f) * p.vs;  // dir.norm()*voxel_scale (dense_esdf.py:285)
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    __syncthreads();
    if (threadIdx.x == 0) { tile.active = 0; tile.any_write = 0; }
    __syncthreads();
    if (p.a.epoch[b] < -1) continue;  // block of another submap (uniform per CTA)
    if constexpr (TILED) {
      if (p.g.ghost[b]) continue;  // the owner's values: a source only
    }
    if (threadIdx.x < 27) {
      const int n = p.a.nbr[b * 27 + threadIdx.x];
      tile.nbr[threadIdx.x] = n;
      if (n >= 0 && *(volatile int*)&epoch[n] >= sweep - 1) tile.active = 1;  // the wave front reaches this block
    }
    __syncthreads();
    if (!tile.active) continue;
    for (int c = threadIdx.x; c < T * T * T; c += blockDim.x) {
      const int lz = c % T - 1, ly = (c / T) % T - 1, lx = c / (T * T) - 1;
      const int nbk = tile.nbr[(((lx + B) >> S) * 3 + ((ly + B) >> S)) * 3 + ((lz + B) >> S)];
      float ev = 0.0f;
      unsigned char cl = P::NONE;
      if (nbk >= 0) {
        const size_t off = (size_t)nbk * B3 + es_voff<S>(lx, ly, lz);
        if constexpr (RAISE) {
          cl = *(volatile unsigned char*)&p.a.cls[off];
          ev = p.field()[off];  // old values: nothing writes the field during the raise wave
        } else {
          p.stage(off, ev, cl);
        }
      }
      tile.e[c] = ev;
      tile.cls[c] = cl;
    }
    __syncthreads();
    // to local convergence (values and flags only move monotonically, so in-place racy updates are safe)
    for (int iter = 0; iter < 64; ++iter) {
      if (threadIdx.x == 0) tile.changed = 0;
      __syncthreads();
      bool mine = false;
      for (int v = threadIdx.x; v < B3; v += blockDim.x) {
        const int c0 = es_tidx<S>(v);
        const unsigned char cl = tile.cls[c0];
        if constexpr (RAISE) {
          if (cl != P::MIN_SIDE && cl != P::MAX_SIDE) continue;  // flagged or not a target: nothing to decide
          const float cur = tile.e[c0];
          bool hit = false;
          es_for_26<T>(c0, d1, d2, d3, [&](int cn, float dis) {
            const unsigned char hf = tile.cls[cn];
            const unsigned char hc = hf & ES_CLS;  // the neighbour's class at the last update
            if (!(hf & (ES_CH | ES_SU)) || !P::raise_source(hc)) return;
            const float he = tile.e[cn];
            hit |= (cl == P::MIN_SIDE ? P::cand_min(hc, he, dis) : P::cand_max(hc, he, dis)) == cur;
          });
          if (hit) { tile.cls[c0] = cl | ES_SU; mine = true; }
        } else {
          if (!P::target(cl)) continue;
          float best = tile.e[c0];
          const float cur = best;
          es_for_26<T>(c0, d1, d2, d3, [&](int cn, float dis) {
            const unsigned char hc = tile.cls[cn];
            if (!P::source(cl, hc)) return;
            const float he = tile.e[cn];
            if (cl == P::MIN_SIDE) best = fminf(best, P::cand_min(hc, he, dis)); else best = fmaxf(best, P::cand_max(hc, he, dis));
          });
          if (best != cur) { tile.e[c0] = best; mine = true; }
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
      const size_t base = (size_t)b * B3;
      for (int v = threadIdx.x; v < B3; v += blockDim.x) {
        if constexpr (RAISE) {
          const unsigned char cl = tile.cls[es_tidx<S>(v)];
          if (cl & ES_SU) p.a.cls[base + v] = cl;
        } else {
          p.field()[base + v] = tile.e[es_tidx<S>(v)];
        }
      }
      if (threadIdx.x == 0) {
        __threadfence();
        epoch[b] = sweep;
        changed[sweep] = 1;
        if constexpr (TILED) p.a.xmark[b] = 1;
      }
    }
  }
}

// pool index of block (bx, by, bz) of the submap for a query, or -1: absent, newer than the last update, or (GHOSTS: the
// TSDF's tiled map) a ghost block while the field is not a completed tiled ESDF
template <class P>
__device__ __forceinline__ int es_qblock(const P& p, int nb_seen, int bx, int by, int bz) {
  const int b = ts_find(p.g, ts_pack_key(p.submap, bx, by, bz));
  if constexpr (P::GHOSTS) return (b >= 0 && b < nb_seen && (p.ghosts || !p.g.ghost[b])) ? b : -1;
  else return (b >= 0 && b < nb_seen) ? b : -1;
}
// The 8 interpolation corners of the cell with low corner (i0, j0, k0) on blocks of edge 1 << S: e[dx*4 + dy*2 + dz] is
// the value of corner (i0+dx, j0+dy, k0+dz).  find(bx, by, bz) -> pool index of a block, or -1 when it does not count;
// each distinct corner block is looked up once (the corner cube spans 2, 4 or 8 blocks only where i0 is the last voxel
// of its block on some axis).  read(off, e) -> whether the corner at pool offset off has a value, stored in e.  False
// (e unspecified) when a block is refused or a corner has no value.  The ESDF queries and the SDF-to-SDF registration
// (tslam_register.cu) and rendering (tslam_render.cu) read their corners through this one function.
template <int S, class Find, class Read>
__device__ __forceinline__ bool es_corners(int i0, int j0, int k0, Find find, Read read, float e[8]) {
  constexpr int M = (1 << S) - 1, B3 = 1 << 3 * S;
  const bool sx = (i0 & M) == M, sy = (j0 & M) == M, sz = (k0 & M) == M;
  const int x0 = i0 >> S, y0 = j0 >> S, z0 = k0 >> S;
  // b[dx*4 + dy*2 + dz]: block of corner (i0+dx, j0+dy, k0+dz); a corner that shares its block with a lower one reuses it
  int b[8];
  b[0] = find(x0, y0, z0);
  b[1] = sz ? find(x0, y0, z0 + 1) : b[0];
  b[2] = sy ? find(x0, y0 + 1, z0) : b[0];
  b[3] = sy ? (sz ? find(x0, y0 + 1, z0 + 1) : b[2]) : b[1];
  b[4] = sx ? find(x0 + 1, y0, z0) : b[0];
  b[5] = sx ? (sz ? find(x0 + 1, y0, z0 + 1) : b[4]) : b[1];
  b[6] = sx ? (sy ? find(x0 + 1, y0 + 1, z0) : b[4]) : b[2];
  b[7] = sx ? (sy ? (sz ? find(x0 + 1, y0 + 1, z0 + 1) : b[6]) : b[5]) : b[3];
  bool ok = true;
#pragma unroll
  for (int c = 0; c < 8; c++) {
    ok &= b[c] >= 0;
    e[c] = 0.0f;
  }
  if (ok) {
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const size_t off = (size_t)b[c] * B3 + es_voff<S>(i0 + (c >> 2), j0 + ((c >> 1) & 1), k0 + (c & 1));
      ok &= read(off, e[c]);
    }
  }
  return ok;
}

// The zero level that registration, frame tracking and rendering share: the committed TSDF of one submap, interpolated
// over the 8 corners of a cell.  A block counts when it is present and not a ghost (ts_sdf_block); a corner has a value
// when it is observed and its weight is > 0 (ts_sdf_corners); no other threshold.
__device__ __forceinline__ int ts_sdf_block(const TsGrid& g, int sb, int bx, int by, int bz) {
  const int b = ts_find(g, ts_pack_key(sb, bx, by, bz));
  return (b >= 0 && !g.ghost[b]) ? b : -1;
}
// find(bx, by, bz) -> ts_sdf_block's answer (a caller may memoise it); seen(c, off) gets the pool offset of corner c
// (e[c]) for each corner read (all 8 whenever every corner block counts)
template <class Find, class Seen>
__device__ __forceinline__ bool ts_sdf_corners(const TsGrid& g, const int c0[3], Find find, float e[8], Seen seen) {
  return es_corners<TS_BSHIFT>(
      c0[0], c0[1], c0[2], find,
      [&](size_t off, float& ev) {
        const float2 tw = g.tw[off];
        ev = tw.x;
        seen((int)(&ev - e), off);
        return g.obs[off] != 0 && tw.y > 0.0f;
      },
      e);
}
template <class Find>
__device__ __forceinline__ bool ts_sdf_corners(const TsGrid& g, const int c0[3], Find find, float e[8]) {
  return ts_sdf_corners(g, c0, find, e, [](int, size_t) {});
}

// Trilinear interpolation of the field over the 8 voxels around each point (voxel i centred at i*vs, submap-local frame)
// and the exact partial derivatives of that interpolant, as of the last update.  One thread per point, corners from
// es_corners.  Invalid (NaN, valid = 0): a non-finite coordinate, a corner outside the volume, a corner in a block
// es_qblock refuses, a corner whose class at the last update has no value.  The body of each ESDF's query kernel, which
// keeps the grid and the state as separate parameters: built around one rule parameter, the occupancy ESDF's query
// compiles to 40 registers instead of 32 (6 instead of 8 CTAs per SM).
//
// es_point is the answer at one point x (nb_seen = *p.a.nb_seen): whether it is valid, and d, gx, gy, gz (NaN when
// not).  The query kernels and the trajectory solver (tslam_traj.cuh) both read the field through it.
template <class P>
__device__ __forceinline__ bool es_point(const P& p, int nb_seen, const float* x, float& d, float& gx, float& gy, float& gz) {
  constexpr int S = P::SHIFT;
  const float vs = p.vs, qnan = __int_as_float(0x7fc00000);
  // both corners i0, i0 + 1 inside the volume: the low corner and i0 < N - hN - 1 per axis
  float u[3];
  int c0[3];
  bool ok = esq_low_corner(p.g, vs, x, u, c0) && c0[0] < p.g.N - p.g.hN - 1 && c0[1] < p.g.N - p.g.hN - 1 &&
            c0[2] < p.g.Nz - p.g.hNz - 1;
  d = qnan; gx = qnan; gy = qnan; gz = qnan;
  if (ok) {
    const int i0 = c0[0], j0 = c0[1], k0 = c0[2];
    const float fx = __fsub_rn(u[0], (float)i0), fy = __fsub_rn(u[1], (float)j0), fz = __fsub_rn(u[2], (float)k0);
    float e[8];
    ok = es_corners<S>(
        i0, j0, k0, [&](int bx, int by, int bz) { return es_qblock(p, nb_seen, bx, by, bz); },
        [&](size_t off, float& ev) {
          const bool has = P::valid(p.a.cls[off] & ES_CLS);
          ev = p.field()[off];
          return has;
        },
        e);
    if (ok) esq_interp(e, fx, fy, fz, vs, d, gx, gy, gz);
    else d = gx = gy = gz = qnan;
  }
  return ok;
}
template <class P>
__device__ __forceinline__ void es_query(const P& p, long long n, const float* __restrict__ xyz, float* __restrict__ dist,
                                                  float* __restrict__ grad, uint8_t* __restrict__ valid) {
  const int nb_seen = *p.a.nb_seen;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    float d, gx, gy, gz;
    const bool ok = es_point(p, nb_seen, xyz + 3 * q, d, gx, gy, gz);
    dist[q] = d;
    grad[3 * q] = gx; grad[3 * q + 1] = gy; grad[3 * q + 2] = gz;
    valid[q] = ok ? 1 : 0;
  }
}

// One update of the ESDF that p describes (p.a.changed, rchanged and counts lie back to back): full, or incremental.
// Each caller has done its own argument checks and staleness decision.  stats4 (HOST, may be NULL): lower sweeps, raise
// sweeps (-1 = full), changed voxels, suspect voxels.
template <bool TILED = false, class P, class M>
static int es_update(M* m, const P& p, bool full, cudaStream_t st, int32_t* stats4) {
  const int grid = m->sm_count * P::GRID;
  const auto lower = [&](int k) { es_k_wave<P, false, TILED><<<grid, P::THREADS, 0, st>>>(p, k); };
  int h_counts[4] = {0, 0, 0, 0}, n_lower = 0, n_raise = 0, rc;
  TS_CUDA(cudaMemsetAsync(p.a.changed, 0, (2 * (ES_MAX_SWEEPS + 2) + P::COUNTS_CLEARED) * 4, st));  // changed, rchanged, counts
  if (full) {
    es_k_init<P, TILED><<<grid, P::THREADS, 0, st>>>(p);
    TS_LAUNCH_CHECK(m);
    rc = es_wave(m, st, p.a.changed, ES_GROUP, lower, &n_lower);
    if (rc) return rc;
  } else {
    es_k_prepare<P><<<m->sm_count * 2, 256, 0, st>>>(p);
    TS_LAUNCH_CHECK(m);
    es_k_detect<P><<<grid, P::THREADS, 0, st>>>(p);
    TS_LAUNCH_CHECK(m);
    rc = es_wave(m, st, p.a.rchanged, 4, [&](int k) { es_k_wave<P, true, false><<<grid, P::THREADS, 0, st>>>(p, k); }, &n_raise);
    if (rc) return rc;
    es_k_reinit<P><<<grid, P::THREADS, 0, st>>>(p);
    TS_LAUNCH_CHECK(m);
    rc = es_wave(m, st, p.a.changed, 4, lower, &n_lower);
    if (rc) return rc;
    TS_CUDA(cudaMemcpy(h_counts, p.a.counts, 16, cudaMemcpyDeviceToHost));
  }
  if (stats4) { stats4[0] = n_lower; stats4[1] = full ? -1 : n_raise; stats4[2] = h_counts[0]; stats4[3] = h_counts[1]; }
  return TSLAM_OK;
}
