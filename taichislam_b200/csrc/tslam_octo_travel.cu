// libtslam.so - travel-cost fields of a log-odds Octomap (DESIGN.md section 7, "Travel cost on the log-odds Octomap" and
// "Many-source travel costs").
//
// Per submap, as of one update.  Classes as the occupancy ESDF defines them: OCC = known and L > l_occ, FREE = known and
// L <= l_occ, UNKNOWN = not known (every cell of an absent block).  A cell is traversable iff it is inside the volume and
// FREE, and, when clearance > 0, was FREE at the last occupancy-ESDF update of the submap, in a block that update saw,
// with ESDF value >= clearance.  A step between 26-neighbours (edge cost c = vs * {1, sqrtf 2, sqrtf 3}, the ESDF's) is
// allowed iff every cell of the axis-aligned box its two cells span is traversable (no corner cutting).  From the start
// cell c0 = rha(p / vs), when traversable, G(c0) = 0 and
//   G(v) = min over allowed steps h -> v of G(h) + c    (f32, one step at a time), values above max_cost dropped (+inf)
// to the fixed point.  f32 addition is monotone and, below the bound max_cost <= 2^22 vs, G + c > G: the fixed point is
// unique, equals Dijkstra's answer and does not depend on the schedule (DESIGN.md section 7 gives the argument).
//
// One update computes S such fields, one per start, in the same launches.  The single-source API
// (tslam_octo_travel_update and its readers) is the S = 1 case, kept in a state of its own so that it and the
// many-source fields never change each other's answers.  The scheme is the occupancy ESDF's lower wave
// (es_k_wave): a CTA stages one (block, source) item plus a one-voxel halo of G in shared memory and relaxes it
// in place to local convergence (values only decrease); sweep k runs the items with a neighbour item of the same source
// stamped >= k-1, starting from the starts' items, and es_wave drives the sweeps.  A step's box lies inside the 3^3
// neighbourhood of its target cell, so the step rule never leaves the staged tile.
//
// Nothing here writes the map or another tracker's state: no cnt word, mark bit, touched entry, dirty flag or stats
// counter.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>
#include "tslam_esdf_common.cuh"

#define OT_T 10
#define OT_T3 (OT_T * OT_T * OT_T)
#define OT_THREADS 128
#define OT_WORDS 16  // traversable bits per pool block: 512 bits

// bit of neighbourhood offset (dx, dy, dz) in a 27-bit mask: dx outermost, the OFFSETS order of the reference
__host__ __device__ constexpr int ot_bit(int dx, int dy, int dz) { return (dx + 1) * 9 + (dy + 1) * 3 + (dz + 1); }

// The allowed steps into a cell whose 3^3 neighbourhood has traversable mask nm (bit ot_bit): bit ot_bit(d) is set iff
// every cell of the box spanned by the cell and its neighbour d is traversable.  0 when the cell itself is not.
__device__ __forceinline__ unsigned ot_allowed(unsigned nm) {
  if (!((nm >> ot_bit(0, 0, 0)) & 1u)) return 0u;
  unsigned am = 0u;
#pragma unroll
  for (int dx = -1; dx <= 1; dx++)
#pragma unroll
    for (int dy = -1; dy <= 1; dy++)
#pragma unroll
      for (int dz = -1; dz <= 1; dz++) {
        if (dx == 0 && dy == 0 && dz == 0) continue;
        unsigned box = 0u;
#pragma unroll
        for (int a = 0; a <= 1; a++)
#pragma unroll
          for (int b = 0; b <= 1; b++)
#pragma unroll
            for (int c = 0; c <= 1; c++) box |= 1u << ot_bit(a * dx, b * dy, c * dz);
        if ((nm & box) == box) am |= 1u << ot_bit(dx, dy, dz);
      }
  return am;
}

__device__ __forceinline__ int ot_tidx(int lx, int ly, int lz) { return ((lx + 1) * OT_T + (ly + 1)) * OT_T + (lz + 1); }

// cell rha(p / vs) of a point, and whether it is inside the volume (false for a non-finite coordinate)
__device__ __forceinline__ bool ot_cell(const OcGrid& g, float vs, const float* p, int c[3]) {
  const float u0 = __fdiv_rn(p[0], vs), u1 = __fdiv_rn(p[1], vs), u2 = __fdiv_rn(p[2], vs);
  if (!(fabsf(u0) < 1e9f && fabsf(u1) < 1e9f && fabsf(u2) < 1e9f)) return false;  // no out-of-range float -> int conversion
  c[0] = (int)roundf(u0); c[1] = (int)roundf(u1); c[2] = (int)roundf(u2);
  return ts_in_bounds(g, c[0], c[1], c[2]);
}

// pool block of cell c in `submap` when the update saw it, else -1
__device__ __forceinline__ int ot_block(const OcGrid& g, int submap, int nb_seen, const int c[3]) {
  const int b = ts_find(g, ts_pack_key(submap, c[0] >> OC_BSHIFT, c[1] >> OC_BSHIFT, c[2] >> OC_BSHIFT));
  return (b >= 0 && b < nb_seen) ? b : -1;
}

// State scales with the B_t submap blocks that hold a traversable cell (compact slots), not with the pool: per pool
// block only the traversable bits and the slot; per slot the allowed steps of each voxel (fixed during the wave and the
// same for every source) and the compact neighbour table; per (slot, source) item the field and an epoch.  Items are
// numbered t * S + s, so consecutive CTAs of a sweep read the same slot's allowed steps.
struct OtmAux {
  uint32_t* trav;  // [max_blocks*16] traversable bits of the update (pool layout)
  int* slot;       // [max_blocks] compact slot of a block of the update with a traversable cell, else -1
  int* changed;    // [ES_MAX_SWEEPS+2] changed[k] != 0 <=> sweep k changed something (all sources)
  int* counts;     // [4] traversable cells, slots (B_t)
  int* nb_seen;    // blocks in the pool when the last update ran
  int* start;      // [MAX_STARTS*4] start cell i, j, k, inside the volume
  int* sitem;      // [MAX_STARTS] item of the start's cell, -1 when it is not traversable
  int* reach;      // [MAX_STARTS] reachable cells per source
  int* cblk;       // [B_t] pool block of a slot
  int* cnbr;       // [B_t*27] compact slots of the 27 neighbour blocks (-1: absent or without a traversable cell)
  uint32_t* am;    // [B_t*512] allowed steps into each voxel (ot_allowed of its traversable neighbourhood)
  int* epoch;      // [S*B_t] last sweep in which the item changed (-1: idle)
  float* G;        // [S*B_t*512] the fields, +inf where unreachable
  int S, nt;
};

__device__ __forceinline__ float* otm_field(const OtmAux& a, int t, int s) { return a.G + ((size_t)t * a.S + s) * OC_B3; }

struct OtmTile {
  float G[OT_T3];
  int nbr[27];  // neighbour items of the same source (-1: none)
  int active, changed, any_write;
};

// the relaxation loop of a sweep: the staged tile in place to local convergence, am[q] the allowed steps into
// voxel threadIdx.x + q * OT_THREADS; tile.any_write is set when a value changed
__device__ __forceinline__ void ot_relax(OtmTile& tile, const unsigned (&am)[OC_B3 / OT_THREADS], float d1, float d2, float d3,
                                         float max_cost) {
  for (int iter = 0; iter < 64; ++iter) {
    if (threadIdx.x == 0) tile.changed = 0;
    __syncthreads();
    bool mine = false;
#pragma unroll
    for (int q = 0; q < OC_B3 / OT_THREADS; q++) {
      if (!am[q]) continue;
      const int v = threadIdx.x + q * OT_THREADS;
      const int c0 = ot_tidx(v >> 6, (v >> 3) & 7, v & 7);
      const float cur = tile.G[c0];
      float best = cur;
#pragma unroll
      for (int dx = -1; dx <= 1; dx++)
#pragma unroll
        for (int dy = -1; dy <= 1; dy++)
#pragma unroll
          for (int dz = -1; dz <= 1; dz++) {
            const int nz_ = (dx != 0) + (dy != 0) + (dz != 0);
            if (nz_ == 0 || !((am[q] >> ot_bit(dx, dy, dz)) & 1u)) continue;
            const float dis = nz_ == 1 ? d1 : (nz_ == 2 ? d2 : d3);
            const float cand = tile.G[c0 + (dx * OT_T + dy) * OT_T + dz] + dis;
            if (cand <= max_cost) best = fminf(best, cand);  // (+inf + c is +inf: never kept)
          }
      if (best < cur) {
        tile.G[c0] = best;
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
}

// Every pool block the update sees: traversable bits, and a compact slot for the blocks of the submap with a traversable
// cell (counts[0] traversable cells, counts[1] slots).  Slots are handed out in any order: the fields do not depend on it.
__global__ void __launch_bounds__(OT_THREADS) k_octo_travel_multi_classify(OcGrid g, OtmAux a, OcEsdfField ef, int submap, int l_occ,
                                                                           float clearance) {
  __shared__ int s_n;
  const int nb = min(*g.n_blocks, g.max_blocks);
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.nb_seen = nb;
  const bool clear = clearance > 0.0f;
  const int enb = clear ? *ef.nb_seen : 0;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap) {  // (uniform per CTA)
      if (threadIdx.x == 0) a.slot[b] = -1;
      continue;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const size_t base = (size_t)b * OC_B3;
    int cnt = 0;
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
      const int i = bx * OC_B + (v >> 6), j = by * OC_B + ((v >> 3) & 7), k = bz * OC_B + (v & 7);
      const bool t = oc_traversable(g, ef, l_occ, clearance, clear, enb, b, base + v, g.cnt[base + v], i, j, k);
      const unsigned m = __ballot_sync(0xffffffffu, t);
      if ((threadIdx.x & 31) == 0) a.trav[(size_t)b * OT_WORDS + (v >> 5)] = m;
      cnt += t ? 1 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&s_n, cnt);
    __syncthreads();
    if (threadIdx.x == 0) {
      a.slot[b] = s_n ? atomicAdd(&a.counts[1], 1) : -1;
      if (s_n) atomicAdd(&a.counts[0], s_n);
    }
  }
}

// Per slot: its pool block, the compact neighbour table, and the allowed steps into each voxel from the traversable bits
// of its 3^3 block neighbourhood (staged as a 10^3 byte tile)
__global__ void __launch_bounds__(OT_THREADS) k_octo_travel_multi_tables(OcGrid g, OtmAux a) {
  __shared__ unsigned char t_[OT_T3];
  __shared__ int nbr[27];
  const int nb = *a.nb_seen;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    const int t = a.slot[b];
    if (t < 0) continue;  // (uniform per CTA)
    __syncthreads();
    if (threadIdx.x < 27) {
      int s, bx, by, bz;
      ts_unpack_key(g.block_key[b], s, bx, by, bz);
      const int dx = threadIdx.x / 9 - 1, dy = (threadIdx.x / 3) % 3 - 1, dz = threadIdx.x % 3 - 1;
      int n = ts_find(g, ts_pack_key(s, bx + dx, by + dy, bz + dz));
      n = n < nb ? n : -1;
      nbr[threadIdx.x] = n;
      a.cnbr[(size_t)t * 27 + threadIdx.x] = n >= 0 ? a.slot[n] : -1;
      if (threadIdx.x == 0) a.cblk[t] = b;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < OT_T3; c += blockDim.x) {
      const int lz = c % OT_T - 1, ly = (c / OT_T) % OT_T - 1, lx = c / (OT_T * OT_T) - 1;
      const int nbk = nbr[(((lx + 8) >> 3) * 3 + ((ly + 8) >> 3)) * 3 + ((lz + 8) >> 3)];
      const int off = oc_voxel_off(lx, ly, lz);
      t_[c] = nbk >= 0 ? (unsigned char)((a.trav[(size_t)nbk * OT_WORDS + (off >> 5)] >> (off & 31)) & 1u) : 0;
    }
    __syncthreads();
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
      const int c0 = ot_tidx(v >> 6, (v >> 3) & 7, v & 7);
      unsigned nm = 0u;
#pragma unroll
      for (int dx = -1; dx <= 1; dx++)
#pragma unroll
        for (int dy = -1; dy <= 1; dy++)
#pragma unroll
          for (int dz = -1; dz <= 1; dz++) nm |= (unsigned)t_[c0 + (dx * OT_T + dy) * OT_T + dz] << ot_bit(dx, dy, dz);
      a.am[(size_t)t * OC_B3 + v] = ot_allowed(nm);
    }
  }
}

// every item: G = +inf, idle
__global__ void __launch_bounds__(OT_THREADS) k_octo_travel_multi_fill(OtmAux a) {
  const long long items = (long long)a.S * a.nt;
  const float inf = __int_as_float(0x7f800000);
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    float* G = a.G + (size_t)it * OC_B3;
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) G[v] = inf;
    if (threadIdx.x == 0) a.epoch[it] = -1;
  }
}

// one thread per source: G = 0 and epoch 0 at a traversable start cell (its item in sitem), else sitem = -1
__global__ void k_octo_travel_multi_starts(OcGrid g, OtmAux a, int submap) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= a.S) return;
  const int* c = a.start + 4 * s;
  int item = -1;
  if (c[3]) {
    const int b = ot_block(g, submap, *a.nb_seen, c);
    const int t = b >= 0 ? a.slot[b] : -1;
    const int off = oc_voxel_off(c[0], c[1], c[2]);
    if (t >= 0 && ((a.trav[(size_t)b * OT_WORDS + (off >> 5)] >> (off & 31)) & 1u)) {
      item = t * a.S + s;
      otm_field(a, t, s)[off] = 0.0f;
      a.epoch[item] = 0;
    }
  }
  a.sitem[s] = item;
}

// One sweep of the S waves: relax the items the wave fronts reach to local convergence.  An item is active when one of
// its 27 neighbour items of the same source was stamped in the previous sweep or later.
__global__ void __launch_bounds__(OT_THREADS) k_octo_travel_multi_sweep(OtmAux a, int sweep, float vs, float max_cost) {
  __shared__ OtmTile tile;
  if (sweep > 1 && a.changed[sweep - 1] == 0) return;  // already converged: nothing to do
  const long long items = (long long)a.S * a.nt;
  const float d1 = vs, d2 = sqrtf(2.0f) * vs, d3 = sqrtf(3.0f) * vs;  // the edge costs of es_k_wave
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const int t = (int)(it / a.S), s = (int)(it % a.S);
    __syncthreads();
    if (threadIdx.x == 0) { tile.active = 0; tile.any_write = 0; }
    __syncthreads();
    if (threadIdx.x < 27) {
      const int n = a.cnbr[(size_t)t * 27 + threadIdx.x];
      const int ni = n >= 0 ? n * a.S + s : -1;
      tile.nbr[threadIdx.x] = ni;
      if (ni >= 0 && *(volatile int*)&a.epoch[ni] >= sweep - 1) tile.active = 1;
    }
    __syncthreads();
    if (!tile.active) continue;
    for (int c = threadIdx.x; c < OT_T3; c += blockDim.x) {
      const int lz = c % OT_T - 1, ly = (c / OT_T) % OT_T - 1, lx = c / (OT_T * OT_T) - 1;
      const int ni = tile.nbr[(((lx + 8) >> 3) * 3 + ((ly + 8) >> 3)) * 3 + ((lz + 8) >> 3)];
      tile.G[c] = ni >= 0 ? *(volatile float*)&a.G[(size_t)ni * OC_B3 + oc_voxel_off(lx, ly, lz)] : __int_as_float(0x7f800000);
    }
    unsigned am[OC_B3 / OT_THREADS];
#pragma unroll
    for (int q = 0; q < OC_B3 / OT_THREADS; q++) am[q] = a.am[(size_t)t * OC_B3 + threadIdx.x + q * OT_THREADS];
    __syncthreads();
    ot_relax(tile, am, d1, d2, d3, max_cost);
    if (tile.any_write) {
      float* G = a.G + (size_t)it * OC_B3;
      for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) G[v] = tile.G[ot_tidx(v >> 6, (v >> 3) & 7, v & 7)];
      if (threadIdx.x == 0) {
        __threadfence();
        a.epoch[it] = sweep;
        a.changed[sweep] = 1;
      }
    }
  }
}

// reachable cells per source after the waves -> reach[s]
__global__ void __launch_bounds__(OT_THREADS) k_octo_travel_multi_count(OtmAux a) {
  __shared__ int s_n;
  const long long items = (long long)a.S * a.nt;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    if (a.epoch[it] < 0) continue;  // never reached: all +inf (uniform per CTA)
    __syncthreads();
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    int cnt = 0;
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) cnt += isfinite(a.G[(size_t)it * OC_B3 + v]) ? 1 : 0;
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&s_n, cnt);
    __syncthreads();
    if (threadIdx.x == 0 && s_n) atomicAdd(&a.reach[it % a.S], s_n);
  }
}

// (ijk, G) of every reachable cell of field s (blocks without a slot hold no traversable cell and list nothing)
__global__ void __launch_bounds__(OT_THREADS) k_octo_travel_slot_gather(OcGrid g, OtmAux a, int s, long long cap, int32_t* idx, float* cost,
                                                                        unsigned long long* counter) {
  for (int t = blockIdx.x; t < a.nt; t += gridDim.x) {
    if (a.epoch[(size_t)t * a.S + s] < 0) continue;  // never reached: all +inf (uniform per CTA)
    int sm, bx, by, bz;
    ts_unpack_key(g.block_key[a.cblk[t]], sm, bx, by, bz);
    const float* G = otm_field(a, t, s);
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
      const float gv = G[v];
      const bool want = isfinite(gv);
      const long long row = warp_append_u64(want, counter);
      if (want && row < cap) {
        idx[3 * row] = bx * OC_B + (v >> 6);
        idx[3 * row + 1] = by * OC_B + ((v >> 3) & 7);
        idx[3 * row + 2] = bz * OC_B + (v & 7);
        cost[row] = gv;
      }
    }
  }
}

// slot of the cell of a point in the update's blocks, -1 when outside the volume, not finite, in a newer block or in a
// block without a traversable cell (whose cells all read +inf)
__device__ __forceinline__ int otm_slot(const OcGrid& g, const OtmAux& a, int submap, int nb_seen, float vs, const float* p, int c[3]) {
  if (!ot_cell(g, vs, p, c)) return -1;
  const int b = ot_block(g, submap, nb_seen, c);
  return b >= 0 ? a.slot[b] : -1;
}

// cost[s * n + q] = G_s of the cell of point q: one thread per point, looping over the sources
__global__ void __launch_bounds__(256) k_octo_travel_multi_query(OcGrid g, OtmAux a, int submap, long long n, const float* __restrict__ xyz,
                                                                 float vs, float* __restrict__ cost) {
  const int nb_seen = *a.nb_seen;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    int c[3];
    const int t = otm_slot(g, a, submap, nb_seen, vs, xyz + 3 * q, c);
    const int off = t >= 0 ? oc_voxel_off(c[0], c[1], c[2]) : 0;
    for (int s = 0; s < a.S; s++) cost[(size_t)s * n + q] = t >= 0 ? otm_field(a, t, s)[off] : __int_as_float(0x7f800000);
  }
}

// Path from the cell of xyz[q] back to the start of field source[q] (field 0 when source is NULL): from the current cell
// v, the predecessor is the reachable 26-neighbour h with an allowed step and G(h) + c == G(v) exactly, smallest G(h),
// ties to the first in ot_bit order, walked over the compact slots and their allowed steps.  A source outside [0, S)
// writes len 0 and sets OC_ERR_TRAVEL_SOURCE, reported by the next tslam_octo_sync.
__global__ void __launch_bounds__(256) k_octo_travel_multi_path(OcGrid g, OtmAux a, int submap, long long n, const int32_t* __restrict__ source,
                                                                const float* __restrict__ xyz, float vs, int max_len,
                                                                int32_t* __restrict__ cells, int32_t* __restrict__ len) {
  const int nb_seen = *a.nb_seen;
  const float d1 = vs, d2 = sqrtf(2.0f) * vs, d3 = sqrtf(3.0f) * vs;
  const float inf = __int_as_float(0x7f800000);
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const int s = source ? source[q] : 0;
    int L = 0;
    if (s < 0 || s >= a.S) {
      atomicOr(g.err, OC_ERR_TRAVEL_SOURCE);
      len[q] = 0;
      continue;
    }
    int c[3];
    int t = otm_slot(g, a, submap, nb_seen, vs, xyz + 3 * q, c);
    float gv = t >= 0 ? otm_field(a, t, s)[oc_voxel_off(c[0], c[1], c[2])] : inf;
    int32_t* out = cells + 3 * (size_t)q * max_len;
    while (gv < inf) {
      if (L < max_len) { out[3 * L] = c[0]; out[3 * L + 1] = c[1]; out[3 * L + 2] = c[2]; }
      ++L;
      if (gv == 0.0f) break;  // the start: the only cell at 0
      const int bx = c[0] >> OC_BSHIFT, by = c[1] >> OC_BSHIFT, bz = c[2] >> OC_BSHIFT;
      const unsigned am = a.am[(size_t)t * OC_B3 + oc_voxel_off(c[0], c[1], c[2])];
      int best = -1, bt = -1;
      float bg = inf;
#pragma unroll
      for (int e = 0; e < 27; e++) {
        if (e == ot_bit(0, 0, 0)) continue;
        const int dx = e / 9 - 1, dy = (e / 3) % 3 - 1, dz = e % 3 - 1;
        const int i = c[0] + dx, j = c[1] + dy, k = c[2] + dz;
        const int tn = a.cnbr[(size_t)t * 27 + ot_bit((i >> OC_BSHIFT) - bx, (j >> OC_BSHIFT) - by, (k >> OC_BSHIFT) - bz)];
        // every neighbour is read, a disallowed one from a valid slot, so the loads take no branch and issue together
        // (an allowed step's cell is traversable: tn >= 0)
        const bool ok = (am >> e) & 1u;
        const float hg = otm_field(a, ok ? tn : t, s)[oc_voxel_off(i, j, k)];
        const int nz_ = (dx != 0) + (dy != 0) + (dz != 0);
        const float dis = nz_ == 1 ? d1 : (nz_ == 2 ? d2 : d3);
        if (ok && hg < bg && hg + dis == gv) { best = e; bg = hg; bt = tn; }
      }
      if (best < 0) {  // cannot happen at the fixed point: reported by the next tslam_octo_sync, never a silent cut
        atomicOr(g.err, OC_ERR_TRAVEL_PATH);
        L = 0;
        break;
      }
      c[0] += best / 9 - 1; c[1] += (best / 3) % 3 - 1; c[2] += best % 3 - 1;
      t = bt;
      gv = bg;
    }
    len[q] = L;
  }
}

// ---- host side -----------------------------------------------------------------------------------------------------
// per pool block: traversable bits 64 + slot 4 = 68 B; then change flags, counts and the per-source arrays
static size_t otm_blk_bytes(size_t nb) {
  return nb * (OT_WORDS * 4 + 4) + ((ES_MAX_SWEEPS + 2) + 8 + TSLAM_OCTO_TRAVEL_MAX_STARTS * 6) * 4;
}
// per slot: pool block 4 + neighbour table 108 + allowed steps 2048 = 2160 B; per item: field 2048 + epoch 4 = 2052 B
static size_t otm_bytes(size_t nt, size_t S) { return nt * (4 + 27 * 4 + OC_B3 * 4) + S * nt * (OC_B3 * 4 + 4); }

static OtmAux otm_aux(const tslam_octo* m, const OcTravel& f) {
  const size_t nb = (size_t)m->g.max_blocks, S = f.S, nt = f.nt;
  OtmAux a;
  a.trav = (uint32_t*)f.blk;
  a.slot = (int*)(a.trav + nb * OT_WORDS);
  a.changed = a.slot + nb;
  a.counts = a.changed + (ES_MAX_SWEEPS + 2);
  a.nb_seen = a.counts + 4;
  a.start = a.counts + 8;
  a.sitem = a.start + 4 * TSLAM_OCTO_TRAVEL_MAX_STARTS;
  a.reach = a.sitem + TSLAM_OCTO_TRAVEL_MAX_STARTS;
  a.am = (uint32_t*)f.mem;  // (the two 2 KB-per-row arrays first: 128-byte aligned rows)
  a.G = (float*)(a.am + nt * OC_B3);
  a.epoch = (int*)(a.G + S * nt * OC_B3);
  a.cblk = a.epoch + S * nt;
  a.cnbr = a.cblk + nt;
  a.S = f.S;
  a.nt = f.nt;
  return a;
}

int oc_travel_free(tslam_octo* m) {
  for (OcTravel* f : {&m->tr, &m->trm}) {
    if (f->blk) cudaFree(f->blk);
    if (f->mem) cudaFree(f->mem);
    *f = OcTravel{};
  }
  return TSLAM_OK;
}

#define OT_UPDATE "tslam_octo_travel_update"
#define OTM_UPDATE "tslam_octo_travel_multi_update"
#define OT_FEATURE "a travel-cost field"

static int ot_clearance_finite(float clearance, const char* what) {
  if (std::isfinite(clearance) && clearance >= 0.0f) return TSLAM_OK;
  ts_set_error("%s: clearance must be finite and >= 0 (got %g)", what, (double)clearance);
  return TSLAM_E_INVALID;
}

// the clearance and max_cost checks of every travel update, and the occupancy ESDF the clearance test reads
static int ot_params(tslam_octo* m, int32_t submap, float clearance, float max_cost, const char* what, OcEsdfField* ef) {
  const float cost_limit = std::ldexp(m->in.vs, 22);  // keeps G + vs > G for every kept value
  int rc = ot_clearance_finite(clearance, what);
  if (rc) return rc;
  if (!(std::isfinite(max_cost) && max_cost > 0.0f && max_cost <= cost_limit)) {
    ts_set_error("%s: max_cost must be finite, > 0 and <= 2^22 * voxel_scale = %g (got %g)", what, (double)cost_limit, (double)max_cost);
    return TSLAM_E_INVALID;
  }
  return oc_clearance_field(m, submap, clearance, what, ef);
}

int oc_clearance_field(tslam_octo* m, int32_t submap, float clearance, const char* what, OcEsdfField* ef) {
  int rc = ot_clearance_finite(clearance, what);
  if (rc) return rc;
  memset(ef, 0, sizeof(*ef));
  if (clearance > 0.0f) {
    const int rc = oc_esdf_field(m, submap, what, ef);
    if (rc) return rc;
    if (clearance > ef->D) {
      ts_set_error("%s: clearance %g exceeds the occupancy ESDF's max_dist %g", what, (double)clearance, (double)ef->D);
      return TSLAM_E_INVALID;
    }
  }
  return TSLAM_OK;
}

// start cell c0 = rha(p / vs) of a finite point, f32 division as the kernels do it; false when outside the volume
static bool ot_start_cell(const tslam_octo* m, const float* p, int c[3]) {
  for (int q = 0; q < 3; q++) {
    const float u = p[q] / m->in.vs;
    if (!(std::fabs(u) < 1e9f)) return false;
    c[q] = (int)std::round(u);
  }
  return c[0] >= -m->g.hN && c[0] < m->g.N - m->g.hN && c[1] >= -m->g.hN && c[1] < m->g.N - m->g.hN && c[2] >= -m->g.hNz &&
         c[2] < m->g.Nz - m->g.hNz;
}

// The fields of `submap` from the S finite starts[S,3] into f, for both update entry points (`what` names the one called
// in messages).  A refused clearance or max_cost leaves f's last fields readable; from then on f is unreadable until the
// update completes.  Outputs as tslam_octo_travel_multi_update.
static int ot_update(tslam_octo* m, OcTravel& f, int32_t submap, int S, const float* starts, float clearance, float max_cost,
                     const char* what, int32_t* stats2, int32_t* reachable, uint8_t* start_ok, void* stream) {
  OcEsdfField ef;
  int rc = ot_params(m, submap, clearance, max_cost, what, &ef);
  if (rc) return rc;
  f.track.ready = 0;  // until this update has completed
  f.S = S;
  f.nt = 0;  // (until classify has counted the slots)
  if (!f.blk) TS_CUDA(cudaMalloc(&f.blk, otm_blk_bytes((size_t)m->g.max_blocks)));
  std::vector<int> h_start(4 * (size_t)S);
  for (int s = 0; s < S; s++) h_start[4 * s + 3] = ot_start_cell(m, starts + 3 * s, &h_start[4 * s]) ? 1 : 0;
  cudaStream_t st = (cudaStream_t)stream;
  OtmAux a = otm_aux(m, f);
  TS_CUDA(cudaMemsetAsync(a.changed, 0, ((ES_MAX_SWEEPS + 2) + 4) * 4, st));  // changed, counts
  TS_CUDA(cudaMemsetAsync(a.reach, 0, (size_t)S * 4, st));
  TS_CUDA(cudaMemcpyAsync(a.start, h_start.data(), h_start.size() * 4, cudaMemcpyHostToDevice, st));
  const int grid = m->sm_count * 8;
  k_octo_travel_multi_classify<<<grid, OT_THREADS, 0, st>>>(m->g, a, ef, submap, m->lo.l_occ, clearance);
  TS_LAUNCH_CHECK(m);
  int h_counts[2] = {0, 0};
  TS_CUDA(cudaMemcpyAsync(h_counts, a.counts, 8, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  f.nt = h_counts[1];
  const size_t need = std::max(otm_bytes((size_t)f.nt, (size_t)S), (size_t)256);
  if (need > f.bytes) {  // grow geometrically: a map that keeps growing reallocates O(log) times
    const size_t bytes = std::max(need, std::min(2 * f.bytes, otm_bytes((size_t)m->g.max_blocks, (size_t)S)));
    if (f.mem) cudaFree(f.mem);
    f.mem = nullptr;
    f.bytes = 0;
    TS_CUDA(cudaMalloc(&f.mem, bytes));
    f.bytes = bytes;
  }
  a = otm_aux(m, f);
  k_octo_travel_multi_tables<<<grid, OT_THREADS, 0, st>>>(m->g, a);
  TS_LAUNCH_CHECK(m);
  k_octo_travel_multi_fill<<<m->sm_count * 16, OT_THREADS, 0, st>>>(a);
  TS_LAUNCH_CHECK(m);
  k_octo_travel_multi_starts<<<(S + 127) / 128, 128, 0, st>>>(m->g, a, submap);
  TS_LAUNCH_CHECK(m);
  const int sgrid = m->sm_count * 16;
  int sweeps = 0;
  rc = es_wave(m, st, a.changed, ES_GROUP,
               [&](int k) { k_octo_travel_multi_sweep<<<sgrid, OT_THREADS, 0, st>>>(a, k, m->in.vs, max_cost); }, &sweeps);
  if (rc) return rc;
  if (sweeps > ES_MAX_SWEEPS) {  // the last sweep still changed something: the fields are not the fixed point
    ts_set_error("%s: the waves were still changing after %d sweeps; the fields are incomplete and their readers refuse", what, ES_MAX_SWEEPS);
    return TSLAM_E_INVALID;
  }
  k_octo_travel_multi_count<<<sgrid, OT_THREADS, 0, st>>>(a);
  TS_LAUNCH_CHECK(m);
  std::vector<int> h_reach(S), h_item(S);
  TS_CUDA(cudaMemcpyAsync(h_reach.data(), a.reach, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(h_item.data(), a.sitem, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  f.track = OcTrack{1, submap};
  if (stats2) { stats2[0] = sweeps; stats2[1] = h_counts[0]; }
  for (int s = 0; s < S; s++) {
    if (reachable) reachable[s] = h_reach[s];
    if (start_ok) start_ok[s] = h_item[s] >= 0 ? 1 : 0;
  }
  return TSLAM_OK;
}

extern "C" int tslam_octo_travel_update(tslam_octo_t* m, int32_t submap, const float* start3, float clearance, float max_cost,
                                        int32_t* stats4, void* stream) {
  const char* what = "tslam_octo_travel_update";
  if (!m || !start3) return TSLAM_E_INVALID;
  int rc = oc_logodds_submap(m, submap, what, OT_FEATURE);
  if (rc) return rc;
  if (!(std::isfinite(start3[0]) && std::isfinite(start3[1]) && std::isfinite(start3[2]))) {
    ts_set_error("%s: the start must be finite", what);
    return TSLAM_E_INVALID;
  }
  int32_t stats2[2], reachable;
  uint8_t start_ok;
  rc = ot_update(m, m->tr, submap, 1, start3, clearance, max_cost, what, stats2, &reachable, &start_ok, stream);
  if (rc) return rc;
  if (stats4) { stats4[0] = reachable; stats4[1] = stats2[0]; stats4[2] = stats2[1]; stats4[3] = start_ok; }
  return TSLAM_OK;
}

extern "C" int tslam_octo_travel_gather(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, float* cost, int64_t* n_out,
                                        void* stream) {
  if (!m || !n_out || cap < 0 || (cap > 0 && (!idx || !cost))) return TSLAM_E_INVALID;
  const char* what = "tslam_octo_travel_gather";
  int rc = oc_track_readable(m, m->tr.track, submap, what, OT_UPDATE);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return oc_counted_gather(m, st, [&](unsigned long long* ctr) {
    k_octo_travel_slot_gather<<<m->sm_count * 8, OT_THREADS, 0, st>>>(m->g, otm_aux(m, m->tr), 0, cap, idx, cost, ctr);
  }, cap, n_out, what);
}

extern "C" int tslam_octo_travel_query(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, float* cost, void* stream) {
  if (!m || n < 0 || (n && (!xyz || !cost))) return TSLAM_E_INVALID;
  int rc = oc_track_readable(m, m->tr.track, submap, "tslam_octo_travel_query", OT_UPDATE);
  if (rc || n == 0) return rc;
  k_octo_travel_multi_query<<<oc_grid(n, 256, m->sm_count * 16), 256, 0, (cudaStream_t)stream>>>(m->g, otm_aux(m, m->tr), submap, n,
                                                                                                 xyz, m->in.vs, cost);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

extern "C" int tslam_octo_travel_path(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, int32_t max_len, int32_t* cells,
                                      int32_t* len, void* stream) {
  if (!m || n < 0 || (n && (!xyz || !cells || !len))) return TSLAM_E_INVALID;
  const char* what = "tslam_octo_travel_path";
  if (max_len < 1) { ts_set_error("%s: max_len must be >= 1 (got %d)", what, max_len); return TSLAM_E_INVALID; }
  int rc = oc_track_readable(m, m->tr.track, submap, what, OT_UPDATE);
  if (rc || n == 0) return rc;
  k_octo_travel_multi_path<<<oc_grid(n, 256, m->sm_count * 16), 256, 0, (cudaStream_t)stream>>>(m->g, otm_aux(m, m->tr), submap, n,
                                                                                                nullptr, xyz, m->in.vs, max_len, cells, len);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

extern "C" int tslam_octo_travel_multi_update(tslam_octo_t* m, int32_t submap, int32_t n_starts, const float* starts, float clearance,
                                              float max_cost, int32_t* stats2, int32_t* reachable, uint8_t* start_ok, void* stream) {
  const char* what = "tslam_octo_travel_multi_update";
  if (!m || !starts) return TSLAM_E_INVALID;
  int rc = oc_logodds_submap(m, submap, what, OT_FEATURE);
  if (rc) return rc;
  if (n_starts < 1 || n_starts > TSLAM_OCTO_TRAVEL_MAX_STARTS) {
    ts_set_error("%s: n_starts must be in [1, %d] (got %d)", what, TSLAM_OCTO_TRAVEL_MAX_STARTS, n_starts);
    return TSLAM_E_INVALID;
  }
  for (int q = 0; q < 3 * n_starts; q++)
    if (!std::isfinite(starts[q])) {
      ts_set_error("%s: start %d is not finite", what, q / 3);
      return TSLAM_E_INVALID;
    }
  return ot_update(m, m->trm, submap, n_starts, starts, clearance, max_cost, what, stats2, reachable, start_ok, stream);
}

extern "C" int tslam_octo_travel_multi_query(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, float* cost, void* stream) {
  if (!m || n < 0 || (n && (!xyz || !cost))) return TSLAM_E_INVALID;
  int rc = oc_track_readable(m, m->trm.track, submap, "tslam_octo_travel_multi_query", OTM_UPDATE);
  if (rc || n == 0) return rc;
  k_octo_travel_multi_query<<<oc_grid(n, 256, m->sm_count * 16), 256, 0, (cudaStream_t)stream>>>(m->g, otm_aux(m, m->trm), submap, n,
                                                                                                 xyz, m->in.vs, cost);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

extern "C" int tslam_octo_travel_multi_path(tslam_octo_t* m, int32_t submap, int64_t n, const int32_t* source, const float* xyz,
                                            int32_t max_len, int32_t* cells, int32_t* len, void* stream) {
  if (!m || n < 0 || (n && (!source || !xyz || !cells || !len))) return TSLAM_E_INVALID;
  const char* what = "tslam_octo_travel_multi_path";
  if (max_len < 1) { ts_set_error("%s: max_len must be >= 1 (got %d)", what, max_len); return TSLAM_E_INVALID; }
  int rc = oc_track_readable(m, m->trm.track, submap, what, OTM_UPDATE);
  if (rc || n == 0) return rc;
  k_octo_travel_multi_path<<<oc_grid(n, 256, m->sm_count * 16), 256, 0, (cudaStream_t)stream>>>(m->g, otm_aux(m, m->trm), submap, n,
                                                                                                source, xyz, m->in.vs, max_len, cells, len);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
