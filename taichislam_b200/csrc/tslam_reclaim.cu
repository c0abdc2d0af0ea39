// libtslam.so - reclaim of TSDF pool blocks (tslam_tsdf_reclaim, DESIGN.md section 7, "Reclaiming pool blocks").  sm_90a.
//
// Every reader walks the pool as the dense range [0, n_blocks) and takes the slots beyond it to be zero-filled, so blocks
// are not put on a free list: the pool is compacted in place.
//   classify  one CTA per pool block: candidate (submap selected), outside (key only), empty (obs plane, on a fusion
//             destination with valid sums also every sum word, a block flagged for a pending commit is not empty);
//             keep flag, per-submap counts of the non-empty blocks dropped
//   scan      CUB exclusive sum of the keep flags: hole k = the k-th dropped slot below n_keep, mover k = the k-th kept
//             slot at or above n_keep (both ascending)
//   move      mover k -> hole k for every per-block plane (16-byte copies, one CTA per (pair, plane)) and the per-block
//             words (block key, dirty flag, ESDF dirty flag, commit stamp)
//   tail      [n_keep, n_old) of every plane zeroed (cudaMemsetAsync), n_blocks = n_keep
//   rebuild   table cleared, every kept key inserted with its new slot (ts_insert_slot)
#include <cub/cub.cuh>
#include <cmath>
#include <cstring>
#include <vector>
#include "tslam_internal.cuh"

#define RC_PLANES 16  // per-block planes of a map: acc tw obs occ esdf cword col + up to 6 sum planes

enum { RC_C_CAND = 0, RC_C_DROP, RC_C_DROP_NE, RC_C_GHOST, RC_C_N };

struct RcPlane {
  char* p;           // plane base
  unsigned bytes;    // bytes per block (a multiple of 16)
  int limit;         // blocks the plane covers: a hole at or above it is skipped, a mover at or above it reads as zeros
};
struct RcPlanes {
  RcPlane pl[RC_PLANES];
  int n;
};

struct RcSel {
  const uint8_t* mask;  // [max_submaps] or null = every submap
  int rules;
  double cx, cy, cz, r2;
  float vs;
  const long long* sums;  // fusion sum planes when they are valid, else null
  size_t sum_stride;      // elements per sum plane
  int sum_planes;
  int sum_cap;            // blocks the sum planes cover
};

// every 16-byte word of the 4096 * `bytes` bytes of a block's plane, OR-reduced over the CTA (256 threads)
__device__ __forceinline__ bool rc_any_nonzero(const uint4* p, int n16) {
  unsigned any = 0;
  for (int i = threadIdx.x; i < n16; i += blockDim.x) {
    const uint4 v = p[i];
    any |= v.x | v.y | v.z | v.w;
  }
  return __syncthreads_or(any != 0) != 0;
}

// voxel positions of a block along one axis: (float)(16 b + t) * vs, t = 0 .. 15; squared distance of c to their span
__device__ __forceinline__ double rc_axis_d2(double c, int b, float vs) {
  const double lo = (double)((float)(b * TS_B) * vs), hi = (double)((float)(b * TS_B + TS_B - 1) * vs);
  const double q = c < lo ? lo : (c > hi ? hi : c);
  const double d = c - q;
  return d * d;
}

__global__ void __launch_bounds__(256) k_rc_classify(TsGrid g, int nb, RcSel sel, int* keep, int* sub_ne, unsigned long long* ctr) {
  unsigned long long n_cand = 0, n_drop = 0, n_ne = 0, n_ghost = 0;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    n_ghost += g.ghost[b] != 0;
    const bool cand = !sel.mask || sel.mask[s];
    bool outside = false;
    if (cand && (sel.rules & TSLAM_RECLAIM_OUTSIDE))
      outside = (rc_axis_d2(sel.cx, bx, sel.vs) + rc_axis_d2(sel.cy, by, sel.vs)) + rc_axis_d2(sel.cz, bz, sel.vs) > sel.r2;
    const bool forced = cand && ((sel.rules & TSLAM_RECLAIM_ALL) || outside);
    bool drop = false, nonempty = false;
    if (forced || (cand && (sel.rules & TSLAM_RECLAIM_EMPTY))) {
      const size_t base = (size_t)b * TS_B3;
      nonempty = g.dirty_flag[b] != 0 || rc_any_nonzero(reinterpret_cast<const uint4*>(g.obs + base), TS_B3 / 16);
      if (sel.sums && b < sel.sum_cap)
        for (int p = 0; p < sel.sum_planes && !nonempty; p++)
          nonempty = rc_any_nonzero(reinterpret_cast<const uint4*>(sel.sums + (size_t)p * sel.sum_stride + base), TS_B3 / 2);
      drop = forced || !nonempty;
    }
    if (threadIdx.x == 0) {
      keep[b] = drop ? 0 : 1;
      n_cand += cand;
      n_drop += drop;
      if (drop && nonempty) {
        n_ne++;
        atomicAdd(&sub_ne[s], 1);
      }
    }
  }
  if (threadIdx.x == 0) {
    if (n_cand) atomicAdd(&ctr[RC_C_CAND], n_cand);
    if (n_drop) atomicAdd(&ctr[RC_C_DROP], n_drop);
    if (n_ne) atomicAdd(&ctr[RC_C_DROP_NE], n_ne);
    if (n_ghost) atomicAdd(&ctr[RC_C_GHOST], n_ghost);
  }
}

// pos[b] = kept slots before b (exclusive scan of keep): slot b < n_keep dropped is hole b - pos[b]; slot b >= n_keep
// kept is mover pos[b] - pos[n_keep]
__global__ void __launch_bounds__(256) k_rc_pairs(int nb, int n_keep, const int* keep, const int* pos, int* hole, int* mover) {
  const int base = pos[n_keep];
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    if (b < n_keep && !keep[b]) hole[b - pos[b]] = b;
    if (b >= n_keep && keep[b]) mover[pos[b] - base] = b;
  }
}

// blockIdx.y = plane; CTAs stride over the pairs.  Holes and movers are disjoint, so the copies cannot overlap.
__global__ void __launch_bounds__(256) k_rc_move(RcPlanes P, int n_pairs, const int* hole, const int* mover) {
  const RcPlane pl = P.pl[blockIdx.y];
  const int n16 = (int)(pl.bytes / 16);
  for (int q = blockIdx.x; q < n_pairs; q += gridDim.x) {
    const int h = hole[q], m = mover[q];
    if (h >= pl.limit) continue;
    uint4* d = reinterpret_cast<uint4*>(pl.p + (size_t)h * pl.bytes);
    if (m >= pl.limit) {
      for (int i = threadIdx.x; i < n16; i += blockDim.x) d[i] = make_uint4(0u, 0u, 0u, 0u);
    } else {
      const uint4* s = reinterpret_cast<const uint4*>(pl.p + (size_t)m * pl.bytes);
      for (int i = threadIdx.x; i < n16; i += blockDim.x) d[i] = s[i];
    }
  }
}

// the per-block words of the pairs: block key, dirty flag, ESDF dirty flag, commit stamp (ghost flags are all zero:
// a map with ghost blocks is refused)
__global__ void __launch_bounds__(256) k_rc_move_words(TsGrid g, unsigned long long* stamp, int n_pairs, const int* hole, const int* mover) {
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < n_pairs; q += gridDim.x * blockDim.x) {
    const int h = hole[q], m = mover[q];
    g.block_key[h] = g.block_key[m];
    g.dirty_flag[h] = g.dirty_flag[m];
    g.esdf_dirty[h] = g.esdf_dirty[m];
    stamp[h] = stamp[m];
  }
}

__global__ void __launch_bounds__(256) k_rc_rebuild(TsGrid g, int n_keep) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < n_keep; b += gridDim.x * blockDim.x)
    if (!ts_insert_slot(g, g.block_key[b], b)) atomicOr(g.err, TS_ERR_TABLE_FULL);
}

__global__ void __launch_bounds__(256) k_rc_keys(TsGrid g, int nb, long long cap, int32_t* keys4) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb && b < cap; b += gridDim.x * blockDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    keys4[4 * (size_t)b] = s;
    keys4[4 * (size_t)b + 1] = bx;
    keys4[4 * (size_t)b + 2] = by;
    keys4[4 * (size_t)b + 3] = bz;
  }
}

// ---------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------
static size_t rc_align(size_t x) { return (x + 255) & ~(size_t)255; }

static int rc_pool_size(tslam_tsdf* m, cudaStream_t st, int* nb) {
  TS_CUDA(cudaMemcpyAsync(nb, m->g.n_blocks, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (*nb > m->g.max_blocks) *nb = m->g.max_blocks;
  return TSLAM_OK;
}

// every per-block plane of m with its bytes per block; the fusion sum planes up to the blocks they cover
static RcPlanes rc_planes(tslam_tsdf* m, const TsFuseView& fz) {
  RcPlanes P;
  P.n = 0;
  const TsGrid& g = m->g;
  auto add = [&](void* p, unsigned bytes, int limit) {
    if (p) P.pl[P.n++] = RcPlane{(char*)p, bytes, limit};
  };
  add(g.acc, TS_B3 * 8, g.max_blocks);
  add(g.tw, TS_B3 * 8, g.max_blocks);
  add(g.obs, TS_B3, g.max_blocks);
  add(g.occ, TS_B3, g.max_blocks);
  add(g.esdf, TS_B3 * 4, g.max_blocks);
  add(g.cword, TS_B3 * 8, g.max_blocks);
  add(g.col, TS_B3 * 16, g.max_blocks);
  if (fz.sums)
    for (int p = 0; p < fz.planes; p++) add(fz.sums + (size_t)p * fz.cap_blocks * TS_B3, TS_B3 * 8, (int)fz.cap_blocks);
  return P;
}

extern "C" int tslam_tsdf_reclaim(tslam_tsdf_t* m, int32_t rules, const uint8_t* submaps, const double* center3, double radius,
                                  int64_t* stats6, void* stream) {
  const int known = TSLAM_RECLAIM_ALL | TSLAM_RECLAIM_EMPTY | TSLAM_RECLAIM_OUTSIDE;
  if (rules == 0 || (rules & ~known)) { ts_set_error("reclaim: rules 0x%x must be a non-empty set of TSLAM_RECLAIM_ALL / _EMPTY / _OUTSIDE", (unsigned)rules); return TSLAM_E_INVALID; }
  if (rules & TSLAM_RECLAIM_OUTSIDE) {
    if (!std::isfinite(radius) || radius < 0.0) { ts_set_error("reclaim: radius %g must be finite and >= 0", radius); return TSLAM_E_INVALID; }
    if (!center3) { ts_set_error("reclaim: OUTSIDE needs a centre (center3 is NULL)"); return TSLAM_E_INVALID; }
    if (!std::isfinite(center3[0]) || !std::isfinite(center3[1]) || !std::isfinite(center3[2])) {
      ts_set_error("reclaim: centre (%g, %g, %g) is not finite", center3[0], center3[1], center3[2]);
      return TSLAM_E_INVALID;
    }
  }
  if (!m) { ts_set_error("reclaim: NULL handle"); return TSLAM_E_INVALID; }

  if (m->tile_cuts_set) { ts_set_error("reclaim: the map is a tiled map (tile cuts set): not supported"); return TSLAM_E_INVALID; }
  if (m->esdf_tiled == 1) { ts_set_error("reclaim: a tiled ESDF exchange is open (tslam_esdf_tiled_begin without _end)"); return TSLAM_E_INVALID; }
  const TsFuseView fz = ts_fuse_view(m);
  if (fz.phase != 0) { ts_set_error("reclaim: a tiled fusion update is in progress on this map"); return TSLAM_E_INVALID; }

  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  int nb = 0;
  rc = rc_pool_size(m, st, &nb);
  if (rc) return rc;

  // scratch: keep[nb], pos[nb], hole[nb], mover[nb], sub_ne[S], ctr[RC_C_N], mask[S], CUB temp
  const int S = m->cfg.max_submaps;
  size_t scan_tmp = 0;
  TS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (int*)nullptr, (int*)nullptr, nb, st));
  const size_t nbs = rc_align((size_t)(nb + 1) * 4), ss = rc_align((size_t)S * 4), cs = rc_align(RC_C_N * 8);
  rc = rg_reserve(&m->rc_mem, &m->rc_bytes, 4 * nbs + ss + cs + rc_align(scan_tmp) + 256 + (size_t)S);
  if (rc) return rc;
  char* w = (char*)m->rc_mem;
  int* keep = (int*)w; w += nbs;
  int* pos = (int*)w; w += nbs;
  int* hole = (int*)w; w += nbs;
  int* mover = (int*)w; w += nbs;
  int* sub_ne = (int*)w; w += ss;
  unsigned long long* ctr = (unsigned long long*)w; w += cs;
  uint8_t* mask = (uint8_t*)w; w += rc_align((size_t)S);
  void* tmp = w;

  RcSel sel;
  sel.mask = nullptr;
  if (submaps) {
    TS_CUDA(cudaMemcpyAsync(mask, submaps, (size_t)S, cudaMemcpyHostToDevice, st));
    sel.mask = mask;
  }
  sel.rules = rules;
  sel.cx = sel.cy = sel.cz = sel.r2 = 0.0;
  if (rules & TSLAM_RECLAIM_OUTSIDE) { sel.cx = center3[0]; sel.cy = center3[1]; sel.cz = center3[2]; sel.r2 = radius * radius; }
  sel.vs = m->in.vs;
  const bool sums_valid = fz.sums && fz.valid;
  sel.sums = sums_valid ? fz.sums : nullptr;
  sel.sum_stride = fz.cap_blocks * TS_B3;
  sel.sum_planes = fz.planes;
  sel.sum_cap = (int)fz.cap_blocks;

  TS_CUDA(cudaMemsetAsync(sub_ne, 0, (size_t)S * 4, st));
  TS_CUDA(cudaMemsetAsync(ctr, 0, RC_C_N * 8, st));
  if (nb > 0) {
    k_rc_classify<<<oc_grid(nb, 1, m->sm_count * 8), 256, 0, st>>>(m->g, nb, sel, keep, sub_ne, ctr);
    TS_LAUNCH_CHECK(m);
  }
  unsigned long long hc[RC_C_N];
  std::vector<int> h_ne(S);
  TS_CUDA(cudaMemcpyAsync(hc, ctr, sizeof(hc), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(h_ne.data(), sub_ne, (size_t)S * 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (hc[RC_C_GHOST]) { ts_set_error("reclaim: the map holds %llu ghost blocks (a tiled map): not supported", hc[RC_C_GHOST]); return TSLAM_E_INVALID; }

  const int n_drop = (int)hc[RC_C_DROP], n_keep = nb - n_drop;
  int n_pairs = 0;
  if (n_drop > 0) {
    // pairs: the dropped slots below n_keep, as many as the kept slots at or above it
    TS_CUDA(cub::DeviceScan::ExclusiveSum(tmp, scan_tmp, keep, pos, nb, st));
    TS_CUDA(cudaMemcpyAsync(&n_pairs, pos + n_keep, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
    n_pairs = n_keep - n_pairs;
    if (n_pairs > 0) {
      k_rc_pairs<<<oc_grid(nb, 256, m->sm_count * 8), 256, 0, st>>>(nb, n_keep, keep, pos, hole, mover);
      TS_LAUNCH_CHECK(m);
      const RcPlanes P = rc_planes(m, fz);
      k_rc_move<<<dim3((unsigned)oc_grid(n_pairs, 1, m->sm_count * 4), (unsigned)P.n), 256, 0, st>>>(P, n_pairs, hole, mover);
      TS_LAUNCH_CHECK(m);
      k_rc_move_words<<<oc_grid(n_pairs, 256, m->sm_count * 4), 256, 0, st>>>(m->g, m->blk_stamp, n_pairs, hole, mover);
      TS_LAUNCH_CHECK(m);
    }
    // tail [n_keep, nb) of every plane and per-block word
    const RcPlanes P = rc_planes(m, fz);
    for (int i = 0; i < P.n; i++) {
      const int hi = nb < P.pl[i].limit ? nb : P.pl[i].limit;
      if (hi > n_keep) TS_CUDA(cudaMemsetAsync(P.pl[i].p + (size_t)n_keep * P.pl[i].bytes, 0, (size_t)(hi - n_keep) * P.pl[i].bytes, st));
    }
    const size_t nt = (size_t)n_drop;
    TS_CUDA(cudaMemsetAsync(m->g.block_key + n_keep, 0, nt * 8, st));
    TS_CUDA(cudaMemsetAsync(m->g.dirty_flag + n_keep, 0, nt * 4, st));
    TS_CUDA(cudaMemsetAsync(m->g.esdf_dirty + n_keep, 0, nt * 4, st));
    TS_CUDA(cudaMemsetAsync(m->blk_stamp + n_keep, 0, nt * 8, st));
    TS_CUDA(cudaMemsetAsync(m->g.ghost + n_keep, 0, nt, st));
    // the table: cleared (overflow entries go with it), every kept key at its slot
    TS_CUDA(cudaMemsetAsync(m->g.table, 0xFF, m->table_cap * 8, st));
    if (n_keep > 0) {
      k_rc_rebuild<<<oc_grid(n_keep, 256, m->sm_count * 8), 256, 0, st>>>(m->g, n_keep);
      TS_LAUNCH_CHECK(m);
    }
    TS_CUDA(cudaMemcpyAsync(m->g.n_blocks, &n_keep, 4, cudaMemcpyHostToDevice, st));
    TS_CUDA(cudaStreamSynchronize(st));
    // what indexes pool slots without moving with its block: the incremental mesh and the ESDF's kept state
    m->mesh_epoch++;
    m->esdf_full_needed = 1;
    for (int s = 0; s < S; s++)
      if (h_ne[s]) fz_written(m->ver, s);  // lost observed content; empty blocks are no content change
  }
  if (stats6) {
    stats6[0] = nb;
    stats6[1] = (int64_t)hc[RC_C_CAND];
    stats6[2] = n_drop;
    stats6[3] = (int64_t)hc[RC_C_DROP_NE];
    stats6[4] = n_pairs;
    stats6[5] = n_keep;
  }
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_block_keys(tslam_tsdf_t* m, int64_t cap, int32_t* keys4, int64_t* n_out, void* stream) {
  if (!m || !n_out || cap < 0 || (cap > 0 && !keys4)) { ts_set_error("block_keys: NULL handle, n_out or keys4, or cap < 0"); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  int nb = 0;
  rc = rc_pool_size(m, st, &nb);
  if (rc) return rc;
  if (nb > 0 && cap > 0) {
    k_rc_keys<<<oc_grid(nb, 256, m->sm_count * 8), 256, 0, st>>>(m->g, nb, cap, keys4);
    TS_LAUNCH_CHECK(m);
    TS_CUDA(cudaStreamSynchronize(st));
  }
  *n_out = nb;
  if (nb > cap) { ts_set_error("block_keys: %d pool blocks > capacity %lld", nb, (long long)cap); return TSLAM_E_CAPACITY; }
  return TSLAM_OK;
}
