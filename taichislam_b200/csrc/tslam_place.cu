// libtslam.so - place recognition between TSDF submaps (tslam_tsdf_place_describe, tslam_place_match; DESIGN.md section 7,
// "Loop detection"): a Scan Context descriptor (Kim & Kim, IROS 2018) of each submap, built from the points registration
// selects, and a batched search that returns, per query submap, a shortlist of database entries with a coarse 4-DoF pose
// (yaw, x, y) for each.  The caller verifies the shortlisted pairs with tslam_tsdf_register started from that pose.
//   describe   the registration point selection (rg_select_count / rg_select_fill, tslam_register.cu), then one CTA per
//              submap (k_pl_describe): its points are levelled (x = M p_v), binned into 20 rings x 60 sectors and a
//              128 x 128 bird's-eye grid, and each bin keeps the min and max height through shared-memory atomics on an
//              order-preserving integer image of the f32 height.  The CTA's epilogue writes the polar spans, the ring key
//              and the bitmap (one ballot per 32 cells), so the 140 KB of bins never leave shared memory.
//   match      k_pl_shortlist (one CTA per query: ring distances, then top_k rounds of a block-wide min over
//              (distance, index) keys); k_pl_shift (one warp per (query, slot), shifts across lanes); k_pl_bev (one CTA
//              per (query, slot, yaw): both bitmaps in shared memory, offsets across threads, popc of shifted 128-bit
//              rows); k_pl_pick (the best of the three yaws per (query, slot)).
// Min and max commute and every sum runs in a fixed order, so every output is the same bits whatever the order of the
// atomics, and a query's outputs do not depend on the other queries of the call.
#include <cmath>
#include <cstring>
#include <vector>
#include "tslam_internal.cuh"

#define PL_R 20                       // rings
#define PL_S 60                       // sectors
#define PL_BINS (PL_R * PL_S)
#define PL_G 128                      // bird's-eye cells per axis
#define PL_CELLS (PL_G * PL_G)
#define PL_WORDS (PL_CELLS / 32)      // 4 words per row
#define PL_DT 1024                    // threads of k_pl_describe
#define PL_OFF 32                     // offsets dx, dy in [-PL_OFF, PL_OFF]
#define PL_NOFF ((2 * PL_OFF + 1) * (2 * PL_OFF + 1))
#define PL_MAX_N 1024

struct PlTables {           // host-made f32 tables of a describe call
  float B[PL_R];            // (r_max (i + 1) / 20)^2
  float c[PL_S + 1], s[PL_S + 1];  // cos, sin (2 pi k / 60), k = 0 .. 60 (entry 60 = entry 0)
  float cell, h_min;        // r_max / 64, h_min
};
struct PlYaw { float c[2 * PL_S], s[2 * PL_S]; };  // cos, sin (2 pi h / 120): yaw h x 3 degrees

// order-preserving u32 image of a finite f32 (0 is below every image, ~0u above: the empty bin's max and min)
__device__ __forceinline__ unsigned pl_key(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float pl_unkey(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// CTA q: the points pts[rng[2q] .. rng[2q + 1]) of entry q, levelled by M[q] (f32 row-major, pose_apply with t = 0)
__global__ void __launch_bounds__(PL_DT) k_pl_describe(const float4* __restrict__ pts, const long long* __restrict__ rng,
                                                       const float* __restrict__ M, PlTables tb, float* __restrict__ sc,
                                                       float* __restrict__ ring, unsigned* __restrict__ bev) {
  extern __shared__ unsigned pl_sh[];
  unsigned* pmin = pl_sh;
  unsigned* pmax = pl_sh + PL_BINS;
  unsigned* bmin = pl_sh + 2 * PL_BINS;
  unsigned* bmax = bmin + PL_CELLS;
  __shared__ int s_ring[PL_R];
  const int q = blockIdx.x;
  for (int i = threadIdx.x; i < PL_BINS; i += PL_DT) { pmin[i] = 0xffffffffu; pmax[i] = 0u; }
  for (int i = threadIdx.x; i < PL_CELLS; i += PL_DT) { bmin[i] = 0xffffffffu; bmax[i] = 0u; }
  if (threadIdx.x < PL_R) s_ring[threadIdx.x] = 0;
  float R[9];
#pragma unroll
  for (int i = 0; i < 9; i++) R[i] = M[9 * q + i];
  const float t0[3] = {0.0f, 0.0f, 0.0f};
  __syncthreads();
  const long long e = rng[2 * q + 1];
  for (long long i = rng[2 * q] + threadIdx.x; i < e; i += PL_DT) {
    const float4 p = pts[i];
    float x0, x1, x2;
    pose_apply(R, t0, p.x, p.y, p.z, x0, x1, x2);
    const unsigned kz = pl_key(x2);
    const float r2 = x0 * x0 + x1 * x1;
    if (r2 < tb.B[PL_R - 1]) {
      int r = 0;
      while (!(r2 < tb.B[r])) r++;
      int s = 0;  // the first wedge k with f_k >= 0 and f_{k+1} < 0; none (rho^2 = 0): sector 0
      float f = tb.c[0] * x1 - tb.s[0] * x0;
      for (int k = 0; k < PL_S; k++) {
        const float g = tb.c[k + 1] * x1 - tb.s[k + 1] * x0;
        if (f >= 0.0f && g < 0.0f) { s = k; break; }
        f = g;
      }
      atomicMin(&pmin[r * PL_S + s], kz);
      atomicMax(&pmax[r * PL_S + s], kz);
    }
    const float fu = floorf(x0 / tb.cell), fv = floorf(x1 / tb.cell);
    if (fu >= -64.0f && fu < 64.0f && fv >= -64.0f && fv < 64.0f) {
      const int c = ((int)fu + 64) * PL_G + ((int)fv + 64);
      atomicMin(&bmin[c], kz);
      atomicMax(&bmax[c], kz);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < PL_BINS; i += PL_DT) {
    const bool any = pmax[i] != 0u;
    sc[(size_t)q * PL_BINS + i] = any ? pl_unkey(pmax[i]) - pl_unkey(pmin[i]) : 0.0f;
    if (any) atomicAdd(&s_ring[i / PL_S], 1);
  }
  const int lane = threadIdx.x & 31;
  for (int wd = threadIdx.x >> 5; wd < PL_WORDS; wd += PL_DT / 32) {
    const int c = wd * 32 + lane;
    const bool bit = bmax[c] != 0u && pl_unkey(bmax[c]) - pl_unkey(bmin[c]) >= tb.h_min;
    const unsigned word = __ballot_sync(0xffffffffu, bit);
    if (lane == 0) bev[(size_t)q * PL_WORDS + wd] = word;
  }
  __syncthreads();
  if (threadIdx.x < PL_R) ring[q * PL_R + threadIdx.x] = (float)s_ring[threadIdx.x] / 60.0f;
}

__device__ __forceinline__ unsigned long long pl_warp_min(unsigned long long v) {
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w < v ? w : v;
  }
  return v;
}

// CTA qi: query q = queries[qi] against every entry d < n_db (thread d).  key = (f32 bits of the ring distance, d), ~0
// when d is not eligible; top_k rounds take the least key and retire it.  match -1 / distance 0 past the eligible ones.
__global__ void __launch_bounds__(PL_MAX_N) k_pl_shortlist(int n_db, const float* __restrict__ ring, const long long* __restrict__ npts,
                                                           const long long* __restrict__ ids, const int* __restrict__ queries,
                                                           int top_k, long long min_gap, long long min_points, int* __restrict__ info,
                                                           float* __restrict__ dist) {
  __shared__ unsigned long long s_w[PL_MAX_N / 32];
  __shared__ unsigned long long s_best;
  __shared__ float s_kq[PL_R];
  const int qi = blockIdx.x, q = queries[qi], d = threadIdx.x, lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  if (threadIdx.x < PL_R) s_kq[threadIdx.x] = ring[q * PL_R + threadIdx.x];
  __syncthreads();
  unsigned long long key = ~0ull;
  if (d < n_db && d != q && npts[q] >= min_points && npts[d] >= min_points) {
    const long long a = ids[q], b = ids[d];
    const unsigned long long gap = a >= b ? (unsigned long long)a - (unsigned long long)b : (unsigned long long)b - (unsigned long long)a;
    if (gap >= (unsigned long long)min_gap) {
      float acc = 0.0f;
      for (int i = 0; i < PL_R; i++) {
        const float t = s_kq[i] - ring[d * PL_R + i];
        acc = acc + t * t;
      }
      key = (unsigned long long)__float_as_uint(acc) << 32 | (unsigned)d;
    }
  }
  for (int k = 0; k < top_k; k++) {
    const unsigned long long m = pl_warp_min(key);
    if (lane == 0) s_w[wp] = m;
    __syncthreads();
    if (wp == 0) {
      const unsigned long long v = pl_warp_min(lane < (int)(blockDim.x >> 5) ? s_w[lane] : ~0ull);
      if (lane == 0) s_best = v;
    }
    __syncthreads();
    const unsigned long long best = s_best;
    if (threadIdx.x == 0) {
      const size_t o = (size_t)qi * top_k + k;
      info[6 * o] = best == ~0ull ? -1 : (int)(best & 0xffffffffu);
      dist[3 * o] = best == ~0ull ? 0.0f : __uint_as_float((unsigned)(best >> 32));
    }
    if (key == best) key = ~0ull;  // the index makes the key unique
    __syncthreads();
  }
}

#define PL_SW 4  // warps (pairs) per CTA of k_pl_shift
// warp per pair pr = qi top_k + slot: D(m) for the shifts m = lane, lane + 32, argmin (ties to the smaller m)
__global__ void __launch_bounds__(PL_SW * 32) k_pl_shift(const float* __restrict__ sc, const int* __restrict__ queries, int top_k,
                                                         int n_pairs, int* __restrict__ info, float* __restrict__ dist) {
  __shared__ float s_a[PL_SW][PL_BINS], s_b[PL_SW][PL_BINS], s_na[PL_SW][PL_S], s_nb[PL_SW][PL_S];
  const int wp = threadIdx.x >> 5, lane = threadIdx.x & 31, pr = blockIdx.x * PL_SW + wp;
  if (pr >= n_pairs) return;  // (uniform per warp; no CTA barrier follows)
  const int d = info[6 * pr];
  if (d < 0) {
    if (lane == 0) { info[6 * pr + 1] = 0; dist[3 * pr + 1] = 1.0f; }
    return;
  }
  const int q = queries[pr / top_k];
  float* A = s_a[wp];
  float* B = s_b[wp];
  for (int i = lane; i < PL_BINS; i += 32) { A[i] = sc[(size_t)q * PL_BINS + i]; B[i] = sc[(size_t)d * PL_BINS + i]; }
  __syncwarp();
  for (int j = lane; j < PL_S; j += 32) {
    float a2 = 0.0f, b2 = 0.0f;
    for (int i = 0; i < PL_R; i++) {
      a2 = a2 + A[i * PL_S + j] * A[i * PL_S + j];
      b2 = b2 + B[i * PL_S + j] * B[i * PL_S + j];
    }
    s_na[wp][j] = sqrtf(a2);
    s_nb[wp][j] = sqrtf(b2);
  }
  __syncwarp();
  float best = INFINITY;
  int bm = 0;
  for (int m = lane; m < PL_S; m += 32) {
    float acc = 0.0f;
    int nj = 0;
    for (int j = 0; j < PL_S; j++) {
      const int jb = j + m < PL_S ? j + m : j + m - PL_S;
      const float na = s_na[wp][j], nb = s_nb[wp][jb];
      if (!(na != 0.0f && nb != 0.0f)) continue;
      float dot = 0.0f;
      for (int i = 0; i < PL_R; i++) dot = dot + A[i * PL_S + j] * B[i * PL_S + jb];
      acc = acc + dot / (na * nb);
      nj++;
    }
    const float D = nj ? 1.0f - acc / (float)nj : 1.0f;
    if (D < best) { best = D; bm = m; }  // m ascends per lane: ties keep the smaller m
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int om = __shfl_xor_sync(0xffffffffu, bm, o);
    if (ob < best || (ob == best && om < bm)) { best = ob; bm = om; }
  }
  if (lane == 0) { info[6 * pr + 1] = bm; dist[3 * pr + 1] = best; }
}

// 128-bit row (lo = words 0, 1; hi = words 2, 3; bit v of the row is bit v of the pair) shifted toward higher v by sh
__device__ __forceinline__ void pl_shift_row(unsigned long long lo, unsigned long long hi, int sh, unsigned long long& ol,
                                             unsigned long long& oh) {
  if (sh == 0) { ol = lo; oh = hi; }
  else if (sh > 0) { ol = lo << sh; oh = (hi << sh) | (lo >> (64 - sh)); }
  else { const int r = -sh; oh = hi >> r; ol = (lo >> r) | (hi << (64 - r)); }
}

// CTA (pr, y): q's bitmap rotated by the yaw (2 m* + y - 1) x 3 degrees, correlated with d's over every (dx, dy); key[pr 3
// + y] = (score, 127 - |dx| - |dy|, 2 - y, 32 - dy, 32 - dx) packed so that the largest key is the best; popq = popc(rot q)
__global__ void __launch_bounds__(256) k_pl_bev(const unsigned* __restrict__ bev, const int* __restrict__ queries, int top_k,
                                                const int* __restrict__ info, PlYaw yt, unsigned long long* __restrict__ keys,
                                                int* __restrict__ popc) {
  __shared__ unsigned long long s_q[PL_G][2], s_d[PL_G][2];
  __shared__ int s_rng[4];  // rows holding a bit: q' min, max, d min, max
  __shared__ int s_pop[2];
  __shared__ unsigned long long s_w[8];
  const int pr = blockIdx.x / 3, y = blockIdx.x % 3, lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int d = info[6 * pr];
  if (d < 0) {  // (uniform per CTA)
    if (threadIdx.x == 0) { keys[blockIdx.x] = 0ull; popc[2 * blockIdx.x] = 0; popc[2 * blockIdx.x + 1] = 0; }
    return;
  }
  const int q = queries[pr / top_k];
  const int h = (2 * info[6 * pr + 1] + y - 1 + 2 * PL_S) % (2 * PL_S);
  const float c = yt.c[h], s = yt.s[h];
  const unsigned* Q = bev + (size_t)q * PL_WORDS;
  const unsigned* Dm = bev + (size_t)d * PL_WORDS;
  if (threadIdx.x == 0) { s_rng[0] = PL_G; s_rng[1] = -1; s_rng[2] = PL_G; s_rng[3] = -1; s_pop[0] = 0; s_pop[1] = 0; }
  __syncthreads();
  unsigned* sq = reinterpret_cast<unsigned*>(s_q);
  unsigned* sd = reinterpret_cast<unsigned*>(s_d);
  int pq = 0, pd = 0;
  for (int wd = wp; wd < PL_WORDS; wd += 8) {
    const int cell = wd * 32 + lane, u = cell >> 7, v = cell & 127;
    const float a = (float)(u - 64) + 0.5f, b = (float)(v - 64) + 0.5f;
    const float xs = c * a + s * b, ys = c * b - s * a;  // Rz(-psi) (a, b)
    const float fu = floorf(xs), fv = floorf(ys);
    bool bit = false;
    if (fu >= -64.0f && fu < 64.0f && fv >= -64.0f && fv < 64.0f) {
      const int su = (int)fu + 64, sv = (int)fv + 64;
      bit = (Q[su * 4 + (sv >> 5)] >> (sv & 31)) & 1u;
    }
    const unsigned w = __ballot_sync(0xffffffffu, bit);
    const unsigned wdd = Dm[wd];
    if (lane == 0) {
      sq[wd] = w;
      sd[wd] = wdd;
      pq += __popc(w);
      pd += __popc(wdd);
      if (w) { atomicMin(&s_rng[0], wd >> 2); atomicMax(&s_rng[1], wd >> 2); }
      if (wdd) { atomicMin(&s_rng[2], wd >> 2); atomicMax(&s_rng[3], wd >> 2); }
    }
  }
  if (lane == 0) { atomicAdd(&s_pop[0], pq); atomicAdd(&s_pop[1], pd); }
  __syncthreads();
  const int qa = s_rng[0], qb = s_rng[1], da = s_rng[2], db = s_rng[3];
  unsigned long long best = 0ull;
  for (int o = threadIdx.x; o < PL_NOFF; o += blockDim.x) {
    const int dx = o / (2 * PL_OFF + 1) - PL_OFF, dy = o % (2 * PL_OFF + 1) - PL_OFF;  // neighbours share dx: same rows
    const int u0 = max(da, qa + dx), u1 = min(db, qb + dx);
    int score = 0;
    for (int u = u0; u <= u1; u++) {
      unsigned long long ol, oh;
      pl_shift_row(s_q[u - dx][0], s_q[u - dx][1], dy, ol, oh);
      score += __popcll(ol & s_d[u][0]) + __popcll(oh & s_d[u][1]);
    }
    const int man = abs(dx) + abs(dy);
    const unsigned long long k = (unsigned long long)score << 32 | (unsigned long long)(127 - man) << 24 |
                                 (unsigned long long)(2 - y) << 16 | (unsigned long long)(PL_OFF - dy) << 8 | (unsigned)(PL_OFF - dx);
    best = k > best ? k : best;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, best, o);
    best = w > best ? w : best;
  }
  if (lane == 0) s_w[wp] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long v = 0ull;
    for (int i = 0; i < 8; i++) v = s_w[i] > v ? s_w[i] : v;
    keys[blockIdx.x] = v;
    popc[2 * blockIdx.x] = s_pop[0];
    popc[2 * blockIdx.x + 1] = s_pop[1];
  }
}

// thread per pair: the best of its three yaw keys -> yaw index, dx, dy, score, overlap
__global__ void __launch_bounds__(256) k_pl_pick(int n_pairs, const unsigned long long* __restrict__ keys, const int* __restrict__ popc,
                                                 int* __restrict__ info, float* __restrict__ dist) {
  const int pr = blockIdx.x * blockDim.x + threadIdx.x;
  if (pr >= n_pairs) return;
  int* o = info + 6 * pr;
  if (o[0] < 0) {
    o[2] = o[3] = o[4] = o[5] = 0;
    dist[3 * pr + 2] = 0.0f;
    return;
  }
  unsigned long long k = keys[3 * pr];
  for (int y = 1; y < 3; y++) k = keys[3 * pr + y] > k ? keys[3 * pr + y] : k;
  const int y = 2 - (int)(k >> 16 & 0xff), score = (int)(k >> 32);
  o[2] = y;
  o[3] = PL_OFF - (int)(k & 0xff);
  o[4] = PL_OFF - (int)(k >> 8 & 0xff);
  o[5] = score;
  const int pq = popc[2 * (3 * pr + y)], pd = popc[2 * (3 * pr + y) + 1], den = pq < pd ? pq : pd;
  dist[3 * pr + 2] = den > 0 ? (float)score / (float)den : 0.0f;
}

// ---- host ------------------------------------------------------------------------------------------------------------
static bool pl_pos(float v) { return std::isfinite(v) && v > 0.0f; }

extern "C" int tslam_tsdf_place_describe(tslam_tsdf_t* m, int32_t n, const int32_t* submaps, const float* M9, const tslam_place_params_t* params,
                                         float* sc, float* ring, uint32_t* bev, int64_t* n_points, void* stream) {
  static const char* fn = "tslam_tsdf_place_describe";
  if (n < 1 || n > PL_MAX_N) {
    ts_set_error("%s: n %d outside [1, %d]", fn, n, PL_MAX_N);
    return TSLAM_E_INVALID;
  }
  if (!submaps || !M9 || !params || !sc || !ring || !bev || !n_points) {
    ts_set_error("%s: NULL array or params", fn);
    return TSLAM_E_INVALID;
  }
  const tslam_place_params_t pp = *params;
  if (!pl_pos(pp.r_max) || !pl_pos(pp.h_min) || !pl_pos(pp.band) || !std::isfinite(pp.min_weight)) {
    ts_set_error("%s: r_max, h_min and band must be finite and > 0, min_weight finite", fn);
    return TSLAM_E_INVALID;
  }
  for (int i = 0; i < 9 * n; i++) {
    if (!std::isfinite(M9[i])) {
      ts_set_error("%s: submap %d: levelled rotation not finite", fn, i / 9);
      return TSLAM_E_INVALID;
    }
  }
  if (!m) {
    ts_set_error("%s: NULL handle", fn);
    return TSLAM_E_INVALID;
  }
  for (int i = 0; i < n; i++) {
    if (submaps[i] < 0 || submaps[i] >= m->cfg.max_submaps) {
      ts_set_error("%s: entry %d: submap %d out of range", fn, i, submaps[i]);
      return TSLAM_E_INVALID;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (!rc) rc = ts_check_deferred_async(m, st);
  if (rc) return rc;
  // one selection slot per distinct submap; entry i reads its slot's range (a repeated submap is described again)
  std::vector<int> slot_of(1024, -1), slot_sub, ent_slot(n);
  for (int i = 0; i < n; i++) {
    int& sl = slot_of[submaps[i]];
    if (sl < 0) { sl = (int)slot_sub.size(); slot_sub.push_back(submaps[i]); }
    ent_slot[i] = sl;
  }
  const int U = (int)slot_sub.size();
  RgSel sel;
  std::vector<int> slot_cnt;
  rc = rg_select_count(m, slot_of, U, pp.band, pp.min_weight, sel, slot_cnt, st);
  if (rc) return rc;
  std::vector<long long> slot_p0(U + 1, 0);
  for (int u = 0; u < U; u++) slot_p0[u + 1] = slot_p0[u] + slot_cnt[u];
  // entry i reads the records [ranges[2i], ranges[2i + 1]) of its slot
  std::vector<long long> ranges(2 * (size_t)n);
  for (int i = 0; i < n; i++) { ranges[2 * i] = slot_p0[ent_slot[i]]; ranges[2 * i + 1] = slot_p0[ent_slot[i] + 1]; }
  const size_t pts_b = ((size_t)slot_p0[U] * 16 + 255) & ~(size_t)255, rg_b = ((size_t)n * 16 + 255) & ~(size_t)255;
  rc = rg_reserve(&m->reg_pts, &m->reg_pts_bytes, pts_b + rg_b + (size_t)n * 36);
  if (rc) return rc;
  float4* pts = (float4*)m->reg_pts;
  long long* d_rng = (long long*)((char*)m->reg_pts + pts_b);
  float* d_M = (float*)((char*)m->reg_pts + pts_b + rg_b);
  if (slot_p0[U] > 0) {
    rc = rg_select_fill(m, sel, pp.band, pp.min_weight, pts, st);
    if (rc) return rc;
  }
  TS_CUDA(cudaMemcpyAsync(d_rng, ranges.data(), (size_t)n * 16, cudaMemcpyHostToDevice, st));
  TS_CUDA(cudaMemcpyAsync(d_M, M9, (size_t)n * 36, cudaMemcpyHostToDevice, st));
  PlTables tb;
  for (int i = 0; i < PL_R; i++) {
    const double r = (double)pp.r_max * (double)(i + 1) / 20.0;
    tb.B[i] = (float)(r * r);
  }
  for (int k = 0; k <= PL_S; k++) {
    const double a = 2.0 * M_PI * (double)(k % PL_S) / (double)PL_S;
    tb.c[k] = (float)std::cos(a);
    tb.s[k] = (float)std::sin(a);
  }
  tb.cell = pp.r_max / 64.0f;
  tb.h_min = pp.h_min;
  const int smem = (2 * PL_BINS + 2 * PL_CELLS) * 4;
  TS_CUDA(cudaFuncSetAttribute(k_pl_describe, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_pl_describe<<<n, PL_DT, smem, st>>>(pts, d_rng, d_M, tb, sc, ring, bev);
  TS_LAUNCH_CHECK(m);
  for (int i = 0; i < n; i++) n_points[i] = (int64_t)(ranges[2 * i + 1] - ranges[2 * i]);
  return TSLAM_OK;
}

extern "C" int tslam_place_match(int32_t n_db, const float* sc, const float* ring, const uint32_t* bev, const int64_t* n_points,
                                 const int64_t* ids, int32_t n_q, const int32_t* queries, int32_t top_k, int64_t min_gap,
                                 int64_t min_points, int32_t* info6, float* dist3, void* stream) {
  static const char* fn = "tslam_place_match";
  if (n_db < 1 || n_db > PL_MAX_N || n_q < 1 || n_q > PL_MAX_N) {
    ts_set_error("%s: n_db %d and n_q %d must be in [1, %d]", fn, n_db, n_q, PL_MAX_N);
    return TSLAM_E_INVALID;
  }
  if (top_k < 1 || top_k > TSLAM_PLACE_MAX_TOP_K || min_gap < 0) {
    ts_set_error("%s: top_k %d outside [1, %d] or min_gap %lld < 0", fn, top_k, TSLAM_PLACE_MAX_TOP_K, (long long)min_gap);
    return TSLAM_E_INVALID;
  }
  if (!sc || !ring || !bev || !n_points || !ids || !queries || !info6 || !dist3) {
    ts_set_error("%s: NULL array", fn);
    return TSLAM_E_INVALID;
  }
  for (int i = 0; i < n_q; i++) {
    if (queries[i] < 0 || queries[i] >= n_db) {
      ts_set_error("%s: query %d: entry %d out of range", fn, i, queries[i]);
      return TSLAM_E_INVALID;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int P = n_q * top_k;
  const size_t qb = ((size_t)n_q * 4 + 255) & ~(size_t)255, kb = ((size_t)P * 3 * 8 + 255) & ~(size_t)255;
  char* w = nullptr;
  TS_CUDA(cudaMallocAsync((void**)&w, qb + kb + (size_t)P * 3 * 8, st));
  int* d_q = (int*)w;
  unsigned long long* keys = (unsigned long long*)(w + qb);
  int* pop = (int*)(w + qb + kb);
  PlYaw yt;
  for (int h = 0; h < 2 * PL_S; h++) {
    const double a = 2.0 * M_PI * (double)h / (double)(2 * PL_S);
    yt.c[h] = (float)std::cos(a);
    yt.s[h] = (float)std::sin(a);
  }
  cudaError_t e = cudaMemcpyAsync(d_q, queries, (size_t)n_q * 4, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    k_pl_shortlist<<<n_q, PL_MAX_N, 0, st>>>(n_db, ring, (const long long*)n_points, (const long long*)ids, d_q, top_k, (long long)min_gap,
                                              (long long)min_points, info6, dist3);
    k_pl_shift<<<(P + PL_SW - 1) / PL_SW, PL_SW * 32, 0, st>>>(sc, d_q, top_k, P, info6, dist3);
    k_pl_bev<<<3 * P, 256, 0, st>>>(bev, d_q, top_k, info6, yt, keys, pop);
    k_pl_pick<<<(P + 255) / 256, 256, 0, st>>>(P, keys, pop, info6, dist3);
    e = cudaGetLastError();
  }
  const cudaError_t f = cudaFreeAsync(w, st);
  if (e == cudaSuccess) e = f;
  if (e != cudaSuccess) {
    ts_set_error("%s: %s", fn, cudaGetErrorString(e));
    return TSLAM_E_CUDA;
  }
  return TSLAM_OK;
}
