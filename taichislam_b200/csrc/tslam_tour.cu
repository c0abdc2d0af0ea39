// libtslam.so - open exploration tours over a travel-cost matrix (DESIGN.md section 7, "Exploration tours").
//
// tslam_tour_open orders the goals of an f32 cost matrix C[n,n] (node 0 the start, nodes 1..n-1 the goals) into an open
// tour from node 0: R independent restarts of a best-improvement 2-opt / Or-opt local search, one CTA per restart.
//
// Costs are exact.  Every finite off-diagonal entry is an integer multiple q of the unit U = 2^(e_lo - 23), e_lo the least
// floor(log2 x) over the positive finite off-diagonal entries, and q < 2^52 once the range e_hi - e_lo is at most 28.  A
// leg weighs (inf, q) = (1, 0) for +inf and (0, q) otherwise; tour costs are int32 / int64 sums compared
// lexicographically.  So each restart's sequence of moves is fixed by the contract, not by the order of any sum, and
// tests/tour_reference.py restates it in numpy bit for bit.
//
// Per restart, in shared memory: the tour t[0..m] with a sentinel node n at t[m+1] (legs into it weigh 0, which makes
// "after the last node" an ordinary position), a second buffer for the applied move, and the forward and reverse prefix
// sums F[k] = sum_{p<k} w(t[p], t[p+1]), Rv[k] = sum_{p<k} w(t[p+1], t[p]).  With them a 2-opt delta needs two matrix
// reads and an Or-opt delta three.  C itself is staged in shared memory when it fits next to them, else read through L2.
#include <algorithm>
#include <climits>
#include "tslam_internal.cuh"

#define TOUR_THREADS 256
#define TOUR_WARPS (TOUR_THREADS / 32)
#define TOUR_MAX_N TSLAM_OCTO_TRAVEL_MAX_STARTS
#define TOUR_MAX_RESTARTS 4096
#define TOUR_MAX_RANGE 28
#define TOUR_NO_MOVE INT_MAX

// a leg weight or a sum of them: infinite legs, then q in units U
struct TW {
  int inf;
  long long q;
};
__device__ __forceinline__ TW operator+(TW a, TW b) { return {a.inf + b.inf, a.q + b.q}; }
__device__ __forceinline__ TW operator-(TW a, TW b) { return {a.inf - b.inf, a.q - b.q}; }
__device__ __forceinline__ TW shfl_up(TW v, int d) { return {__shfl_up_sync(~0u, v.inf, d), __shfl_up_sync(~0u, v.q, d)}; }

// the forward and the reverse leg of one tour position, scanned together
struct TW2 {
  TW f, r;
};
__device__ __forceinline__ TW2 operator+(TW2 a, TW2 b) { return {a.f + b.f, a.r + b.r}; }
__device__ __forceinline__ TW2 operator-(TW2 a, TW2 b) { return {a.f - b.f, a.r - b.r}; }
__device__ __forceinline__ TW2 shfl_up(TW2 v, int d) { return {shfl_up(v.f, d), shfl_up(v.r, d)}; }
__device__ __forceinline__ int shfl_up(int v, int d) { return __shfl_up_sync(~0u, v, d); }

// (cost delta or cost, move key or restart) ordered lexicographically; keys are unique, so the order is total
struct TBest {
  int inf;
  long long q;
  int key;
};
__device__ __forceinline__ bool tb_less(const TBest& a, const TBest& b) {
  return a.inf != b.inf ? a.inf < b.inf : a.q != b.q ? a.q < b.q : a.key < b.key;
}

// The weight of entry x of a validated matrix: x = (2^23 + frac) * 2^(e - 23) with e = floor(log2 x) in [e_lo, e_lo + 28],
// so q = x / 2^(e_lo - 23) = (2^23 + frac) << (e - e_lo), exactly, in integer arithmetic.
__device__ __forceinline__ TW tour_w(float x, int e_lo) {
  const unsigned b = __float_as_uint(x);
  if (b == 0x7f800000u) return {1, 0};
  if ((b & 0x7fffffffu) == 0u) return {0, 0};
  return {0, (long long)((b & 0x7fffffu) | 0x800000u) << ((int)(b >> 23) - 127 - e_lo)};
}

// exclusive prefix over the CTA in thread order; every thread calls it
template <class T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* wsum) {
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  T inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const T o = shfl_up(inc, d);
    if (lane >= d) inc = inc + o;
  }
  if (lane == 31) wsum[wp] = inc;
  __syncthreads();
  T ex = inc - v;
  for (int w = 0; w < wp; w++) ex = ex + wsum[w];
  __syncthreads();
  return ex;
}

// the least TBest of the CTA, returned to every thread; sh holds blockDim.x / 32 + 1 entries
__device__ __forceinline__ TBest block_min(TBest v, TBest* sh) {
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) {
    const TBest o{__shfl_down_sync(~0u, v.inf, d), __shfl_down_sync(~0u, v.q, d), __shfl_down_sync(~0u, v.key, d)};
    if (tb_less(o, v)) v = o;
  }
  const int nw = blockDim.x >> 5;
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    TBest b = sh[0];
    for (int w = 1; w < nw; w++)
      if (tb_less(sh[w], b)) b = sh[w];
    sh[nw] = b;
  }
  __syncthreads();
  return sh[nw];
}

__device__ __forceinline__ unsigned long long tour_mix64(unsigned long long z) {  // the SplitMix64 finaliser
  z ^= z >> 30;
  z *= 0xbf58476d1ce4e5b9ull;
  z ^= z >> 27;
  z *= 0x94d049bb133111ebull;
  z ^= z >> 31;
  return z;
}

// The validation and exponent pass.  words (pre-set to 0, INT_MAX, INT_MIN, 0): OR of refusal flags (1 NaN, 2 negative,
// 4 subnormal) over the off-diagonal entries, least and greatest floor(log2 x) of the positive finite ones, and m = the
// number of goals g >= 1 with C[0][g] finite.
__global__ void __launch_bounds__(256) k_tour_scan(int n, const float* __restrict__ C, int* words) {
  int flags = 0, lo = INT_MAX, hi = INT_MIN, kept = 0;
  const int nn = n * n;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < nn; k += gridDim.x * blockDim.x) {
    const int a = k / n, b = k - a * n;
    if (a == b) continue;
    const float x = C[k];
    const unsigned u = __float_as_uint(x), ex = (u >> 23) & 0xffu;
    if (x != x) flags |= 1;
    else if ((u >> 31) && (u & 0x7fffffffu)) flags |= 2;  // -0 is a zero
    else if (x > 0.0f && ex != 0xffu) {
      if (ex == 0u) flags |= 4;
      lo = min(lo, (int)ex - 127);
      hi = max(hi, (int)ex - 127);
    }
    if (a == 0 && ex != 0xffu) kept++;
  }
  flags = __reduce_or_sync(~0u, flags);
  lo = __reduce_min_sync(~0u, lo);
  hi = __reduce_max_sync(~0u, hi);
  kept = __reduce_add_sync(~0u, kept);
  if ((threadIdx.x & 31) == 0) {
    if (flags) atomicOr(&words[0], flags);
    if (lo != INT_MAX) { atomicMin(&words[1], lo); atomicMax(&words[2], hi); }
    if (kept) atomicAdd(&words[3], kept);
  }
}

// One restart per CTA (blockIdx.x = r).  Dynamic shared memory: F and Rv as (int32 inf, int64 q) arrays of m + 2, the
// tour and its move buffer as int32 of n + 2, then C when STAGE.
template <bool STAGE>
__global__ void __launch_bounds__(TOUR_THREADS, 4) k_tour_search(int n, const float* __restrict__ C, int m, int e_lo,
                                                              unsigned long long seed, int max_passes, int* tours,
                                                              long long* cost2, int* passes_out, unsigned char* converged) {
  extern __shared__ __align__(16) unsigned char tour_smem[];
  __shared__ TW2 wsum[TOUR_WARPS];
  __shared__ TBest red[TOUR_WARPS + 1];
  long long* Fq = reinterpret_cast<long long*>(tour_smem);
  long long* Rq = Fq + (n + 2);
  int* Fi = reinterpret_cast<int*>(Rq + (n + 2));
  int* Ri = Fi + (n + 2);
  int* t = Ri + (n + 2);
  int* nt = t + (n + 2);
  const float* Cm = C;
  if constexpr (STAGE) {
    float* Cs = reinterpret_cast<float*>(nt + (n + 2));
    for (int k = threadIdx.x; k < n * n; k += TOUR_THREADS) Cs[k] = C[k];
    Cm = Cs;
    __syncthreads();
  }
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wp = tid >> 5;
  // w(a, b) for a != b; legs into the sentinel n weigh nothing
  auto w = [&](int a, int b) -> TW { return b == n ? TW{0, 0} : tour_w(Cm[a * n + b], e_lo); };

  // the kept goals in ascending order, into nt[0..m-1]: a CTA-wide compaction of chunks of consecutive goals
  {
    const int ch = (n + TOUR_THREADS - 1) / TOUR_THREADS, g0 = 1 + tid * ch;
    int cnt = 0;
    for (int g = g0; g < min(g0 + ch, n); g++) cnt += isinf(Cm[g]) ? 0 : 1;
    int o = block_exclusive_scan(cnt, reinterpret_cast<int*>(wsum));
    for (int g = g0; g < min(g0 + ch, n); g++)
      if (!isinf(Cm[g])) nt[o++] = g;
  }
  if (tid == 0) {
    t[0] = 0;
    t[m + 1] = nt[m + 1] = n;
  }
  __syncthreads();
  if (r == 0) {
    // nearest neighbour: step s takes the least (w(cur, g), g) among the goals still in nt[0..left-1]
    int cur = 0;
    for (int s = 1, left = m; s <= m; s++, left--) {
      TBest b{INT_MAX, LLONG_MAX, TOUR_NO_MOVE};
      for (int k = tid; k < left; k += TOUR_THREADS) {
        const TW x = w(cur, nt[k]);
        const TBest c{x.inf, x.q, (nt[k] << 10) | k};  // node first: ties go to the smaller node
        if (tb_less(c, b)) b = c;
      }
      b = block_min(b, red);
      cur = b.key >> 10;
      if (tid == 0) {
        t[s] = cur;
        nt[b.key & 1023] = nt[left - 1];
      }
      __syncthreads();
    }
  } else if (tid == 0) {
    // Fisher-Yates over the ascending kept goals
    for (int k = 0; k < m; k++) t[1 + k] = nt[k];
    for (int i = m - 1; i >= 1; i--) {
      const unsigned long long z = tour_mix64(seed ^ ((unsigned long long)r << 32) ^ (unsigned long long)i);
      const int j = (int)(z % (unsigned long long)(i + 1));
      const int x = t[1 + i];
      t[1 + i] = t[1 + j];
      t[1 + j] = x;
    }
  }
  __syncthreads();

  int passes = 0;
  bool done = false;
  while (true) {
    {  // F and Rv of the current tour: thread k scans positions [k * ch, (k + 1) * ch) of the m legs
      const int ch = (m + TOUR_THREADS - 1) / TOUR_THREADS, p0 = tid * ch, p1 = min(p0 + ch, m);
      TW2 s{{0, 0}, {0, 0}};
      for (int p = p0; p < p1; p++) s = s + TW2{w(t[p], t[p + 1]), w(t[p + 1], t[p])};
      TW2 o = block_exclusive_scan(s, wsum);
      if (tid == 0) { Fi[0] = Ri[0] = 0; Fq[0] = Rq[0] = 0; }
      for (int p = p0; p < p1; p++) {
        o = o + TW2{w(t[p], t[p + 1]), w(t[p + 1], t[p])};
        Fi[p + 1] = o.f.inf; Fq[p + 1] = o.f.q;
        Ri[p + 1] = o.r.inf; Rq[p + 1] = o.r.q;
      }
      if (p1 == m && p0 < p1) { Fi[m + 1] = o.f.inf; Fq[m + 1] = o.f.q; }  // the leg into the sentinel weighs 0
      if (m == 0 && tid == 0) { Fi[1] = 0; Fq[1] = 0; }
      __syncthreads();
    }
    // Every move, each thread keeping its least delta.  A thread meets its moves in increasing key order, so a strict
    // comparison keeps the first of equal deltas.  2-opt: warp per i, lanes over j.  Key i << 10 | j.
    TBest b{INT_MAX, LLONG_MAX, TOUR_NO_MOVE};
    for (int i = 1 + wp; i < m; i += TOUR_WARPS) {
      const int a = t[i - 1], c = t[i];
      const TW base = TW{Fi[i - 1], Fq[i - 1]} - TW{Ri[i], Rq[i]};
      for (int j = i + 1 + lane; j <= m; j += 32) {
        const TW d = base + w(a, t[j]) + w(c, t[j + 1]) + TW{Ri[j], Rq[j]} - TW{Fi[j + 1], Fq[j + 1]};
        if (d.inf < b.inf || (d.inf == b.inf && d.q < b.q)) b = TBest{d.inf, d.q, (i << 10) | j};
      }
    }
    // Or-opt: warp per (L, i), lanes over p.  Key L << 20 | i << 10 | p, above every 2-opt key.
    for (int row = wp; row < 3 * m; row += TOUR_WARPS) {
      const int L = row / m + 1, i = row - (L - 1) * m + 1, e = i + L - 1;
      if (e > m) continue;
      const int s0 = t[i], s1 = t[e];
      const TW cut = w(t[i - 1], t[e + 1]) - (TW{Fi[e + 1], Fq[e + 1]} - TW{Fi[e], Fq[e]}) -
                     (TW{Fi[i], Fq[i]} - TW{Fi[i - 1], Fq[i - 1]});
      for (int p = lane; p <= m; p += 32) {
        if (p >= i - 1 && p <= e) continue;
        const TW d = cut + w(t[p], s0) + w(s1, t[p + 1]) - (TW{Fi[p + 1], Fq[p + 1]} - TW{Fi[p], Fq[p]});
        if (d.inf < b.inf || (d.inf == b.inf && d.q < b.q)) b = TBest{d.inf, d.q, (L << 20) | (i << 10) | p};
      }
    }
    b = block_min(b, red);
    if (b.key == TOUR_NO_MOVE || !(b.inf < 0 || (b.inf == 0 && b.q < 0))) {
      done = true;
      break;
    }
    if (passes == max_passes) break;
    // apply: nt[k] = t[src(k)], then swap the buffers
    const int L = b.key >> 20, i = (b.key >> 10) & 1023, jp = b.key & 1023;
    for (int k = tid; k <= m; k += TOUR_THREADS) {
      int s = k;
      if (L == 0) {
        if (k >= i && k <= jp) s = i + jp - k;
      } else if (jp < i) {  // the segment moves back to follow t[jp]
        if (k > jp && k <= jp + L) s = i + k - jp - 1;
        else if (k > jp + L && k <= i + L - 1) s = k - L;
      } else {  // ... or forward to follow t[jp]
        if (k >= i && k <= jp - L) s = k + L;
        else if (k > jp - L && k <= jp) s = i + k - (jp - L + 1);
      }
      nt[k] = t[s];
    }
    __syncthreads();
    int* x = t;
    t = nt;
    nt = x;
    passes++;
  }

  for (int k = tid; k < n; k += TOUR_THREADS) tours[(size_t)r * n + k] = k <= m ? t[k] : -1;
  if (tid == 0) {
    cost2[2 * (size_t)r] = Fi[m];
    cost2[2 * (size_t)r + 1] = Fq[m];
    passes_out[r] = passes;
    converged[r] = done ? 1 : 0;
  }
}

// the restart with the least cost, ties to the smallest r
__global__ void __launch_bounds__(1024) k_tour_pick(int R, const long long* cost2, int* best) {
  __shared__ TBest red[33];
  TBest b{INT_MAX, LLONG_MAX, INT_MAX};
  for (int r = threadIdx.x; r < R; r += blockDim.x) {
    const TBest c{(int)cost2[2 * r], cost2[2 * r + 1], r};
    if (tb_less(c, b)) b = c;
  }
  b = block_min(b, red);
  if (threadIdx.x == 0) best[0] = b.key;
}

extern "C" int tslam_tour_open(int32_t n, const float* cost, int32_t restarts, uint64_t seed, int32_t max_passes, int32_t* tours,
                               int64_t* cost2, int32_t* passes, uint8_t* converged, int32_t* best, int32_t* info2, void* stream) {
  const char* what = "tslam_tour_open";
  if (!cost || !tours || !cost2 || !passes || !converged || !best || !info2) {
    ts_set_error("%s: NULL array", what);
    return TSLAM_E_INVALID;
  }
  if (n < 1 || n > TOUR_MAX_N) {
    ts_set_error("%s: n must be in [1, %d] (got %d)", what, TOUR_MAX_N, n);
    return TSLAM_E_INVALID;
  }
  if (restarts < 1 || restarts > TOUR_MAX_RESTARTS) {
    ts_set_error("%s: restarts must be in [1, %d] (got %d)", what, TOUR_MAX_RESTARTS, restarts);
    return TSLAM_E_INVALID;
  }
  if (max_passes < 0) {
    ts_set_error("%s: max_passes must be >= 0 (got %d)", what, max_passes);
    return TSLAM_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  // the scan's four words live in the first 16 bytes of cost2 (R >= 1 rows of two int64) until the search writes it
  int* words = reinterpret_cast<int*>(cost2);
  int h[4] = {0, INT_MAX, INT_MIN, 0};
  TS_CUDA(cudaMemcpyAsync(words, h, sizeof(h), cudaMemcpyHostToDevice, st));
  k_tour_scan<<<std::min((n * n + 255) / 256, 512), 256, 0, st>>>(n, cost, words);
  TS_CUDA(cudaGetLastError());
  TS_CUDA(cudaMemcpyAsync(h, words, sizeof(h), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (h[0]) {
    ts_set_error("%s: the matrix holds %s off the diagonal", what,
                 (h[0] & 1) ? "a NaN" : (h[0] & 2) ? "a negative value" : "a subnormal value");
    return TSLAM_E_INVALID;
  }
  const int e_lo = h[1] == INT_MAX ? 0 : h[1], e_hi = h[1] == INT_MAX ? 0 : h[2];
  if (e_hi - e_lo > TOUR_MAX_RANGE) {
    ts_set_error("%s: the positive finite entries span 2^%d .. 2^%d, a range above 2^%d", what, e_lo, e_hi + 1, TOUR_MAX_RANGE);
    return TSLAM_E_INVALID;
  }
  const int m = h[3];
  info2[0] = m;
  info2[1] = e_lo - 23;
  // stage C in shared memory when it fits beside the tour arrays
  int dev = 0, optin = 0;
  TS_CUDA(cudaGetDevice(&dev));
  TS_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  cudaFuncAttributes fa;
  TS_CUDA(cudaFuncGetAttributes(&fa, k_tour_search<true>));
  const size_t tour_bytes = (size_t)(n + 2) * 32, c_bytes = (size_t)n * n * 4;  // F, Rv: 12 B per entry; t, nt: 4 B
  const bool stage = tour_bytes + c_bytes + fa.sharedSizeBytes <= (size_t)optin;
  const size_t smem = tour_bytes + (stage ? c_bytes : 0);
  if (stage) {
    TS_CUDA(cudaFuncSetAttribute(k_tour_search<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_tour_search<true><<<restarts, TOUR_THREADS, smem, st>>>(n, cost, m, e_lo, seed, max_passes, tours, (long long*)cost2,
                                                              passes, converged);
  } else {
    TS_CUDA(cudaFuncSetAttribute(k_tour_search<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_tour_search<false><<<restarts, TOUR_THREADS, smem, st>>>(n, cost, m, e_lo, seed, max_passes, tours, (long long*)cost2,
                                                               passes, converged);
  }
  TS_CUDA(cudaGetLastError());
  k_tour_pick<<<1, 1024, 0, st>>>(restarts, (const long long*)cost2, best);
  TS_CUDA(cudaGetLastError());
  return TSLAM_OK;
}
