// Sizing of the packed fields of the per-frame bucket grid (tslam_integrate.cu).  Host-only C++ without CUDA, so that the
// bounds can be unit-tested without a GPU.
#pragma once
#include <cmath>
#include <cstdint>

#define TS_BK_SLOT_FIELD 25      // bits of an index entry left beside the 39-bit key: slot + 1 and the launch epoch
#define TS_BK_MIN_EPOCH_BITS 4   // fewer epoch bits than this: clearing mode (no epoch, the consumer zeroes every entry)
#define BK_MAX_SLOTS ((1u << 25) - 2u)  // record slots the slot + 1 field can name when it takes all TS_BK_SLOT_FIELD bits

static inline int ts_bit_length(uint64_t x) {
  int b = 0;
  while (x) { b++; x >>= 1; }
  return b;
}

// Width of the index entry's slot + 1 field.  A depth frame's slots are < bucket_cap, a point cloud's are < its point
// count <= max_points.  Returns TS_BK_SLOT_FIELD (clearing mode) when the epoch would get fewer than
// TS_BK_MIN_EPOCH_BITS.
static inline int ts_bucket_slot_bits(uint32_t bucket_cap, uint32_t max_points) {
  const int d = ts_bit_length(bucket_cap), p = ts_bit_length(max_points);
  const int s = d > p ? d : p;
  return TS_BK_SLOT_FIELD - s < TS_BK_MIN_EPOCH_BITS ? TS_BK_SLOT_FIELD : s;
}

// A bucket record keeps its point count and its depth sum in one 64-bit word, cnt << shift | sum(d), d in 2^-20 m fixed
// point.  In a launch where one bucket can collect at most n points, each with 0 <= d <= dmax_m metres, the count needs
// bit_length(n) bits and the sum stays below n * q, q the largest fixed-point depth.  Returns the shift that gives the
// count exactly the bits it needs, or -1 when the sum could then reach into the count: such a launch keeps the counts in
// a plane of their own and the word holds the depth sum alone.
static inline int ts_bucket_cnt_shift(uint64_t n, double dmax_m) {
  if (n == 0) n = 1;
  const int shift = 64 - ts_bit_length(n);
  const double qd = std::ceil(dmax_m * 1048576.0) + 1.0;  // >= round(d * 2^20) for every d <= dmax_m
  if (!(qd >= 0.0) || qd >= 18446744073709551616.0) return -1;
  const unsigned __int128 sum = (unsigned __int128)n * (unsigned __int128)(uint64_t)qd;
  return sum < ((unsigned __int128)1 << shift) ? shift : -1;
}
