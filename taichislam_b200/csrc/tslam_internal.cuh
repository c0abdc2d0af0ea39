// Internal structures of libtslam.so (sm_90a).  Not part of the ABI.
//
// HBM layout of a TSDF map (replaces Taichi's pointer->dense SNode tree,
// dense_tsdf.py:108-118):
//   * one open-addressing hash table  slot -> (key40 | block24)   8 B/slot
//   * a pool of 16^3-voxel blocks stored as per-field PLANES (SoA across the pool,
//     4096 consecutive voxels of one block are contiguous in every plane):
//         acc  float2[4096]  pending (sum w*d, sum w) of not-yet-committed frames
//         tw   float2[4096]  committed (TSDF, W_TSDF)   (f16 x2 in the reference)
//         obs  u8[4096]      TSDF_observed
//         occ  i8[4096]      occupy
//     A voxel update of the ray-march kernel is ONE 8-byte vector reduction
//     (REDG.E.ADD.F32x2) into `acc`; whole blocks are streamed by the commit /
//     marching-cubes / export kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <utility>
#include <vector>
#include "../../include/tslam.h"

#define TS_B 16
#define TS_B3 4096
#define TS_BSHIFT 4
#define TS_BMASK 15

// packed hash word:  [63:24] key (s:10 | bx:10 | by:10 | bz:10), [23:0] block index
#define TS_EMPTY 0xFFFFFFFFFFFFFFFFull
#define TS_IDX_MASK 0xFFFFFFull
#define TS_IDX_PENDING 0xFFFFFEull
#define TS_IDX_OVERFLOW 0xFFFFFDull
#define TS_MAX_BLOCKS 0xFFFFF0

#define TS_ERR_POOL_FULL 1
#define TS_ERR_TABLE_FULL 2
#define TS_ERR_RAYLIST_FULL 4
#define TS_ERR_BUCKET_RANGE 8   // a point further than 4095 voxels from the sensor origin: beyond the bucket index's key range
#define TS_PROF_RING 512
// Kernel stamps of a profiled integrate launch (tslam_tsdf_kernel_ms2): one row of TS_PROF_WORDS %globaltimer words per
// launch, [2k] = entry of CTA 0 of kernel k, [2k + 1] = exit of its last CTA (atomicMax: the timer only grows, so a
// row reused from 512 launches earlier needs no clearing).  The row travels to the kernels by value; with profiling
// off they get a null pointer and stamp nothing.
#define TS_PROF_WORDS 16
enum { TS_K_BUCKET = 0, TS_K_COUNT, TS_K_CLASS_SCAN, TS_K_SCATTER, TS_K_MARCH, TS_K_COLLECT, TS_K_COMMIT, TS_K_N };
__device__ __forceinline__ unsigned long long ts_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// at kernel entry, by every thread: CTA 0 (dispatched first) stores the start
__device__ __forceinline__ void ts_stamp_begin(unsigned long long* prof, int k) {
  if (prof && (blockIdx.x | blockIdx.y | blockIdx.z | threadIdx.x) == 0) prof[2 * k] = ts_globaltimer();
}
// by one thread of a CTA once the CTA's work is done: raises the kernel's end
__device__ __forceinline__ void ts_stamp_end_thread(unsigned long long* prof, int k) {
  if (prof) asm volatile("red.relaxed.gpu.global.max.u64 [%0], %1;" ::"l"(prof + 2 * k + 1), "l"(ts_globaltimer()) : "memory");
}
// at kernel exit, by every thread of the CTA (a barrier when profiling: the CTA's last thread is done)
__device__ __forceinline__ void ts_stamp_end(unsigned long long* prof, int k) {
  if (!prof) return;
  __syncthreads();
  if (threadIdx.x == 0) ts_stamp_end_thread(prof, k);
}

struct TsGrid {
  unsigned long long* table;  // hash words
  uint32_t table_mask;        // capacity-1 (power of two)
  int max_blocks;
  int* n_blocks;              // device allocation counter
  unsigned long long* block_key;  // [max_blocks] reverse map (key40)
  float2* acc;                // [max_blocks*4096]
  float2* tw;                 // [max_blocks*4096]
  uint8_t* obs;               // [max_blocks*4096]
  int8_t* occ;                // [max_blocks*4096]
  unsigned long long* cword;  // [max_blocks*4096] texture: winning colour word per voxel (null unless texture_enabled)
  float4* col;                // [max_blocks*4096] texture: committed colour rgb (+pad)
  uint8_t* ghost;             // [max_blocks] 1 = halo copy of a block owned by another rank (multi-GPU tiling)
  float* esdf;                // [max_blocks*4096] (allocated lazily by the ESDF path)
  int* esdf_dirty;            // [max_blocks] block committed since the last ESDF update (seeds the incremental wave)
  int* dirty_flag;            // [max_blocks]
  int* dirty_list;            // [max_blocks]
  int* n_dirty;
  int* err;                   // device error flags
  int hN, hNz, N, Nz;         // bounds: i in [-hN, N-hN)
};

__host__ __device__ __forceinline__ unsigned long long ts_pack_key(int s, int bx, int by, int bz) {
  return ((unsigned long long)(s & 1023) << 30) | ((unsigned long long)((bx + 512) & 1023) << 20) |
         ((unsigned long long)((by + 512) & 1023) << 10) | (unsigned long long)((bz + 512) & 1023);
}
__host__ __device__ __forceinline__ void ts_unpack_key(unsigned long long k, int& s, int& bx, int& by, int& bz) {
  s = (int)((k >> 30) & 1023);
  bx = (int)((k >> 20) & 1023) - 512;
  by = (int)((k >> 10) & 1023) - 512;
  bz = (int)(k & 1023) - 512;
}
__device__ __forceinline__ uint32_t ts_hash(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return (uint32_t)k;
}
template <class G>
__device__ __forceinline__ bool ts_in_bounds(const G& g, int i, int j, int k) {
  return i >= -g.hN && i < g.N - g.hN && j >= -g.hN && j < g.N - g.hN && k >= -g.hNz && k < g.Nz - g.hNz;
}
__device__ __forceinline__ int ts_voxel_off(int i, int j, int k) {
  return (((i & TS_BMASK) << TS_BSHIFT) | (j & TS_BMASK)) << TS_BSHIFT | (k & TS_BMASK);
}
__device__ __forceinline__ unsigned long long ts_ld_volatile(const unsigned long long* p) {
  return *(const volatile unsigned long long*)p;
}

// read-only lookup: block index or -1   (G = TsGrid or OcGrid)
template <class G>
__device__ __forceinline__ int ts_find(const G& g, unsigned long long key) {
  uint32_t slot = ts_hash(key) & g.table_mask;
  for (uint32_t probe = 0; probe <= g.table_mask; ++probe) {
    unsigned long long cur = ts_ld_volatile(&g.table[slot]);
    if (cur == TS_EMPTY) return -1;
    if ((cur >> 24) == key) {
      unsigned idx = (unsigned)(cur & TS_IDX_MASK);
      return (idx >= TS_IDX_OVERFLOW) ? -1 : (int)idx;
    }
    slot = (slot + 1) & g.table_mask;
  }
  return -1;
}

// lookup, activating a zero-filled block on miss (Taichi "write activates").
// Returns -1 when the pool is exhausted (error flag raised, sample dropped).
template <class G>
__device__ __forceinline__ int ts_get_or_alloc(const G& g, unsigned long long key) {
  uint32_t slot = ts_hash(key) & g.table_mask;
  for (uint32_t probe = 0; probe <= g.table_mask; ++probe) {
    unsigned long long cur = ts_ld_volatile(&g.table[slot]);
    if (cur == TS_EMPTY) {
      unsigned long long prev = atomicCAS(&g.table[slot], TS_EMPTY, (key << 24) | TS_IDX_PENDING);
      if (prev == TS_EMPTY) {
        int idx = atomicAdd(g.n_blocks, 1);
        unsigned long long word;
        if (idx >= g.max_blocks) {
          atomicSub(g.n_blocks, 1);
          atomicOr(g.err, TS_ERR_POOL_FULL);
          word = (key << 24) | TS_IDX_OVERFLOW;
          idx = -1;
        } else {
          g.block_key[idx] = key;
          word = (key << 24) | (unsigned long long)idx;
        }
        __threadfence();
        atomicExch(&g.table[slot], word);
        return idx;
      }
      cur = prev;
    }
    if ((cur >> 24) == key) {
      while ((cur & TS_IDX_MASK) == TS_IDX_PENDING) {
        __nanosleep(32);
        cur = ts_ld_volatile(&g.table[slot]);
      }
      unsigned idx = (unsigned)(cur & TS_IDX_MASK);
      return (idx >= TS_IDX_OVERFLOW) ? -1 : (int)idx;
    }
    slot = (slot + 1) & g.table_mask;
  }
  atomicOr(g.err, TS_ERR_TABLE_FULL);
  return -1;
}

// Insert `key` at pool slot `slot` into a table that does not hold it: the rebuild of the table after a compaction of
// the pool (tslam_reclaim.cu), between launches, so ts_get_or_alloc_cached's L1 argument still holds.  False when the
// table is full.
template <class G>
__device__ __forceinline__ bool ts_insert_slot(const G& g, unsigned long long key, int slot) {
  uint32_t h = ts_hash(key) & g.table_mask;
  for (uint32_t probe = 0; probe <= g.table_mask; ++probe) {
    if (atomicCAS(&g.table[h], TS_EMPTY, (key << 24) | (unsigned long long)slot) == TS_EMPTY) return true;
    h = (h + 1) & g.table_mask;
  }
  return false;
}

// Touched blocks are flagged with a fire-and-forget store (no load on the ray-march critical
// path); k_collect_dirty compacts the flags into dirty_list before a commit.
__device__ __forceinline__ void ts_mark_dirty(const TsGrid& g, int blk) { g.dirty_flag[blk] = 1; }

// Fast lookup for the hot loops: first probe through L1 (plain cached load).  Entries are only
// ever inserted while kernels run (the table is cleared between launches, where L1 is
// invalidated), so a cached hit is always valid; anything else falls back to the coherent path.
template <class G>
__device__ __forceinline__ int ts_get_or_alloc_cached(const G& g, unsigned long long key) {
  const uint32_t slot = ts_hash(key) & g.table_mask;
  const unsigned long long cur = __ldca(&g.table[slot]);
  if ((cur >> 24) == key) {
    const unsigned idx = (unsigned)(cur & TS_IDX_MASK);
    if (idx < TS_IDX_OVERFLOW) return (int)idx;
  }
  return ts_get_or_alloc(g, key);
}

// ---------------------------------------------------------------------------
// arithmetic helpers shared by the integrate kernels (tslam_integrate.cu, tslam_march.cu)
// ---------------------------------------------------------------------------
#define WMAX 1000.0f          // dense_tsdf.py:8
#define FIXQ 1048576.0f       // 2^20: fixed-point quantum of the per-frame bucket sums
#define FIXQ_D 1048576.0

// ---------------------------------------------------------------------------
// small device helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ int iroundf(float x) { return (int)roundf(x); }  // ti.round(x, i32) mapping_common.py:263-266
__device__ __forceinline__ float sgnf(float v) { return (float)((0.0f < v) - (v < 0.0f)); }  // mapping_common.py:5-7

// x / vs, correctly rounded, without the slow-path check of the generic IEEE division: rvs = RN(1/vs) comes
// from the host; q1 = fma(fma(-q0, vs, x), rvs, q0) is the correctly rounded quotient (Markstein) for the
// operand ranges that occur here (|x| < 1e4 m, vs ~ 1e-2..1 m: no overflow / underflow / denormals).
__device__ __forceinline__ float div_vs(float x, float vs, float rvs) {
  const float q0 = __fmul_rn(x, rvs);
  const float e = __fmaf_rn(-q0, vs, x);
  return __fmaf_rn(e, rvs, q0);
}

// warp-aggregated append to an int32 row counter: the row of this lane, or -1 when it does not want one
__device__ __forceinline__ int warp_append_i32(bool want, int* counter) {
  const unsigned m = __ballot_sync(0xffffffffu, want);
  if (!m) return -1;
  const int lane = threadIdx.x & 31;
  const int leader = __ffs(m) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(counter, __popc(m));
  base = __shfl_sync(0xffffffffu, base, leader);
  return want ? base + __popc(m & ((1u << lane) - 1)) : -1;
}
// the same on an unsigned 64-bit counter (the count-then-fill gathers)
__device__ __forceinline__ long long warp_append_u64(bool want, unsigned long long* counter) {
  const unsigned m = __ballot_sync(0xffffffffu, want);
  if (!m) return -1;
  const int lane = threadIdx.x & 31;
  const int leader = __ffs(m) - 1;
  unsigned long long base = 0;
  if (lane == leader) base = atomicAdd(counter, (unsigned long long)__popc(m));
  base = __shfl_sync(0xffffffffu, base, leader);
  return want ? (long long)(base + __popc(m & ((1u << lane) - 1))) : -1;
}

// Low interpolation corner of an ESDF query point (k_esdf_query, k_octo_esdf_query, and k_owner_points which routes the
// points of a tiled map to the rank that answers them): u = x / vs per axis, correctly rounded, c = floor(u).  False
// when a coordinate is not finite or the corner lies outside the volume; NaN and +-inf fail the range test, so no
// out-of-range value reaches the float -> int conversion.  G = TsGrid or OcGrid.
template <class G>
__device__ __forceinline__ bool esq_low_corner(const G& g, float vs, const float* p, float u[3], int c[3]) {
  u[0] = __fdiv_rn(p[0], vs); u[1] = __fdiv_rn(p[1], vs); u[2] = __fdiv_rn(p[2], vs);
  const bool ok = u[0] >= (float)(-g.hN) && u[0] < (float)(g.N - g.hN) && u[1] >= (float)(-g.hN) && u[1] < (float)(g.N - g.hN) &&
                  u[2] >= (float)(-g.hNz) && u[2] < (float)(g.Nz - g.hNz);
  if (ok) { c[0] = (int)floorf(u[0]); c[1] = (int)floorf(u[1]); c[2] = (int)floorf(u[2]); }
  return ok;
}

// Cell of a planner-query point (sxyz_to_ijk, mapping_common.py:257-261): c = (int)roundf(x / vs) per axis, and whether
// it lies in the volume.  The probe of the planner queries (tslam_query.cu), the tiled ray march and the routing of
// point queries (k_tsdf_raycast_tiled, k_owner_cells) share this one expression, so a point is routed to the rank that
// owns the cell the probe reads.  A NaN coordinate converts to index 0 and +-inf saturates (out of the volume), in all
// of them alike.
__device__ __forceinline__ bool ts_query_cell(const TsGrid& g, float x, float y, float z, float vs, int c[3]) {
  c[0] = (int)roundf(x / vs); c[1] = (int)roundf(y / vs); c[2] = (int)roundf(z / vs);
  return ts_in_bounds(g, c[0], c[1], c[2]);
}

// BaseMap.raycast (mapping_common.py:165-178) marches sample j = 0 .. raycast_steps - 1 of a ray; sample j depends on
// (pos, dir, j) alone.  k_raycast and k_tsdf_raycast_tiled both take their samples from here, so a tiled ray that
// continues at sample j on another rank visits the same points, bit for bit, as one uninterrupted march.
__device__ __forceinline__ int raycast_steps(float max_dist, float vs) { return (int)(max_dist / vs); }  // :167, range(float) truncates
__device__ __forceinline__ void raycast_sample(float3 pos, float3 dir, int j, float vs, float& x, float& y, float& z, float& len) {
  len = (float)j * vs;                                                             // :173
  x = dir.x * len + pos.x; y = dir.y * len + pos.y; z = dir.z * len + pos.z;     // :174
}

// TSDF and observed byte of in-volume cell c of submap s as the planner queries read them: a block that is absent reads
// (0, 0), i.e. occupied and unobserved, and so does a ghost block unless Ghosts.
template <bool Ghosts>
__device__ __forceinline__ void ts_query_read(const TsGrid& g, int s, const int c[3], float& t, int& o) {
  const int blk = ts_find(g, ts_pack_key(s, c[0] >> TS_BSHIFT, c[1] >> TS_BSHIFT, c[2] >> TS_BSHIFT));
  if (blk >= 0 && (Ghosts || !g.ghost[blk])) {
    const size_t off = (size_t)blk * TS_B3 + ts_voxel_off(c[0], c[1], c[2]);
    t = g.tw[off].x;
    o = g.obs[off];
  }
}

// (x, y, z) = R l + T of a submap pose (row-major R), summed as ((R0 lx + R1 ly) + R2 lz) + T0: the build has
// -fmad=false, so these are the bits of the reference's f32 expression (submap_i_j_k_to_xyz, mapping_common.py:229-232)
__device__ __forceinline__ void pose_apply(const float* R, const float* T, float lx, float ly, float lz, float& x, float& y, float& z) {
  x = ((R[0] * lx + R[1] * ly) + R[2] * lz) + T[0];
  y = ((R[3] * lx + R[4] * ly) + R[5] * lz) + T[1];
  z = ((R[6] * lx + R[7] * ly) + R[8] * lz) + T[2];
}

// position of voxel (i, j, k) of submap s as the exporters write it (tslam_tsdf.cu, tslam_esdf.cu)
__device__ __forceinline__ void voxel_xyz(const TsGrid& g, bool global_map, const float* pR, const float* pT, int s, int i, int j,
                                          int k, float vs, float& x, float& y, float& z) {
  const float lx = (float)i * vs, ly = (float)j * vs, lz = (float)k * vs;  // ijk_to_xyz mapping_common.py:221-223
  if (global_map) { x = lx; y = ly; z = lz; return; }                      // i_j_k_to_xyz
  pose_apply(pR + 9 * s, pT + 3 * s, lx, ly, lz, x, y, z);                 // submap_i_j_k_to_xyz :229-232
}

// Placement of one observed source voxel by the submap -> global fusions (k_fuse, k_fz_splat; dense_tsdf.py:293-303):
// (i, j, k) of submap pose (R, T) lands at g = pose_apply(i vs, j vs, k vs) / vs in the global grid, and splats into the
// 7 upper trilinear corners lo + (c >> 2 & 1, c >> 1 & 1, c & 1), c = 1 .. 7, of lo = floor(g) (c = 0 is skipped: the
// reference quirk :300) with weight wt.  Both fusions call these two, so they place every term alike.
struct TsSplatPos {
  float gx, gy, gz;
  int lo0, lo1, lo2;
};
// (lx, ly, lz) = (float)i * vs, ... are formed by the caller (the expression order of k_fuse's arguments is kept)
__device__ __forceinline__ TsSplatPos ts_splat_pos(const float* R, const float* T, float lx, float ly, float lz, float vs) {
  float x, y, z;
  pose_apply(R, T, lx, ly, lz, x, y, z);  // :293-294
  TsSplatPos p;
  p.gx = x / vs; p.gy = y / vs; p.gz = z / vs;
  p.lo0 = (int)floorf(p.gx); p.lo1 = (int)floorf(p.gy); p.lo2 = (int)floorf(p.gz);  // :296
  return p;
}
// corner c of p: its cell (ci, cj, ck), weight wt (:303), and whether it lies in the volume of `dst`
__device__ __forceinline__ bool ts_splat_corner(const TsGrid& dst, const TsSplatPos& p, int c, int& ci, int& cj, int& ck, float& wt) {
  ci = p.lo0 + ((c >> 2) & 1); cj = p.lo1 + ((c >> 1) & 1); ck = p.lo2 + (c & 1);
  wt = (1.0f - fabsf((float)ci - p.gx)) * (1.0f - fabsf((float)cj - p.gy)) * (1.0f - fabsf((float)ck - p.gz));
  return ts_in_bounds(dst, ci, cj, ck);
}

__device__ __forceinline__ void red_add_f32x2(float2* addr, float a, float b) {
  // one 8-byte vector reduction without return value: REDG.E.ADD.F32x2 (sm_90+).  Spelled in PTX because
  // atomicAdd(float2*) was lowered to ATOMG (response sector per update) inside the divergent march loop.
  asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

__device__ __forceinline__ void red_add_u64(unsigned long long* addr, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.add.u64 [%0], %1;" ::"l"(addr), "l"(v) : "memory");
}
__device__ __forceinline__ void red_add_u32(unsigned int* addr, unsigned int v) {
  asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}

// both marches: a ray whose weight is < 2^14 fixed-point units (relative rounding error > 3e-5) takes f32 reductions
#define MB_MIN_WQ 16384
#define RM_TAB 4096          // shared block-lookup table: 16^3 entries indexed by the low 4 bits of the block coords
// block lookup for the march loop: shared-memory table first (global loads queue behind the reduction traffic in
// the in-order L1TEX pipe: measured as the top stall), hash grid on a miss.
__device__ __forceinline__ int rm_lookup(const TsGrid& g, unsigned long long* tab, unsigned long long key, int bx, int by, int bz) {
  const int h = ((bx & 15) << 8) | ((by & 15) << 4) | (bz & 15);
  const unsigned long long w = tab[h];
  if ((w >> 24) == key) return (int)(w & TS_IDX_MASK);
  const int blk = ts_get_or_alloc_cached(g, key);
  if (blk >= 0) {
    ts_mark_dirty(g, blk);
    tab[h] = (key << 24) | (unsigned long long)blk;  // benign race: any writer stores a valid word
  }
  return blk;
}
// read-only form for a kernel that runs after an earlier kernel activated the blocks (the table does not change while
// it runs): pool index, -1 when the block is not in the grid, -2 when its activation failed (pool exhausted).
__device__ __forceinline__ int rm_find(const TsGrid& g, unsigned long long* tab, unsigned long long key, int bx, int by, int bz) {
  const int h = ((bx & 15) << 8) | ((by & 15) << 4) | (bz & 15);
  const unsigned long long w = tab[h];
  if ((w >> 24) == key) return (int)(w & TS_IDX_MASK);
  uint32_t slot = ts_hash(key) & g.table_mask;
  for (uint32_t probe = 0; probe <= g.table_mask; ++probe) {
    const unsigned long long cur = g.table[slot];
    if (cur == TS_EMPTY) return -1;
    if ((cur >> 24) == key) {
      const unsigned idx = (unsigned)(cur & TS_IDX_MASK);
      if (idx >= TS_IDX_OVERFLOW) return -2;
      tab[h] = cur;
      return (int)idx;
    }
    slot = (slot + 1) & g.table_mask;
  }
  return -1;
}


// ---------------------------------------------------------------------------
// per-frame parameters of one integrate launch, passed BY VALUE as a
// __grid_constant__ kernel parameter (no H2D copy, no lifetime hazards)
// ---------------------------------------------------------------------------
struct TsFrame {
  float R[9];
  float T[3];
  int submap;
  unsigned int seq;  // frame sequence number of the map (texture: later frames overwrite earlier colours)
};
struct TsBatch {
  TsFrame f[TSLAM_MAX_BATCH];  // 64 * 56 B = 3584 B
};

struct TsIntrin {
  float fx, fy, cx, cy;
  float dmin_mm, dmax_mm;  // f32(min_ray*1000), f32(max_ray*1000)
  float vs;
  float rvs;               // RN(1/vs), for the exact FMA division in the march loop
  float rfx, rfy;          // RN(1/fx), RN(1/fy): div_vs(t, fx, rfx) unprojects a pixel when fdiv is set
  int fdiv;                // div_vs is correctly rounded for every dividend with divisor fx and with fy (ts_fill_intrin)
  float max_steps;         // f32(max_ray_length / voxel_scale)
  float max_ray;           // f32(max_ray_length)
  int internal_voxels;
  int step;
  // texture (dense_tsdf.py:204-211, mapping_common.py:43-58)
  float fxc, fyc, cxc, cyc;
  int tex;         // texture_enabled
  int same_proj;   // color_same_proj
};

// The depth rule of every reader of depth frames (k_bucket_depth, tslam_tsdf_track_depth): a pixel of d mm is kept when
// d != 0 and min_ray <= d <= max_ray (dense_tsdf.py:196-199), and its camera-frame point (x, y, dep) is
// unproject_point_dep (mapping_common.py:31-41, dense_tsdf.py:201): dep = df / 1000, x = ((i - cx) dep) / fx,
// y = ((j - cy) dep) / fy, each quotient correctly rounded without IEEE division: div_vs gives df / 1000 for every
// uint16 df (tests/test_gpu_bucket_merge.py checks all of them), and t / fx and t / fy where ts_fill_intrin proved the
// form.
__device__ __forceinline__ bool ts_depth_kept(const TsIntrin& in, uint16_t d) {
  const float df = (float)d;
  return d != 0 && !(df > in.dmax_mm || df < in.dmin_mm);
}
__device__ __forceinline__ float3 ts_unproject(const TsIntrin& in, int i, int j, uint16_t d) {
  const float dep = div_vs((float)d, 1000.0f, 1.0f / 1000.0f);
  const float tx = ((float)i - in.cx) * dep, ty = ((float)j - in.cy) * dep;
  return make_float3(in.fdiv ? div_vs(tx, in.fx, in.rfx) : tx / in.fx, in.fdiv ? div_vs(ty, in.fy, in.rfy) : ty / in.fy, dep);
}

// per-frame bucket record (dense_tsdf.py:64-70 new_pcl_count / new_pcl_sum_pos / new_pcl_z), exact fixed-point sums
// (2^-20 m) in one 32-byte sector.  cd = cnt << cnt_shift | sum(d): the depth sum is non-negative, and the launch picks
// cnt_shift so that neither field can overflow into the other (ts_bucket_launch); a launch in which no shift can do that
// keeps the counts in a plane of their own instead (TsBucketLaunch::cnt).  The opener of a bucket stores the
// whole record; nobody clears it.  Textured maps keep the colour sums (new_pcl_sum_color, exact integer channel sums)
// in a second plane of uint4 {r, g, b, 0} at the same slot.
struct __align__(32) TsBucket {
  long long sx, sy, sz;
  unsigned long long cd;
};
// per-launch parameters of the bucket index (tslam_integrate.cu, ts_bucket_launch)
struct TsBucketLaunch {
  unsigned long long etag;  // launch epoch in the entry's epoch field; 0 in clearing mode
  int slot_bits;            // width of the slot + 1 field; 25 in clearing mode (no epoch field)
  int cnt_shift;            // cd = cnt << cnt_shift | sum(d)
  uint32_t* cnt;            // counts of the records when one bucket can collect more points than the word has room for
                            // (cd = sum(d) alone); else null
  uint32_t* bpos;           // clearing mode only: index entry of every opened record, zeroed by the consumer; else null
};

// The two ray set-ups (ray_setup, tslam_march.cu; k_raymarch, tslam_integrate.cu) read a bucket and form its ray
// through these two functions, so that both know the record format once and round alike (the parity tests compare
// their voxel indices bit for bit).
struct TsBucketSums {
  long long sx, sy, sz, sd;  // exact fixed-point sums of the points and of their depths
  int cnt;                   // points in the bucket
};
// record `id`, read with two 16-byte loads.  The record needs no clearing (its next opener stores it whole); in clearing
// mode its index entry is handed back zeroed (PCLroot.deactivate_all(), dense_tsdf.py:163).
__device__ __forceinline__ TsBucketSums ts_read_bucket(const TsBucket* buckets, unsigned long long* bidx, const TsBucketLaunch& bl, uint32_t id) {
  const uint4* q = reinterpret_cast<const uint4*>(&buckets[id]);  // sx sy | sz cd
  const uint4 q0 = q[0], q1 = q[1];
  if (bl.bpos) bidx[bl.bpos[id]] = 0ull;
  TsBucketSums b;
  b.sx = (long long)((unsigned long long)q0.x | ((unsigned long long)q0.y << 32));
  b.sy = (long long)((unsigned long long)q0.z | ((unsigned long long)q0.w << 32));
  b.sz = (long long)((unsigned long long)q1.x | ((unsigned long long)q1.y << 32));
  const unsigned long long cd = (unsigned long long)q1.z | ((unsigned long long)q1.w << 32);
  b.sd = bl.cnt ? (long long)cd : (long long)(cd & ((1ull << bl.cnt_shift) - 1ull));
  b.cnt = bl.cnt ? (int)bl.cnt[id] : (int)(cd >> bl.cnt_shift);
  return b;
}
// The ray of a bucket with cnt > 0 (process_new_pcl, dense_tsdf.py:240-251), seen from sensor origin T.  Returns false
// when the mean has no positive length (the ray marches no step); the other fields are then unset.
struct TsRayGeom {
  float mx, my, mz;  // pos_s2p: the exact mean (:243)
  float L;           // its length (:244)
  float ux, uy, uz;  // unit direction (:245)
  float Px, Py, Pz;  // pos_p = mean + T (:246)
  int oi, oj, ok;    // occupy voxel sxyz_to_ijk(pos_p) (:248)
  int n;             // march steps (:249-251)
  float w;           // sample weight w_x_p(d >= 0, z) = 1/z^2 with z = new_pcl_z/c (:216-225, :247, :262)
};
__device__ __forceinline__ bool ts_ray_geom(const TsBucketSums& b, const float* T, const TsIntrin& in, TsRayGeom& r) {
  const float vs = in.vs;
  const double den = (double)b.cnt * FIXQ_D;
  r.mx = (float)((double)b.sx / den);
  r.my = (float)((double)b.sy / den);
  r.mz = (float)((double)b.sz / den);
  const float zc = (float)((double)b.sd / den);
  r.L = sqrtf((r.mx * r.mx + r.my * r.my) + r.mz * r.mz);
  if (!(r.L > 0.0f)) return false;
  r.ux = r.mx / r.L; r.uy = r.my / r.L; r.uz = r.mz / r.L;
  r.Px = r.mx + T[0]; r.Py = r.my + T[1]; r.Pz = r.mz + T[2];
  r.oi = iroundf(r.Px / vs); r.oj = iroundf(r.Py / vs); r.ok = iroundf(r.Pz / vs);
  r.n = (int)fminf(r.L / vs + (float)in.internal_voxels, in.max_steps);
  r.w = 1.0f / (zc * zc);
  return true;
}

struct TsCounters {  // device-side statistics (tslam_tsdf_get_stats)
  unsigned long long n_px, n_valid, n_rays, n_updates, n_oob;
  // block-binned ray march (tslam_march.cu): diagnostics, not part of the parity counters
  unsigned long long n_segs, n_items, n_slow, n_fallback, n_generic, n_verify_bad;
  // segments the two walks of the binned march disagreed about (k_seg_scatter, k_march_blocks): must stay 0
  unsigned long long n_seg_guard;
};

// ---------------------------------------------------------------------------
// block-binned ray march (tslam_march.cu)
// ---------------------------------------------------------------------------
// One record per live ray (= per-frame bucket), written by k_ray_setup: unit direction, length, sensor origin in
// VOXEL units (T/vs) and the ray's sample weight 1/z^2 (dense_tsdf.py:243-247,262).
struct __align__(16) TsRay {
  float ux, uy, uz, L;
  float tx, ty, tz, w;
};
// aux word per ray: [31:16] n = number of march steps (dense_tsdf.py:249-251), [15:8] frame of the batch, [0] wide
// (more than 65535 steps: generic path)
#define TS_AUX_WIDE 1u
// A segment = run of consecutive march steps of one ray whose samples fall (approximately - every sample is
// re-checked exactly by the march kernel) into one 16^3 voxel block.  jc = frame << 24 | j0 << 8 | count (count <= 32).
struct TsSeg { uint32_t ray, jc; };
// generic-list records use jc = j0 << 12 | count (count <= 4095)
struct TsItem { int blk; uint32_t seg0, nseg, pad; };  // work item of k_march_blocks: <= MR_CHUNK segments of one block
#define MR_CHUNK 4096
struct TsMarchCtl {  // device-side control block of one launch (zeroed by the last CTA of k_march_blocks)
  int n_touched;     // blocks that received at least one segment
  int n_items;       // work items built by k_seg_class_scan
  int n_full;        // always 0 (k_seg_class_scan writes it, nobody reads it: the items are listed longest first)
  int item_cursor;   // persistent-CTA work cursor of k_march_blocks
  int n_gen;         // generic-list records
  int overflow;      // segments or work items did not fit: every segment goes through the generic path this launch
  unsigned int total_segs;
  unsigned int fmax_bits;  // float bits of max over rays of max(w, w*|ds|max): sizes the fixed-point scale of the launch
  int scale_k;       // shared-memory sums are kept in units of 2^-scale_k (k_seg_class_scan: largest k with max * 2^k < 2^30)
  int ticket;        // CTAs of k_march_blocks done: the last one clears this block
  int ticket_scan;   // CTAs of k_seg_class_scan done: the last one runs the scan
  int gen_cursor;    // generic-list cursor of k_march_blocks
  int pad2;
  int pad[3];
};
struct TsMarchWs {
  TsRay* rays;         // [ray_list_cap]
  uint32_t* aux;       // [ray_list_cap]
  TsSeg* seg;          // [seg_cap] segments grouped by block, ordered by length inside a block
  uint32_t seg_cap;
  int* seg_count;      // [max_blocks * 64] segments per (block, class, replica) (k_seg_count); k_seg_scatter counts
                       // each back down to 0 as it fills the run
  uint32_t* seg_rel;   // [max_blocks * 64] end of the (class, replica) range inside the block's run
  uint32_t* seg_off;   // [max_blocks] start of the block's run
  int* touched;        // [max_blocks] blocks with segments
  uint32_t* blk_total; // [max_blocks] segments of touched[i]
  uint32_t* blk_cost;  // [max_blocks] samples of touched[i] (upper estimate from the length classes)
  TsItem* items;       // [item_cap]
  uint32_t item_cap;
  TsSeg* gen;          // [gen_cap] generic-path records (volume boundary, over-long rays, overflow)
  uint32_t gen_cap;
  TsMarchCtl* ctl;
  float near_eps;      // |frac - 0.5| below this -> exact index path
};

// Change tracking of a map as a source or destination of the incremental fusions (tslam_tsdf_fuse_update,
// tslam_octo_fuse_update).  Every entry that writes a submap's voxels calls fz_written, which bumps that submap's content
// version and the map's write generation; an update compares both against what it recorded when it last ran.
struct FzVer {
  unsigned long long serial;        // process-unique number of the handle (an address can be reused by a new handle)
  unsigned long long write_gen;     // writes of the map by any entry other than the incremental fusion into it
  unsigned long long* content_ver;  // [n] host: writes of each submap's voxels
  int n;                            // max_submaps
};
// tslam_fuse.cu: at create (a fresh serial, versions zero) and destroy
void fz_ver_init(FzVer& v, int max_submaps);
void fz_ver_free(FzVer& v);
void fz_written(FzVer& v, int submap);  // submap's voxels were written (submap < 0: every submap)

// host-side handle
struct tslam_tsdf {
  tslam_tsdf_config_t cfg;
  int device;
  TsGrid g;
  TsIntrin in;
  size_t table_cap;
  // integrate workspace
  // per-frame bucket grid, split in two: a small open-addressing INDEX (8 B per entry: launch epoch + record slot +
  // 39-bit key) that the bucket kernel probes, and the 32-byte RECORDS with the exact sums (every warp of the bucket
  // kernel owns 32 of them), filled in the order the buckets are opened - so the ray set-up reads them in short runs
  TsBucket* buckets;   // records [TSLAM_MAX_BATCH * bucket_cap]; frame f owns [f * bucket_cap, (f + 1) * bucket_cap)
  uint4* bcol;         // colour sums of the records (texture_enabled only)
  unsigned long long* bidx;  // index [TSLAM_MAX_BATCH * bucket_cap]
  uint32_t bucket_cap; // power of two
  int bk_slot_bits;    // width of the index entry's slot + 1 field (25: clearing mode, no epoch field)
  unsigned int bk_epoch, bk_epoch_max;  // epoch of the last launch, 1 .. 2^(25 - bk_slot_bits) - 1
  uint32_t* bpos;      // clearing mode only: [TSLAM_MAX_BATCH * bucket_cap] index entry of every opened record
  uint32_t* bcnt;      // [TSLAM_MAX_BATCH * bucket_cap] record counts, for launches whose counts do not fit the packed
                       // word; allocated only when the handle accepts such launches
  uint32_t* ray_list;  // [TSLAM_MAX_BATCH * max_rays_per_frame]
  uint32_t ray_list_cap;
  int* n_rays;         // device counter
  uint16_t* depth_stage;  // device staging for host depth input [TSLAM_MAX_BATCH * max_image_pixels]
  uint8_t* tex_stage;     // device staging for host textures [2 * TSLAM_MAX_BATCH * max_image_pixels * 3] (texture_enabled only)
  uint8_t* rgb_stage;     // device staging for point-cloud colours
  unsigned int frame_seq; // frames integrated since the last renormalisation of the colour words (ts_seq_renorm)
  int q_th, q_tw, q_has_tex;
  // pinned host frames are not copied: q_hptr[q] = their device alias; the sampled rows are fetched over PCIe by
  // k_gather_rows in groups of TS_GATHER_GROUP frames (q_gathered = frames already handed to a gather launch)
  const uint16_t* q_hptr[TSLAM_MAX_BATCH];
  int q_gathered;
  int zero_copy;  // 1 = borrow page-locked frames (tslam_tsdf_set_frame_mode / TSLAM_ZERO_COPY=1); 0 = copy (default)
  // copy mode, pageable frames: the call copies the SAMPLED ROWS of the frame into this page-locked ring on the host (the
  // caller may reuse its buffer at once) and the GPU fetches them from there like a borrowed frame
  uint16_t* h_ring;       // [2][TSLAM_MAX_BATCH][ring_frame_cap] host, mapped
  uint16_t* h_ring_dev;   // its device alias
  size_t ring_frame_cap;  // elements per frame slot
  int stage_mode;         // pageable frames: 1 = through the ring (default), 0 = through cudaMemcpyAsync (TSLAM_FRAME_COPY=dma)
  int pinned_mode;        // copy mode, page-locked source: 2 = awaited DMA copy (default), 0 = through the ring like pageable frames, 1 = awaited row fetch
  int q_open, q_await;    // a frame's hand-over has begun (tslam_tsdf_queue_depth_begin) / its DMA copy is still to be awaited
  int q_sstride[TSLAM_MAX_BATCH];  // source row stride of the queued frame in 16-byte units
  int queue_launch[2];  // frames per queue launch, alternating (TSLAM_QUEUE_LAUNCH="a,b", default 32,32)
  int q_phase;          // which of the two thresholds the current launch uses (back to 0 at every flush)
  int trace;         // TSLAM_TRACE=1: print a per-launch timeline of the queue (debug)
  cudaEvent_t tr_ev[2][4];  // per staging buffer: copy stream first op / last op, main stream launch begin / end
  cudaEvent_t tr_base;
  int tr_have[2];
  int rm_reserve;    // SMs left out of the ray-march grid (2 once page-locked frames are being gathered, else 0)
  float* points_stage;    // device staging for host point clouds
  TsCounters* counters;
  float* pose_R;       // device pose table [max_submaps*9]
  float* pose_T;       // [max_submaps*3]
  float* colormap;     // device jet LUT [1024*3]
  int* scratch_i;      // small device scratch (counters for gather etc.)
  void* esdf_aux;      // ESDF: neighbour table, epochs, per-sweep change flags, class bytes (allocated with g.esdf)
  int esdf_full_needed, esdf_submap;  // the next update recomputes everything (first use, reset, bulk load) / submap of the kept state
  int esdf_tiled;      // tiled ESDF (tslam_esdf_tiled_*): 0 = none (plain update), 1 = begun, exchange in progress, 2 = ended
  void* mc_scratch;    // marching cubes: per-block triangle counts / offsets (allocated on first use)
  // Change tracking for the incremental mesh (tslam_mesh_*, tslam_mc.cu).  Every commit (k_commit_tma) and
  // every ghost import (k_ghost_unpack) takes the next commit_seq and stores it in blk_stamp[] of each block it writes;
  // every other writer of the tw / obs / col planes, and whatever recycles pool slots, bumps mesh_epoch instead
  // (DESIGN.md section 4 lists them).
  unsigned long long* blk_stamp;  // [max_blocks] commit_seq of the last commit / ghost import that wrote the block
  unsigned long long commit_seq;
  unsigned long long mesh_epoch;
  long long launches;
  int n_integrate_calls;
  int profiling;
  unsigned long long* prof;  // device profiling ring: TS_PROF_RING launches x TS_PROF_WORDS kernel stamps (allocated lazily)
  unsigned char prof_ran[TS_PROF_RING];  // per ring row: bit k = kernel k (TS_K_*) stamped that row
  long long prof_launches;   // integrate launches recorded since profiling was switched on
  int sm_count;
  int tile_cuts_set, tile_cuts_tiles[3], tile_cuts[3][17];  // data-driven tile boundaries of a tiled global map (tslam_dist.cu)
  int* tile_hist;      // device scratch of tslam_tsdf_dirty_hist (allocated on first use)
  TsMarchWs mw;        // block-binned ray march workspace (tslam_march.cu)
  // SDF-to-SDF registration (tslam_tsdf_register, tslam_register.cu) with this map as the reference map: per pool block
  // scratch of the point selection, and the point records and per-iteration sums (each grown geometrically)
  void* reg_blk;
  size_t reg_blk_bytes;
  void* reg_pts;
  size_t reg_pts_bytes;
  void* render_jobs;   // per-camera jobs of tslam_tsdf_render (tslam_render.cu), grown geometrically
  size_t render_jobs_bytes;
  void* traj_mem;      // inputs, outputs and solver work of tslam_esdf_trajectory (tslam_traj.cuh), grown geometrically
  size_t traj_mem_bytes;
  void* rc_mem;        // keep flags, scan, hole / mover lists and counters of tslam_tsdf_reclaim (tslam_reclaim.cu), grown geometrically
  size_t rc_bytes;
  FzVer ver;                        // change tracking of the incremental fusion (writes of the tw / obs / occ / col planes)
  unsigned long long ghost_gen;     // ... of which ghost imports (tslam_tsdf_ghost_unpack): the tiled update ignores them
  struct TsFuse* fz;                // state of this map as the destination of tslam_tsdf_fuse_update (first call allocates)
  int march_verify;    // TSLAM_MARCH_VERIFY=1: every fast-path index is re-computed exactly, mismatches counted
  bool clamp_on_commit;
  // frame queue of the per-frame API (tslam_tsdf_queue_depth): double-buffered device staging fed by a copy stream
  int q_n, q_buf, q_h, q_w;
  float q_R[TSLAM_MAX_BATCH * 9];
  float q_T[TSLAM_MAX_BATCH * 3];
  int q_s[TSLAM_MAX_BATCH];
  cudaStream_t copy_stream;
  cudaEvent_t ev_copied[2], ev_free[2];
  bool ev_free_valid[2];
};

// ---------------------------------------------------------------------------
// Octomap: hash grid of 8^3 blocks of u32 hit counters (taichi_octomap.py:63-84
// builds a K-ary pointer tree with one allocation per leaf instead)
// ---------------------------------------------------------------------------
#define OC_B 8
#define OC_B3 512
#define OC_BSHIFT 3
#define OC_BMASK 7
struct OcGrid {
  unsigned long long* table;
  uint32_t table_mask;
  int max_blocks;
  int* n_blocks;
  unsigned long long* block_key;
  unsigned int* cnt;  // [max_blocks*512]
  unsigned long long* cw;  // texture_enabled: [max_blocks*512] colour word (integrate seq << 24 | r << 16 | g << 8 | b), atomicMax
  int* err;
  int hN, hNz, N, Nz;
};
__device__ __forceinline__ int oc_voxel_off(int i, int j, int k) {
  return (((i & OC_BMASK) << OC_BSHIFT) | (j & OC_BMASK)) << OC_BSHIFT | (k & OC_BMASK);
}
// Placement of source voxel v of block (bx, by, bz) of a submap at pose (R, T) by the Octomap fusions (k_octo_fuse and
// the incremental update, tslam_octo_fuse.cu; taichi_octomap.py:182-186): x = R (i vs, j vs, k vs) + T lands in the
// nearest dst cell (int)roundf(x / vs) per axis.  Both call this one helper, so they place every voxel alike.
__device__ __forceinline__ void oc_fuse_cell(const float* R, const float* T, int bx, int by, int bz, int v, float vs, int& i, int& j,
                                             int& k) {
  float x, y, z;
  pose_apply(R, T, (float)(bx * OC_B + (v >> 6)) * vs, (float)(by * OC_B + ((v >> 3) & 7)) * vs, (float)(bz * OC_B + (v & 7)) * vs, x, y, z);
  i = (int)roundf(x / vs); j = (int)roundf(y / vs); k = (int)roundf(z / vs);
}
// Log-odds occupancy (tslam_octo_create_logodds, DESIGN.md section 7): the cnt plane holds w = (L << 1) | 1 for a
// known voxel and 0 for an unknown one, so a zeroed block reads unknown.  L is Q10 fixed point, clamped to
// [l_min, l_max] after every update.
__host__ __device__ __forceinline__ bool lo_known(unsigned int w) { return (w & 1u) != 0; }
__host__ __device__ __forceinline__ int lo_val(unsigned int w) { return (int)w >> 1; }
__host__ __device__ __forceinline__ unsigned int lo_word(int L) { return ((unsigned int)L << 1) | 1u; }
// Voxel class of a log-odds word, for every tracker: UNKNOWN = not known, OCC = known and L > l_occ, FREE = known and
// L <= l_occ.  The values are a data format: the occupancy ESDF stores them in its class bytes, and the travel-cost
// field reads them back from there (OcEsdfField::free_cls).
enum { OC_UNK = 0, OC_FREE = 1, OC_OCC = 2 };
__device__ __forceinline__ unsigned char oc_class(unsigned int w, int l_occ) {
  return !lo_known(w) ? OC_UNK : (lo_val(w) > l_occ ? OC_OCC : OC_FREE);
}
// Occupancy rule of the Octomap readers (planner queries, LoD export, fusion, gather) for a cnt word c: OcHits for a hit
// counter, OcLogodds for a log-odds map.  The readers are written once over the rule (tslam_query.cu, tslam_octo.cu).
struct OcHits {
  float thres;  // (float)min_occupy_thres
  // is_occupy (taichi_octomap.py:86-88); an absent cell reads 0, so there is no c > 0 test
  __device__ __forceinline__ bool occ(unsigned int c) const { return (float)c > thres; }
  __device__ __forceinline__ bool unknown(unsigned int) const { return false; }
  // LoD export: the group's corner voxel exists (c > 0) and is occupied (:90-114)
  __device__ __forceinline__ bool export_occ(unsigned int c) const { return c > 0 && (float)c > thres; }
  // fusion: which source voxels are carried over (:181), and how one adds to its target voxel (occupy[ijk_] += c, :183-186)
  __device__ __forceinline__ bool fuse_src(unsigned int c) const { return (float)c > thres; }
  __device__ __forceinline__ void fuse_add(unsigned int* p, unsigned int c) const { atomicAdd(p, c); }
  // gather: the voxels with a hit, and their count
  static __device__ __forceinline__ bool gather_keep(unsigned int c) { return c > 0; }
  static __device__ __forceinline__ unsigned int gather_val(unsigned int c) { return c; }
};
struct OcLogodds {
  int l_occ;
  __device__ __forceinline__ bool occ(unsigned int c) const { return lo_known(c) && lo_val(c) > l_occ; }
  __device__ __forceinline__ bool unknown(unsigned int c) const { return !lo_known(c); }
  __device__ __forceinline__ bool export_occ(unsigned int c) const { return lo_known(c) && lo_val(c) > l_occ; }
  // every known voxel is carried over; the target collects (sum L) << 1 by additions of L << 1 and its known bit by an
  // OR, so the result does not depend on the order (k_octo_lo_clamp clamps it once all sums are in)
  __device__ __forceinline__ bool fuse_src(unsigned int c) const { return lo_known(c); }
  __device__ __forceinline__ void fuse_add(unsigned int* p, unsigned int c) const {
    red_add_u32(p, (unsigned int)lo_val(c) << 1);
    atomicOr(p, 1u);
  }
  // gather: the known voxels, and their L (int32 bits)
  static __device__ __forceinline__ bool gather_keep(unsigned int c) { return lo_known(c); }
  static __device__ __forceinline__ unsigned int gather_val(unsigned int c) { return (unsigned int)lo_val(c); }
};
#define OC_MARK_WORDS 32  // mark words per block: 0..15 hit bits, 16..31 miss bits of its 512 voxels (128 B per block)
struct OcLo {             // per-frame workspace of a log-odds map (allocated in log-odds mode only)
  uint32_t* mark;         // [max_blocks * 32] hit / miss bits of the frame, cleared by k_octo_lo_apply
  int* touched_flag;      // [max_blocks] 1 = the block is on the touched list of this frame
  int* touched;           // [max_blocks] blocks touched by the frame, in first-touch order
  int* ctr;               // [0] ray records, [1] touched blocks of the frame
  float4* rays;           // [ray_cap] ray endpoint (map frame, metres); w = 1 clipped (misses only), 0 ends in a hit
  unsigned long long* stats;  // [4] rays cast, in-volume miss-cell visits, hit voxels, voxels updated
  float min_ray, max_ray; // f32(min_ray_length), f32(max_ray_length)
  int l_hit, l_miss, l_min, l_max, l_occ;
};
// What a tracker of a log-odds map (occupancy ESDF, frontiers, travel-cost fields) kept can be read for `submap` iff an
// update for that submap has completed and no reset, fusion (tslam_octo_fuse, or a full tslam_octo_fuse_update) or
// failed update came after it (oc_track_readable).  Integration and an incremental tslam_octo_fuse_update leave it
// readable: readers answer as of their last update, and both flag the blocks they change for the next incremental one.
struct OcTrack {
  int ready;   // set when an update completes; cleared when one begins, and by reset and fusion (oc_track_invalidate_all)
  int submap;  // submap of that update
};
// S travel-cost fields of one submap as of one update (tslam_octo_travel.cu), allocated by the first update
struct OcTravel {
  void* blk;      // per pool block: traversable bits, compact slot (68 B); change flags, per-source arrays
  void* mem;      // per compact slot: allowed steps, neighbour table; per (slot, source): field, epoch (grown geometrically)
  size_t bytes;   // bytes of mem
  OcTrack track;  // the kept fields
  int S, nt;      // sources and compact slots of the kept fields
};
struct tslam_octo {
  tslam_octo_config_t cfg;
  OcGrid g;
  TsIntrin in;
  size_t table_cap;
  uint16_t* depth_stage;
  float* points_stage;
  uint8_t* tex_stage;     // texture_enabled: device staging of a host colour image / point colours
  unsigned int frame_seq; // integrate calls so far
  float* pose_R;
  float* pose_T;
  int* scratch_i;
  long long launches;
  int sm_count;
  int logodds;            // 1 = log-odds occupancy (fixed at creation), 0 = hit counter
  OcLo lo;
  int ray_cap;            // ray records per frame: max(max_image_pixels, max_points)
  // occupancy ESDF of a log-odds map (tslam_octo_esdf_*, tslam_octo_esdf.cu), allocated by the first update
  void* esdf_mem;         // field, class bytes, neighbour table, epochs, change flags
  int* esdf_dirty;        // [max_blocks] block updated by k_octo_lo_apply since the last ESDF update; NULL until then
  OcTrack esdf_track;     // the kept field (not ready: the next update recomputes everything)
  float esdf_D;           // truncation distance of the kept field
  // frontier tracker of a log-odds map (tslam_octo_frontier_*, tslam_octo_frontier.cu), allocated by the first update
  void* fr_mem;           // per pool block: frontier mask, dirty and region flags, region list, popcount, offset (84 B)
  int* fr_dirty;          // [max_blocks] block updated by k_octo_lo_apply since the last frontier update; NULL until then
  OcTrack fr_track;       // the kept frontier set (not ready: the next update recomputes everything)
  int fr_nb;              // pool blocks the last update saw
  int fr_n, fr_nc;        // frontier voxels and clusters of the last update
  void* fr_vox;           // per frontier voxel: union-find parent, cluster slot of a root (grown on demand)
  long long fr_vox_cap;
  void* fr_clu;           // per cluster: label, record, sort keys / values, ordinal (grown on demand)
  long long fr_clu_cap;
  void* fr_tmp;           // CUB scan / sort scratch
  size_t fr_tmp_bytes;
  // viewpoint gain (tslam_octo_view_gain_*, tslam_octo_view.cu): per-view bitmaps of a chunk of views, or the frontier
  // rows of the frontier gain (grown on demand, freed by tslam_octo_destroy)
  void* vw_mem;
  size_t vw_bytes;
  // travel-cost fields of a log-odds map (tslam_octo_travel_*, tslam_octo_travel.cu): the single-source field
  // (tslam_octo_travel_update, S = 1) and the many-source fields (tslam_octo_travel_multi_update), kept apart
  OcTravel tr, trm;
  // inputs, outputs and solver work of tslam_octo_esdf_trajectory (tslam_traj.cuh), grown geometrically
  void* traj_mem;
  size_t traj_mem_bytes;
  FzVer ver;                        // change tracking of the incremental fusion (writes of the cnt / cw planes)
  struct FzState* fz;               // state of this map as the destination of tslam_octo_fuse_update (first call allocates)
};
int oc_esdf_free(tslam_octo* m);      // tslam_octo_esdf.cu
int oc_frontier_free(tslam_octo* m);  // tslam_octo_frontier.cu
int oc_view_free(tslam_octo* m);      // tslam_octo_view.cu
int oc_travel_free(tslam_octo* m);    // tslam_octo_travel.cu
// tslam_octo_esdf.cu: the occupancy ESDF of `submap` as of its last update, for the clearance test of the travel-cost
// field.  Refused like tslam_octo_esdf_gather (the message naming `what`).  A voxel at pool offset o was FREE at that
// update, in a block it saw, with field value e[o] iff o / 512 < *nb_seen and (cls[o] & cls_mask) == free_cls (OC_FREE).
struct OcEsdfField {
  const float* e;            // [max_blocks*512] field, in the cnt plane's layout
  const unsigned char* cls;  // [max_blocks*512] class byte of the update
  const int* nb_seen;        // DEVICE: pool blocks the update saw
  float D;                   // its truncation distance
  unsigned char free_cls, cls_mask;
};
int oc_esdf_field(tslam_octo* m, int32_t submap, const char* what, OcEsdfField* f);
// The traversability rule of the travel-cost fields, for cell (i, j, k) with map word w at pool offset o = b * 512 + v:
// inside the volume and FREE, and with clear (clearance > 0) also FREE at the last ESDF update, in a block it saw
// (b < enb = *ef.nb_seen), with ESDF value >= clearance.  The travel classify and the viewpoint candidates test it.
__device__ __forceinline__ bool oc_traversable(const OcGrid& g, const OcEsdfField& ef, int l_occ, float clearance, bool clear, int enb,
                                               int b, size_t o, unsigned int w, int i, int j, int k) {
  bool t = ts_in_bounds(g, i, j, k) && lo_known(w) && lo_val(w) <= l_occ;
  if (t && clear) t = b < enb && (ef.cls[o] & ef.cls_mask) == ef.free_cls && ef.e[o] >= clearance;
  return t;
}
// tslam_octo_travel.cu: the clearance check of every call that tests oc_traversable - finite and >= 0, and when > 0 a
// readable occupancy ESDF of `submap` (into *ef) whose max_dist is >= clearance; *ef is zeroed when clearance == 0
int oc_clearance_field(tslam_octo* m, int32_t submap, float clearance, const char* what, OcEsdfField* ef);
// tslam_octo_frontier.cu: the m->fr_n rows (ijk, cluster ordinal) of the frontier set into idx[fr_n * 3], cluster[fr_n]
// (DEVICE), in compact order, on st; the caller has checked m->fr_track
int oc_frontier_rows(tslam_octo* m, int32_t* idx, int32_t* cluster, cudaStream_t st);
// tslam_octo_frontier.cu: the m->fr_nc cluster records in label (ordinal) order into rec16[fr_nc * 16] (DEVICE), as
// tslam_octo_frontier_clusters writes them, on st; the caller has checked m->fr_track
int oc_frontier_records(tslam_octo* m, int64_t* rec16, cudaStream_t st);
// tracker bits of g.err next to TS_ERR_POOL_FULL / TS_ERR_TABLE_FULL: the next synchronising call names every bit that is
// set (oc_deferred, tslam_octo.cu)
#define OC_ERR_VIEW_WINDOW 16  // g.err: a viewpoint-gain walk left its view's bitmap window (tslam_octo_view.cu)
#define OC_ERR_TRAVEL_PATH 32  // g.err: a travel path found no predecessor (impossible at the field's fixed point; tslam_octo_travel.cu)
#define OC_ERR_TRAVEL_SOURCE 64  // g.err: a many-source travel path named a source outside [0, S) (tslam_octo_travel.cu)
#define OC_ERR_FUSE_MISSING 128  // g.err: a removal of tslam_octo_fuse_update found no dst block (tslam_octo_fuse.cu)

// Amanatides-Woo traversal of the log-odds map in voxel units (DESIGN.md section 7, "Traversal"): p0 = origin / vs,
// p1 = endpoint / vs, cells c = round_half_away(p).  The k-th boundary crossing of axis a is at
// t = ((c_a + 0.5 s_a) - p0_a) * (1 / (p1_a - p0_a)), recomputed from the current cell (no accumulated increments); each
// step takes the axis with the smallest t among those with steps left, ties to the lower axis.  The step counts
// |c1 - c0| per axis are integers, so the path always has |c1 - c0|_1 + 1 cells.  The viewpoint-gain kernels walk with
// it; k_octo_lo_walk (tslam_octo.cu) spells out the same expressions, because calling the helper there changes that
// kernel's SASS (the step becomes a jump table).  The gain tests check the two paths agree bit for bit.
struct OcWalk {
  int cx, cy, cz;   // current cell
  int lx, ly, lz;   // steps left per axis
  int sx, sy, sz;   // step direction per axis
  float p0x, p0y, p0z, hx, hy, hz, ix, iy, iz, tx, ty, tz;
};
__device__ __forceinline__ void oc_walk_begin(OcWalk& w, float p0x, float p0y, float p0z, float p1x, float p1y, float p1z) {
  w.p0x = p0x; w.p0y = p0y; w.p0z = p0z;
  w.cx = (int)roundf(p0x); w.cy = (int)roundf(p0y); w.cz = (int)roundf(p0z);
  const int ex = (int)roundf(p1x), ey = (int)roundf(p1y), ez = (int)roundf(p1z);
  w.lx = abs(ex - w.cx); w.ly = abs(ey - w.cy); w.lz = abs(ez - w.cz);
  w.sx = ex > w.cx ? 1 : -1; w.sy = ey > w.cy ? 1 : -1; w.sz = ez > w.cz ? 1 : -1;
  w.hx = 0.5f * (float)w.sx; w.hy = 0.5f * (float)w.sy; w.hz = 0.5f * (float)w.sz;
  w.ix = w.lx ? 1.0f / (p1x - p0x) : 0.0f; w.iy = w.ly ? 1.0f / (p1y - p0y) : 0.0f; w.iz = w.lz ? 1.0f / (p1z - p0z) : 0.0f;
  w.tx = (((float)w.cx + w.hx) - p0x) * w.ix; w.ty = (((float)w.cy + w.hy) - p0y) * w.iy; w.tz = (((float)w.cz + w.hz) - p0z) * w.iz;
}
// one step to the next cell of the path; only while steps are left (lx + ly + lz > 0)
__device__ __forceinline__ void oc_walk_step(OcWalk& w) {
  int a = 3;
  float tb = 0.0f;
  if (w.lx > 0) { a = 0; tb = w.tx; }
  if (w.ly > 0 && (a == 3 || w.ty < tb)) { a = 1; tb = w.ty; }
  if (w.lz > 0 && (a == 3 || w.tz < tb)) a = 2;
  if (a == 0) { w.cx += w.sx; --w.lx; w.tx = (((float)w.cx + w.hx) - w.p0x) * w.ix; }
  else if (a == 1) { w.cy += w.sy; --w.ly; w.ty = (((float)w.cy + w.hy) - w.p0y) * w.iy; }
  else { w.cz += w.sz; --w.lz; w.tz = (((float)w.cz + w.hz) - w.p0z) * w.iz; }
}
// k_octo_lo_apply flags the blocks it updates for these change trackers (tslam_octo.cu)
#define OC_TRACK_ESDF 1u
#define OC_TRACK_FRONTIER 2u

// 64-bit max without a return value: RED.E.MAX.64 (atomicMax(unsigned long long*) with an unused result was lowered
// to ATOMG - a response sector per update, seen as 57 M "L2 ATOM sectors" per textured launch in ncu)
__device__ __forceinline__ void ts_red_max_u64(unsigned long long* addr, unsigned long long v) {
  asm volatile("red.relaxed.gpu.global.max.u64 [%0], %1;" ::"l"(addr), "l"(v) : "memory");
}

// colour pixel of depth pixel (i, j): texture[j, i] (color_same_proj) or color_ind_from_depth_pt
// (mapping_common.py:43-58).  The reference tests color_i against h and color_j against w (swapped, :56); what passes
// that test but lies outside the image is an out-of-bounds read there - pixel (0,0) here.  Returns false when even the
// same-projection pixel is outside the colour image.
__device__ __forceinline__ bool ts_color_pixel(const TsIntrin& in, int i, int j, int th, int tw, int& ti, int& tj) {
  tj = j; ti = i;
  if (!in.same_proj) {
    ti = (int)((((float)i - in.cx) / in.fx) * in.fxc + in.cxc);
    tj = (int)((((float)j - in.cy) / in.fy) * in.fyc + in.cyc);
    if (ti < 0 || ti >= th || tj < 0 || tj >= tw || tj >= th || ti >= tw) { ti = 0; tj = 0; }
  }
  return tj < th && ti < tw;
}

// error plumbing (tslam_tsdf.cu)
void ts_set_error(const char* fmt, ...);
int ts_cuda_fail(cudaError_t e, const char* what);
#define TS_CUDA(x)                                    \
  do {                                                \
    cudaError_t _e = (x);                             \
    if (_e != cudaSuccess) return ts_cuda_fail(_e, #x); \
  } while (0)
#define TS_LAUNCH_CHECK(m)                                              \
  do {                                                                  \
    (m)->launches++;                                                    \
    cudaError_t _e = cudaGetLastError();                                \
    if (_e != cudaSuccess) return ts_cuda_fail(_e, "kernel launch");    \
  } while (0)

// Launch with programmatic dependent launch (Hopper): the kernel may start while its predecessor on `st` is still
// running, and must call cudaGridDependencySynchronize() before it reads anything the predecessor writes - on every
// path, so that it never completes before the predecessor.  After an event record or a memset it is an ordinary launch.
template <class... KArgs, class... Args>
static cudaError_t ts_launch_pdl(void (*k)(KArgs...), dim3 grid, int block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3((unsigned)block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, k, std::forward<Args>(args)...);
}

// Tiling of a tiled global map over `world` ranks (tslam_dist.cu, and the tiled incremental fusion in tslam_fuse.cu)
#define TS_MAX_TILES_AXIS 16
struct TsTiling {
  int tiles[3];
  int rank, world;
  int cuts[3][TS_MAX_TILES_AXIS + 1];  // tile k of axis a owns block coordinates [cuts[a][k], cuts[a][k+1])
};

__host__ __device__ __forceinline__ int tile_coord(const TsTiling& t, int axis, int b) {
  int c = 0;
  while (c + 1 < t.tiles[axis] && b >= t.cuts[axis][c + 1]) ++c;  // (blocks outside the cut range belong to the end tiles)
  return c;
}
__host__ __device__ __forceinline__ int tile_owner(const TsTiling& t, int bx, int by, int bz) {
  return (tile_coord(t, 0, bx) * t.tiles[1] + tile_coord(t, 1, by)) * t.tiles[2] + tile_coord(t, 2, bz);
}

// shared across translation units
// tslam_dist.cu: the tiling of m for tiles3 / rank / world (its installed cuts when they match tiles3, else equal slices)
int fill_tiling(tslam_tsdf* m, const int32_t* tiles3, int rank, int world, TsTiling* t);
// tslam_integrate.cu
int ts_integrate_init();                                // once per process, before the first integrate launch
// commit if anything is pending; prof: the stamp row of the profiled integrate launch it belongs to, or null
int ts_flush_pending(tslam_tsdf* m, cudaStream_t st, unsigned long long* prof = nullptr);
// k_collect_dirty + commit of the dirty blocks
int ts_launch_commit(tslam_tsdf* m, cudaStream_t st, int clamp, int fused, unsigned long long* prof = nullptr);
int ts_check_deferred(tslam_tsdf* m);                    // read + translate device error flags (synchronises)
int ts_check_deferred_async(tslam_tsdf* m, cudaStream_t st);  // same, after the work queued on st
double ts_bucket_dmax(const tslam_tsdf* m);
int ts_check_tex(tslam_tsdf* m, const uint8_t* tex, int th, int tw);  // a colour image the map can take, or none
int ts_integrate_depth_impl(tslam_tsdf_t* m, const uint16_t* depth, int mem, int32_t n_frames, int32_t h, int32_t w, const float* R9s,
                            const float* T3s, const int32_t* submap_ids, int flags, void* stream, const uint8_t* tex = nullptr, int th = 0,
                            int tw = 0);
void ts_fuse_free(tslam_tsdf* m);                        // tslam_fuse.cu: the fusion state, at destroy
// the fusion sum planes of m as a destination (tslam_reclaim.cu moves them with their blocks): sums = null when none
struct TsFuseView {
  long long* sums;    // planes x cap_blocks x 4096 int64, plane after plane
  size_t cap_blocks;  // pool blocks the planes cover
  int planes;         // 3, or 6 on textured maps
  int valid;          // the sums describe the map (the last update completed)
  int phase;          // phase of a tiled update in progress, 0 none
};
TsFuseView ts_fuse_view(tslam_tsdf* m);
// tslam_integrate.cu: k_collect_dirty on st (dirty_flag -> dirty_list, n_dirty)
int ts_collect_dirty(tslam_tsdf* m, cudaStream_t st, unsigned long long* prof = nullptr);
// tslam_register.cu: *p holds at least `need` bytes: reallocated (contents dropped) to max(need, 2 x the old size) when smaller
int rg_reserve(void** p, size_t* bytes, size_t need);
// tslam_register.cu: the registration point selection (k_rg_count, sort, k_rg_permute, scan, then k_rg_fill) that
// tslam_tsdf_register and tslam_tsdf_place_describe share; the block arrays it leaves in A->reg_blk
struct RgSel {
  int nb;                                 // pool blocks scanned
  const int* order; const int* cs; const int* off;  // blocks sorted by slot, their counts and exclusive scan
};
int rg_select_count(tslam_tsdf* A, const std::vector<int>& slot_of, int U, float band, float min_weight, RgSel& sel,
                    std::vector<int>& slot_cnt, cudaStream_t st);
int rg_select_fill(tslam_tsdf* A, const RgSel& sel, float band, float min_weight, float4* pts, cudaStream_t st);
// tslam_queue.cu: the per-frame queue's switches, copy stream and events of a new handle / their release
int ts_queue_init(tslam_tsdf* m);
void ts_queue_free(tslam_tsdf* m);
int ts_launch_queue(tslam_tsdf* m, cudaStream_t st);     // integrate the queued frames, if any
// tslam_esdf.cu: per-block exchange mark of the tiled ESDF ([max_blocks]; owned block: ESDF changed since it was last
// packed, ghost block: ESDF unpacked since the last relax), or NULL before the first ESDF update
int* ts_esdf_xmark(tslam_tsdf* m);
// tslam_march.cu: block-binned ray march of the rays listed in m->ray_list (untextured maps)
int ts_march_alloc(tslam_tsdf* m);
void ts_march_free(tslam_tsdf* m);
int ts_march_launch(tslam_tsdf* m, cudaStream_t st, const TsBatch& batch, uint32_t bucket_shift, const TsBucketLaunch& bl, unsigned long long* prof);

// Octomap host helpers shared by its trackers (tslam_octo.cu)
// the arguments every tracker call checks first: a log-odds map (`feature` names what needs one), submap in range
int oc_logodds_submap(tslam_octo* m, int32_t submap, const char* what, const char* feature);
// the state kept in t can be read for `submap` (see OcTrack); `update` names the entry point that computes it
int oc_track_readable(tslam_octo* m, const OcTrack& t, int32_t submap, const char* what, const char* update);
// reads and clears the device error flags (synchronous): TSLAM_E_POOL_FULL for a pool / table bit, else TSLAM_E_INVALID
// naming every tracker bit that is set
int oc_deferred(tslam_octo* m);
// reset and fusion recycle pool slots: no tracker's kept state describes the map any more
void oc_track_invalidate_all(tslam_octo* m);
// *p holds at least `need` bytes: reallocated to exactly `need` when smaller (the contents are not kept)
int oc_reserve(void** p, size_t* bytes, size_t need);
// CTAs for `work` items at `per_cta` per CTA: at least 1, at most cap
static inline int oc_grid(long long work, int per_cta, int cap) {
  const long long g = (work + per_cta - 1) / per_cta;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}
// f(rule) with the occupancy rule of the map's mode (OcHits / OcLogodds): one launch site for both readers' instantiations
template <class F>
static void oc_with_rule(const tslam_octo* m, F f) {
  if (m->logodds) f(OcLogodds{m->lo.l_occ});
  else f(OcHits{(float)m->cfg.min_occupy_thres});
}
// Count-then-fill gather: launch(counter) enqueues one kernel on st that appends its rows through warp_append_u64 on the
// zeroed counter and writes those below cap.  Synchronises; *n_out = the rows found, TSLAM_E_CAPACITY when more than cap.
template <class F>
int oc_counted_gather(tslam_octo* m, cudaStream_t st, F launch, int64_t cap, int64_t* n_out, const char* what) {
  unsigned long long* ctr = (unsigned long long*)(m->scratch_i + 8);
  TS_CUDA(cudaMemsetAsync(ctr, 0, 8, st));
  launch(ctr);
  TS_LAUNCH_CHECK(m);
  unsigned long long v = 0;
  TS_CUDA(cudaMemcpyAsync(&v, ctr, 8, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  *n_out = (int64_t)v;
  if ((int64_t)v > cap) { ts_set_error("%s: %lld rows > capacity %lld", what, (long long)v, (long long)cap); return TSLAM_E_CAPACITY; }
  return TSLAM_OK;
}
