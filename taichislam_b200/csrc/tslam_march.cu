// libtslam.so - block-binned ray march (round 2).  sm_90a.
//
// Replaces the one-thread-per-ray march of round 1 (k_raymarch: one 8-byte global reduction per sample, bound by the
// L2 reduction rate whatever the kernel did) for untextured maps.  process_new_pcl
// (dense_tsdf.py:236-270) becomes
//
//   k_seg_count    one lane per ray.  Ray set-up (one bucket, read sequentially from the dense per-ray array): exact
//                  bucket mean -> unit direction, length, weight, step count n (:240-251), occupy flag (:248), a
//                  32-byte record.  Then a 3-D DDA (seg_generate) cuts the ray into SEGMENTS - runs of consecutive
//                  steps that stay in one 16^3 voxel block - activates the blocks on the way and counts the segments
//                  per (block, length class) with warp-aggregated reductions.  It stores no segment;
//   k_seg_class_scan  per touched block: class counts -> offsets inside the block's run, list of touched blocks;
//                  then its last CTA: exclusive scan over the touched blocks -> run offsets + work items
//                  (<= MR_CHUNK segments of one block each, longest first);
//   k_seg_scatter  walks every ray again from its stored record (the same seg_generate, so the same segments in the
//                  same order) and stores each segment at its place: a block's run is ordered by segment length;
//   k_march_blocks persistent CTAs take work items.  The block's pending sums live in SHARED MEMORY as exact 64-bit
//                  fixed-point words (no-return ATOMS.ADD: an order of magnitude more lane-atomics/s than
//                  global reductions, tools/ubench/atoms_bench.cu).  A warp walks 32 segments of equal length
//                  in lock step, one per lane, ray parameters in registers.  Each sample's voxel index comes from
//                  ONE fused multiply-add per axis in block-local voxel units and is accepted only when its
//                  fractional part is at least near_eps away from .5 - otherwise (~2e-3 of the samples) the lane
//                  recomputes round((u*j*vs + T)/vs) exactly as the reference states it (:253-254), so voxel
//                  indices stay bit-exact; a sample whose exact voxel is not in the item's block takes a global
//                  reduction.  At the end of the item every touched voxel is flushed with ONE coalesced
//                  REDG.ADD.F32x2 into the block's `acc` plane (what k_commit_tma folds into TSDF/W, :264-267).
//                  Once the items run out, its CTAs take the generic path - the exact one-reduction-per-sample march
//                  for what the binned path does not take: segments next to the volume boundary, rays with more than
//                  65535 steps, workspace overflow - zero the fill counters, and the last CTA clears the control block.
//
// Every kernel here is launched with programmatic dependent launch (ts_launch_pdl): its launch and prologue overlap its
// predecessor's tail, and it waits (cudaGridDependencySynchronize) where it first reads the predecessor's output.
//
// Sample value: ds = L - j*vs (the reference forms |P - x| * sign((P - x).m), :258-260, which equals it up to the
// f32 rounding of x: <= 3e-6 m on a 25 m map, tolerance 1e-4).
#include <cstdio>
#include <cstdlib>
#include <type_traits>
#include "tslam_internal.cuh"

#define FULL 0xffffffffu
#define MS_THREADS 256
// shared accumulator layout: word index = x*MB_SX + y*MB_SY + z (skewed strides: consecutive samples of a ray
// spread over the banks whatever its direction - 3.6-way average conflict vs 5.7 for x<<8|y<<4|z)
#define MB_SX 277
#define MB_SY 17
#define MB_WORDS (15 * MB_SX + 15 * MB_SY + 16)  // 4426
                                                // is applied with f32 global reductions instead
#define MB_SMEM (4 * MB_WORDS * 4)
#define SEG_CLS 16                               // length classes per block: (count - 1) >> 1
#define SEG_REP 4                                // counter replicas per (block, class), picked by the ray's group of 256
                                                // (seg_key): the hot blocks' counters would otherwise serialise in
                                                // one L2 slice
#define SEG_KEYS (SEG_CLS * SEG_REP)

// ---------------------------------------------------------------------------
// K2a: ray set-up (process_new_pcl :240-251), first stage of the counting walk: one bucket record -> unit direction,
// length, weight, step count n, occupy flag (:248) and the 32-byte ray record + aux word the march kernels read,
// stored at rays[r] / aux[r] and handed back in ra, rb, raux.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void ray_setup(const TsBatch& batch, const TsIntrin& in, const TsGrid& g, unsigned long long* btab, const TsBucket* buckets,
                                          unsigned long long* bidx, uint32_t bucket_shift, const TsBucketLaunch& bl, uint32_t id, uint32_t r,
                                          const TsMarchWs& w, unsigned int& my_rays, unsigned int& my_fmax, float4& ra, float4& rb, uint32_t& raux) {
  const float vs = in.vs;
  const uint32_t f = id >> bucket_shift;
  const TsBucketSums b = ts_read_bucket(buckets, bidx, bl, id);
  const TsFrame& fr = batch.f[f];
  struct { float ux, uy, uz, tx, ty, tz; int n, s; bool wide; } o;
  o.ux = o.uy = o.uz = o.tx = o.ty = o.tz = 0.0f;
  o.n = 0; o.s = fr.submap; o.wide = false;
  float L = 0.0f, wgt = 0.0f;
  if (b.cnt > 0) {  // :240
    my_rays++;
    TsRayGeom rg;
    if (ts_ray_geom(b, fr.T, in, rg)) {
      L = rg.L;
      o.ux = rg.ux; o.uy = rg.uy; o.uz = rg.uz;
      if (ts_in_bounds(g, rg.oi, rg.oj, rg.ok)) {  // occupy[sxyz_to_ijk(pos_p)] = 1 (:248)
        const int bx = rg.oi >> TS_BSHIFT, by = rg.oj >> TS_BSHIFT, bz = rg.ok >> TS_BSHIFT;
        const int blk = rm_lookup(g, btab, ts_pack_key(o.s, bx, by, bz), bx, by, bz);  // touched blocks are listed even when only `occupy` changed
        if (blk >= 0) g.occ[(size_t)blk * TS_B3 + ts_voxel_off(rg.oi, rg.oj, rg.ok)] = 1;
      }
      o.n = rg.n;
      wgt = rg.w;
      o.tx = (float)((double)fr.T[0] / (double)vs);
      o.ty = (float)((double)fr.T[1] / (double)vs);
      o.tz = (float)((double)fr.T[2] / (double)vs);
      // fixed-point scale of the launch: every |w| and |w*ds| must fit 31 bits (|ds| <= max(L, n*vs - L) + vs)
      const float dmax = fmaxf(L, (float)o.n * vs - L) + vs;
      const unsigned fb = __float_as_uint(fminf(fmaxf(wgt, wgt * dmax), 3.0e38f));  // non-negative floats order like their bits
      if (fb > my_fmax) my_fmax = fb;
      o.wide = o.n > 65535;
    }
  }
  ra = make_float4(o.ux, o.uy, o.uz, L);
  rb = make_float4(o.tx, o.ty, o.tz, wgt);
  raux = ((uint32_t)max(0, min(o.n, 65535)) << 16) | (f << 8) | (o.wide ? TS_AUX_WIDE : 0u);
  float4* dst = reinterpret_cast<float4*>(&w.rays[r]);
  dst[0] = ra;
  dst[1] = rb;
  w.aux[r] = raux;
}

// ---------------------------------------------------------------------------
// K2b: segment walks: 3-D DDA over the 16^3 blocks in voxel-index space, one lane per ray, warp-uniform loop (one
// block crossing per lane and iteration).  Segments are HINTS - every sample is re-checked exactly by the march
// kernel - so the crossing parameters may be off by one step.  The DDA runs twice per launch, in k_seg_count (count
// the segments per block and length class) and k_seg_scatter (store them in the runs k_seg_class_scan laid out): recomputing
// a segment costs a few FMAs per block crossing, storing it in a list and reading it back 24 bytes of traffic.
// ---------------------------------------------------------------------------
// 0 = far outside the volume (every sample is out of bounds), 1 = block inside the block range, 2 = outside but
// adjacent to it (a rounding-boundary sample may still be in bounds: exact path)
__device__ __forceinline__ int block_class(const TsGrid& g, int bx, int by, int bz) {
  const int b0 = (-g.hN) >> TS_BSHIFT, b1 = (g.N - g.hN - 1) >> TS_BSHIFT;
  const int z0 = (-g.hNz) >> TS_BSHIFT, z1 = (g.Nz - g.hNz - 1) >> TS_BSHIFT;
  if (bx >= b0 && bx <= b1 && by >= b0 && by <= b1 && bz >= z0 && bz <= z1) return 1;
  if (bx >= b0 - 1 && bx <= b1 + 1 && by >= b0 - 1 && by <= b1 + 1 && bz >= z0 - 1 && bz <= z1 + 1) return 2;
  return 0;
}
__device__ __forceinline__ void gen_append(const TsMarchWs& w, int* err, uint32_t ray, int j, int cnt) {
  const int p = atomicAdd(&w.ctl->n_gen, 1);
  if ((uint32_t)p < w.gen_cap) w.gen[p] = TsSeg{ray, ((uint32_t)j << 12) | (uint32_t)cnt};
  else atomicOr(err, TS_ERR_RAYLIST_FULL);
}
__device__ __forceinline__ void dda_axis(float u, float t, int& b, float& jc, float& dj, int& sg) {
  b = __float2int_rn(u + t) >> TS_BSHIFT;  // block of the first sample (j = 1)
  if (u > 0.0f) { jc = ((float)(16 * b + 16) - 0.5f - t) / u; dj = 16.0f / u; sg = 1; }
  else if (u < 0.0f) { jc = ((float)(16 * b) - 0.5f - t) / u; dj = -16.0f / u; sg = -1; }
  else { jc = 3.0e38f; dj = 0.0f; sg = 0; }
}

// A ray as both walks see it, decoded from its stored record (rays[r], aux[r]) - never from the set-up's registers -
// so that the two walks start from the same bits.  An all-zero record is a ray with n = 0.
struct SegRay { float ux, uy, uz, tx, ty, tz; int n, s; uint32_t f; bool wide; };
__device__ __forceinline__ SegRay seg_ray(const TsBatch& batch, float4 a, float4 b, uint32_t aux) {
  SegRay q;
  q.ux = a.x; q.uy = a.y; q.uz = a.z;
  q.tx = b.x; q.ty = b.y; q.tz = b.z;
  q.n = (int)(aux >> 16);
  q.f = (aux >> 8) & 255u;
  q.s = batch.f[q.f].submap;
  q.wide = (aux & TS_AUX_WIDE) != 0u;
  return q;
}

// The segment generator of both walks.  emit(cnt, j, bx, by, bz, cls) runs on EVERY lane of the warp once per
// iteration (the callers aggregate over the warp); cnt == 0: no segment on this lane this iteration.  A segment is
// steps j .. j+cnt-1 (cnt <= 32) of the ray in block (bx, by, bz), cls its block_class - 2 (generic path) for every
// segment of a wide ray.  Returns the first step not walked: <= n only when the iteration bound stopped the walk
// (non-finite pose).
template <class Emit>
__device__ __forceinline__ int seg_generate(const TsGrid& g, const SegRay& q, Emit&& emit) {
  int bx, by, bz, sx, sy, sz;
  float jx, jy, jz, dx, dy, dz;
  dda_axis(q.ux, q.tx, bx, jx, dx, sx);
  dda_axis(q.uy, q.ty, by, jy, dy, sy);
  dda_axis(q.uz, q.tz, bz, jz, dz, sz);
  // whole ray inside the block range (both end points are; the cells in between lie between them)?
  bool inside = false;
  if (q.n > 0) {
    const float nf = (float)q.n;
    const int ex = __float2int_rn(__fmaf_rn(q.ux, nf, q.tx)) >> TS_BSHIFT, ey = __float2int_rn(__fmaf_rn(q.uy, nf, q.ty)) >> TS_BSHIFT,
              ez = __float2int_rn(__fmaf_rn(q.uz, nf, q.tz)) >> TS_BSHIFT;
    inside = block_class(g, bx, by, bz) == 1 && block_class(g, ex, ey, ez) == 1;
  }
  int j = 1;
  const int max_iter = 3 * (q.n / 16 + 4);
  for (int it = 0;; ++it) {
    const bool act = j <= q.n && it < max_iter;
    if (!__any_sync(FULL, act)) break;
    int cnt = 0, jl = 0;
    if (act) {
      const float je = fminf(fminf(jx, jy), jz);
      jl = min((int)ceilf(je) - 1, q.n);  // last step strictly before the crossing
      if (jl >= j) cnt = min(jl - j + 1, 32);
    }
    const int cls = cnt == 0 ? 0 : q.wide ? 2 : inside ? 1 : block_class(g, bx, by, bz);
    emit(cnt, j, bx, by, bz, cls);
    j += cnt;
    if (act && j > jl) {  // the run up to the crossing is out: step into the next block
      if (jx <= jy && jx <= jz) { bx += sx; jx += dx; }
      else if (jy <= jz) { by += sy; jy += dy; }
      else { bz += sz; jz += dz; }
    }
  }
  return j;
}

// counter of a segment: (block, length class, replica).  The replica depends on the ray index alone (its group of 256
// rays), so both walks pick the same one, and groups walked at the same time spread a hot block over SEG_REP counters.
__device__ __forceinline__ int seg_key(int blk, int cnt, uint32_t r) {
  return (blk * SEG_CLS + ((cnt - 1) >> 1)) * SEG_REP + (int)((r >> 8) & (SEG_REP - 1));
}

// CTAs per SM of the two walks (tools/bench_march.py on an H100 SXM at 400 W: the counting walk 5-12 % faster with 3 than
// with 4 on S1-S4; the scattering walk with 6 as fast as with 4 on S1-S3 and 13 % faster on S4)
#define WC_MINB 3
#define WS_MINB 6

// K2b-1: counting walk.  Ray set-up, then the segments: activates their blocks (rm_lookup) and counts them per (block,
// class, replica).  Segments for the generic path (wide rays, blocks next to the volume, non-finite poses) are appended
// to `gen` here and only here; segments in blocks far outside the volume are counted out of bounds.
__global__ void __launch_bounds__(MS_THREADS, WC_MINB) k_seg_count(const __grid_constant__ TsBatch batch, TsIntrin in, TsGrid g, const TsBucket* buckets,
                                                                   unsigned long long* bidx, uint32_t bucket_shift, TsBucketLaunch bl,
                                                                   const uint32_t* __restrict__ ray_list,
                                                                   const int* __restrict__ n_rays_p, uint32_t ray_cap, TsMarchWs w, TsCounters* ctr,
                                                                   unsigned long long* prof) {
  __shared__ unsigned long long s_btab[RM_TAB];  // block coordinates -> pool index (direct mapped, rm_lookup)
  ts_stamp_begin(prof, TS_K_COUNT);
  for (int e = threadIdx.x; e < RM_TAB; e += MS_THREADS) s_btab[e] = TS_EMPTY;
  __syncthreads();
  cudaGridDependencySynchronize();  // the ray list and its buckets come from the bucket kernel
  const uint32_t nme = min((uint32_t)*n_rays_p, ray_cap);
  const uint32_t lane = threadIdx.x & 31u;
  unsigned int my_oob = 0, my_rays = 0, my_fmax = 0;
  for (uint32_t base = blockIdx.x * MS_THREADS; base < nme; base += gridDim.x * MS_THREADS) {
    const uint32_t r = base + threadIdx.x;
    float4 ra = make_float4(0.f, 0.f, 0.f, 0.f), rb = ra;
    uint32_t raux = 0u;
    if (r < nme) ray_setup(batch, in, g, s_btab, buckets, bidx, bucket_shift, bl, ray_list[r], r, w, my_rays, my_fmax, ra, rb, raux);
    const SegRay q = seg_ray(batch, ra, rb, raux);
    int j = seg_generate(g, q, [&](int cnt, int j0, int bx, int by, int bz, int cls) {
      int key = -1;
      if (cnt > 0) {
        if (cls == 2) gen_append(w, g.err, r, j0, cnt);
        else if (cls == 0) my_oob += (unsigned)cnt;
        else {
          const int blk = rm_lookup(g, s_btab, ts_pack_key(q.s, bx, by, bz), bx, by, bz);  // activates + marks the block dirty
          if (blk >= 0) key = seg_key(blk, cnt, r);  // (< 0: pool exhausted, the segment is dropped)
        }
      }
      const unsigned mrec = __ballot_sync(FULL, key >= 0);
      if (key >= 0) {
        const unsigned grp = __match_any_sync(mrec, key);
        if ((int)lane == __ffs(grp) - 1) red_add_u32((unsigned int*)&w.seg_count[key], (unsigned)__popc(grp));
      }
    });
    // non-finite pose: hand the rest to the exact path in bounded pieces
    while (j <= q.n) { const int c = min(q.n - j + 1, 4095); gen_append(w, g.err, r, j, c); j += c; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    my_oob += __shfl_xor_sync(FULL, my_oob, o);
    my_rays += __shfl_xor_sync(FULL, my_rays, o);
    my_fmax = max(my_fmax, __shfl_xor_sync(FULL, my_fmax, o));
  }
  if (lane == 0) {
    if (my_oob) atomicAdd(&ctr->n_oob, (unsigned long long)my_oob);
    if (my_rays) atomicAdd(&ctr->n_rays, (unsigned long long)my_rays);
    if (my_fmax) atomicMax(&w.ctl->fmax_bits, my_fmax);
  }
  // after the fmax reduction: k_seg_class_scan's scan reads fmax_bits, and what a kernel writes after its trigger is
  // not ordered before its dependent's cudaGridDependencySynchronize
  cudaTriggerProgrammaticLaunchCompletion();
  ts_stamp_end(prof, TS_K_COUNT);
}

// K2b-2: scattering walk.  The same generator over the same stored records, so the same binned segments in the same
// order per ray.  Each takes a slot of its range with a warp-aggregated returning atomic that counts seg_count[key] down
// from the count of the counting walk (k_seg_class_scan left it there): a group of n finding `left` slots still free takes
// the n slots from end - left on, in lane order, so a range fills from its start in the order the groups arrive.  Guards that
// never fire while the two walks agree route a segment to the generic path instead of writing outside its run, and are
// counted in n_seg_guard: a block that is not in the grid, a run that is already full.  A block whose activation failed
// (pool exhausted) was dropped by the counting walk: its segments are dropped here too.  When the launch overflowed
// (k_seg_class_scan), every binned segment takes the generic path.
__global__ void __launch_bounds__(MS_THREADS, WS_MINB) k_seg_scatter(const __grid_constant__ TsBatch batch, TsGrid g, const int* __restrict__ n_rays_p,
                                                                     uint32_t ray_cap, TsMarchWs w, TsCounters* ctr, unsigned long long* prof) {
  __shared__ unsigned long long s_btab[RM_TAB];  // block coordinates -> pool index (direct mapped, rm_find)
  ts_stamp_begin(prof, TS_K_SCATTER);
  for (int e = threadIdx.x; e < RM_TAB; e += MS_THREADS) s_btab[e] = TS_EMPTY;
  __syncthreads();
  cudaGridDependencySynchronize();  // the runs and the overflow flag come from k_seg_class_scan
  const uint32_t nme = min((uint32_t)*n_rays_p, ray_cap);
  const uint32_t lane = threadIdx.x & 31u;
  const bool overflow = w.ctl->overflow != 0;
  unsigned int my_guard = 0;
  for (uint32_t base = blockIdx.x * MS_THREADS; base < nme; base += gridDim.x * MS_THREADS) {
    const uint32_t r = base + threadIdx.x;
    float4 ra = make_float4(0.f, 0.f, 0.f, 0.f), rb = ra;
    uint32_t raux = 0u;
    if (r < nme) {
      const float4* src = reinterpret_cast<const float4*>(&w.rays[r]);
      ra = src[0]; rb = src[1];
      raux = w.aux[r];
    }
    const SegRay q = seg_ray(batch, ra, rb, raux);
    const uint32_t rj = q.f << 24;  // frame of the ray rides in the top byte of the segment word
    seg_generate(g, q, [&](int cnt, int j0, int bx, int by, int bz, int cls) {
      int key = -1, blk = -1;
      bool to_gen = false;
      if (cnt > 0 && cls == 1) {
        if (overflow) to_gen = true;
        else {
          blk = rm_find(g, s_btab, ts_pack_key(q.s, bx, by, bz), bx, by, bz);
          if (blk >= 0) key = seg_key(blk, cnt, r);
          else if (blk == -1) { to_gen = true; my_guard++; }  // guard: the counting walk activated every binned block
        }
      }
      const unsigned mrec = __ballot_sync(FULL, key >= 0);
      if (key >= 0) {
        const unsigned grp = __match_any_sync(mrec, key);
        const int leader = __ffs(grp) - 1;
        int left = 0;
        if ((int)lane == leader) left = atomicSub(&w.seg_count[key], __popc(grp));
        left = __shfl_sync(grp, left, leader);
        const int k = __popc(grp & ((1u << lane) - 1u));
        if (k < left) w.seg[w.seg_off[blk] + w.seg_rel[key] - (uint32_t)(left - k)] = TsSeg{r, rj | ((uint32_t)j0 << 8) | (uint32_t)cnt};
        else { to_gen = true; my_guard++; }  // guard: more segments than the counting walk counted
      }
      if (to_gen) gen_append(w, g.err, r, j0, cnt);
    });
  }
  cudaTriggerProgrammaticLaunchCompletion();
  for (int o = 16; o > 0; o >>= 1) my_guard += __shfl_xor_sync(FULL, my_guard, o);
  if (lane == 0 && my_guard) atomicAdd(&ctr->n_seg_guard, (unsigned long long)my_guard);
  ts_stamp_end(prof, TS_K_SCATTER);
}

// ---------------------------------------------------------------------------
// K2c: one kernel, two stages.  Grid-wide: per block with segments, class counts -> end of each (class, replica) range
// inside the block's run (seg_rel), list of touched blocks.  seg_count keeps the counts: k_seg_scatter counts each back
// down to 0 as it fills the range from its start (end - count).  Then the CTA that finishes last runs the scan over the
// touched blocks -> run offsets + work items (seg_scan): the scan needs every CTA's list entries, and a kernel boundary
// costs more than the few hundred blocks the class stage handles.
//
// The items are listed LONGEST FIRST (estimated samples, 32 bins): the persistent march kernel takes them in list order,
// so its tail is made of the cheapest items (with the items in block order, SMs idled through a long tail of the
// kernel's time).
// ---------------------------------------------------------------------------
#define SC_THREADS 1024
#define SC_BINS 32
__device__ __forceinline__ int item_bin(uint32_t cnt, uint32_t cost, uint32_t q, uint32_t nq) {
  // a block's run is ordered by segment length: chunk q of nq holds longer segments than chunk q-1 (ramp .5 .. 1.5)
  const uint32_t nseg = min((uint32_t)MR_CHUNK, cnt - q * MR_CHUNK);
  const float est = (float)nseg * ((float)cost / (float)cnt) * (0.5f + ((float)q + 0.5f) / (float)nq);
  return min(SC_BINS - 1, (int)(est * (1.0f / 4096.0f)));
}
// run by the last CTA alone; the class stage's list (touched, blk_total, blk_cost, n_touched) was written by other CTAs,
// so it is read through L2 (__ldcg), once: pass A keeps the first SC_THREADS entries (a few hundred on the bench's map)
// and their run offsets in shared memory, where the histogram and pass B find them without a dependent L2 round trip
// per 32 entries.
__device__ __forceinline__ void seg_scan(const TsMarchWs& w, TsCounters* ctr) {
  __shared__ uint32_t s_a[32];
  __shared__ uint32_t s_run;
  __shared__ unsigned int s_hist[SC_BINS], s_base[SC_BINS];
  __shared__ int s_ovf;
  __shared__ int s_tblk[SC_THREADS];
  __shared__ uint32_t s_tcnt[SC_THREADS], s_tcost[SC_THREADS], s_toff[SC_THREADS];
  const int nt = __ldcg(&w.ctl->n_touched);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  // entry i of the touched list: block, segments, cost, run offset
  auto entry = [&](int i, int& blk, uint32_t& cnt, uint32_t& cost, uint32_t& off) {
    if (i < SC_THREADS) { blk = s_tblk[i]; cnt = s_tcnt[i]; cost = s_tcost[i]; off = s_toff[i]; }
    else { blk = __ldcg(&w.touched[i]); cnt = __ldcg(&w.blk_total[i]); cost = __ldcg(&w.blk_cost[i]); off = __ldcg(&w.seg_off[blk]); }
  };
  if (threadIdx.x == 0) s_run = 0;
  if (threadIdx.x < SC_BINS) s_hist[threadIdx.x] = 0u;
  __syncthreads();
  // pass A: run offsets (exclusive scan of the blocks' segment counts), then the histogram of the items' estimated cost
  for (int base = 0; base < nt; base += SC_THREADS) {
    const int i = base + threadIdx.x;
    int blk = -1;
    uint32_t cnt = 0, cost = 0;
    if (i < nt) { blk = __ldcg(&w.touched[i]); cnt = __ldcg(&w.blk_total[i]); cost = __ldcg(&w.blk_cost[i]); }
    uint32_t a = cnt;  // inclusive warp scan
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t ta = __shfl_up_sync(FULL, a, o);
      if (lane >= o) a += ta;
    }
    if (lane == 31) s_a[wid] = a;
    __syncthreads();
    if (wid == 0) {
      uint32_t ta = s_a[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t ua = __shfl_up_sync(FULL, ta, o);
        if (lane >= o) ta += ua;
      }
      s_a[lane] = ta;  // inclusive over warps
    }
    __syncthreads();
    if (i < nt) {
      const uint32_t off = s_run + (wid ? s_a[wid - 1] : 0u) + a - cnt;
      w.seg_off[blk] = off;
      if (i < SC_THREADS) { s_tblk[i] = blk; s_tcnt[i] = cnt; s_tcost[i] = cost; s_toff[i] = off; }
    }
    __syncthreads();
    if (threadIdx.x == 0) s_run += s_a[31];
    __syncthreads();
  }
  for (int i = wid; i < nt; i += 32) {  // one warp per block, one lane per chunk: the busiest blocks have dozens of chunks
    int blk;
    uint32_t cnt, cost, off;
    entry(i, blk, cnt, cost, off);
    const uint32_t nq = (cnt + MR_CHUNK - 1) / MR_CHUNK;
    for (uint32_t q = lane; q < nq; q += 32) atomicAdd(&s_hist[item_bin(cnt, cost, q, nq)], 1u);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int tot_items = 0;
    for (int b = SC_BINS - 1; b >= 0; b--) { s_base[b] = tot_items; tot_items += s_hist[b]; s_hist[b] = 0u; }  // s_hist becomes the fill cursor
    const uint32_t tot = s_run;
    const bool ovf = tot > w.seg_cap || tot_items > w.item_cap;  // (tot <= seg_cap bounds the items below item_cap)
    s_ovf = ovf ? 1 : 0;
    w.ctl->total_segs = tot;
    w.ctl->overflow = ovf ? 1 : 0;
    w.ctl->n_full = 0;
    w.ctl->n_items = ovf ? 0 : (int)tot_items;
    // fixed-point scale: the largest k with fmax * 2^k < 2^30, clamped to [0, 48]
    const float fm = __uint_as_float(w.ctl->fmax_bits);
    int k = 30;
    if (fm > 0.0f) {
      int ex;
      frexpf(fm, &ex);  // fm = mant * 2^ex, mant in [0.5, 1)  ->  fm < 2^ex
      k = 30 - ex;
    }
    w.ctl->scale_k = max(0, min(48, k));
    atomicAdd(&ctr->n_segs, (unsigned long long)tot);
    atomicAdd(&ctr->n_items, (unsigned long long)(ovf ? 0u : tot_items));
  }
  __syncthreads();
  if (s_ovf) return;
  // pass B: the items, longest bin first
  for (int i = wid; i < nt; i += 32) {
    int blk;
    uint32_t cnt, cost, ex_seg;
    entry(i, blk, cnt, cost, ex_seg);
    const uint32_t nq = (cnt + MR_CHUNK - 1) / MR_CHUNK;
    for (uint32_t q = lane; q < nq; q += 32) {
      const int b = item_bin(cnt, cost, q, nq);
      const uint32_t pos = s_base[b] + atomicAdd(&s_hist[b], 1u);
      w.items[pos] = TsItem{blk, ex_seg + q * MR_CHUNK, min((uint32_t)MR_CHUNK, cnt - q * MR_CHUNK), 0u};
    }
  }
}
__global__ void __launch_bounds__(SC_THREADS, 1) k_seg_class_scan(TsGrid g, TsMarchWs w, TsCounters* ctr, unsigned long long* prof) {
  ts_stamp_begin(prof, TS_K_CLASS_SCAN);
  cudaGridDependencySynchronize();  // seg_count and the dirty flags come from k_seg_count
  const int nb = min(*g.n_blocks, g.max_blocks);
  const uint32_t lane = threadIdx.x & 31u;
  const int stride = gridDim.x * SC_THREADS;
  for (int b0 = blockIdx.x * SC_THREADS; b0 < nb; b0 += stride) {
    const int b = b0 + (int)threadIdx.x;
    unsigned tot = 0, cost = 0;  // segments / samples (upper estimate: class q holds segments of 2q+1 or 2q+2 steps)
    if (b < nb && g.dirty_flag[b]) {
      uint4* c4 = reinterpret_cast<uint4*>(&w.seg_count[(size_t)b * SEG_KEYS]);
      uint4* r4 = reinterpret_cast<uint4*>(&w.seg_rel[(size_t)b * SEG_KEYS]);
#pragma unroll 4
      for (int q = 0; q < SEG_KEYS / 4; q++) {
        const uint4 c = c4[q];
        if ((c.x | c.y | c.z | c.w) == 0u) { continue; }
        tot += c.x + c.y + c.z + c.w;
        r4[q] = make_uint4(tot - c.y - c.z - c.w, tot - c.z - c.w, tot - c.w, tot);  // ends of the ranges
        cost += (c.x + c.y + c.z + c.w) * (unsigned)(2 * (q / (SEG_REP / 4)) + 2);
      }
    }
    const unsigned mt = __ballot_sync(FULL, tot > 0u);
    if (mt) {
      const int leader = __ffs(mt) - 1;
      int p0 = 0;
      if ((int)lane == leader) p0 = atomicAdd(&w.ctl->n_touched, __popc(mt));
      p0 = __shfl_sync(FULL, p0, leader);
      if (tot > 0u) {
        const int p = p0 + __popc(mt & ((1u << lane) - 1u));
        w.touched[p] = b;
        w.blk_total[p] = tot;
        w.blk_cost[p] = cost;
      }
    }
  }
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = atomicAdd(&w.ctl->ticket_scan, 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  seg_scan(w, ctr);
  ts_stamp_end(prof, TS_K_CLASS_SCAN);  // the last CTA ends the kernel
}

// ---------------------------------------------------------------------------
// exact sample index, as the reference states it (:253-254)
// ---------------------------------------------------------------------------
__device__ __forceinline__ void exact_index(float ux, float uy, float uz, const float* T, int j, float vs, float rvs, int& xi, int& yi, int& zi) {
  const float jf = (float)j;
  const float x = (ux * jf) * vs + T[0], y = (uy * jf) * vs + T[1], z = (uz * jf) * vs + T[2];
  xi = iroundf(div_vs(x, vs, rvs));
  yi = iroundf(div_vs(y, vs, rvs));
  zi = iroundf(div_vs(z, vs, rvs));
}

// one sample through the global path: bounds, block lookup (activating), one reduction
__device__ __forceinline__ void global_sample(const TsGrid& g, int s, int xi, int yi, int zi, float a, float wgt, unsigned int& upd,
                                              unsigned int& oob) {
  if ((unsigned)(xi + g.hN) < (unsigned)g.N && (unsigned)(yi + g.hN) < (unsigned)g.N && (unsigned)(zi + g.hNz) < (unsigned)g.Nz) {
    const int blk = ts_get_or_alloc_cached(g, ts_pack_key(s, xi >> TS_BSHIFT, yi >> TS_BSHIFT, zi >> TS_BSHIFT));
    if (blk >= 0) {
      ts_mark_dirty(g, blk);
      red_add_f32x2(&g.acc[(size_t)blk * TS_B3 + ts_voxel_off(xi, yi, zi)], a, wgt);
      upd++;
    }
  } else {
    oob++;
  }
}

// ---------------------------------------------------------------------------
// K2f: the march proper.  Persistent CTAs, one work item (block, <= MR_CHUNK segments) at a time.
//
// A block's run is ordered by segment length (k_seg_scatter), so the 32 segments a warp takes - ONE PER LANE, ray
// parameters in registers - have (nearly) equal length and are walked in lock step.  Lane l starts at step
// (7*l mod cnt) of its segment and wraps around: neighbouring rays are nearly parallel, so with every lane at a
// different depth the 32 shared-memory atomics of a step hit 32 different voxels (same-step marching puts 4-16 rays
// into one voxel half way to the surface: serialised atomics).
//
// Shared accumulators per voxel: two 64-bit sums (A = sum w*ds, B = sum w, units 2^-scale_k) kept as
//   lo  = sum x      mod 2^32
//   hi' = sum (x >> 16)            (arithmetic shift)
// Both are plain no-return ATOMS.ADD - no carry logic, no dependent read of the old value.  With fewer than 2^16
// samples per voxel and item (MR_CHUNK segments x <= 2 samples of a ray in one voxel) the true sum S is the unique
// value with S = lo (mod 2^32) in [hi' * 2^16, hi' * 2^16 + 2^32):  S = hi' * 2^16 + ((lo - (hi' << 16)) mod 2^32).
// ---------------------------------------------------------------------------
__device__ __forceinline__ double mb_sum(unsigned int lo, int hi) {
  return (double)((long long)hi * 65536ll + (long long)(unsigned int)(lo - ((unsigned int)hi << 16)));
}

template <bool VERIFY, int MB_THREADS, int MB_MINB>
__global__ void __launch_bounds__(MB_THREADS, MB_MINB) k_march_blocks(const __grid_constant__ TsBatch batch, TsIntrin in, TsGrid g, TsMarchWs w,
                                                                 TsCounters* ctr, int* n_rays, unsigned long long* prof) {
  ts_stamp_begin(prof, TS_K_MARCH);
  extern __shared__ __align__(16) unsigned int mb_smem[];
  unsigned int* const a_lo = mb_smem;
  int* const a_hi = (int*)(mb_smem + MB_WORDS);
  unsigned int* const b_lo = mb_smem + 2 * MB_WORDS;
  int* const b_hi = (int*)(mb_smem + 3 * MB_WORDS);
  __shared__ int s_item;
  const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  const float vs = in.vs, rvs = in.rvs, eps_hi = 0.5f - w.near_eps;
  for (int e = threadIdx.x; e < 4 * MB_WORDS; e += MB_THREADS) mb_smem[e] = 0u;
  cudaGridDependencySynchronize();  // the items, segments and control block come from k_seg_scatter and before
  const int scale_k = w.ctl->scale_k;
  const float fix = __uint_as_float((unsigned)(127 + scale_k) << 23);   // 2^k
  const double unfix = 1.0 / (double)fix;
  unsigned int my_upd = 0, my_oob = 0, my_slow = 0, my_fb = 0, my_bad = 0;
  const int n_items = w.ctl->n_items;
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) s_item = atomicAdd(&w.ctl->item_cursor, 1);
    __syncthreads();
    const int it = s_item;
    if (it >= n_items) break;
    const TsItem item = w.items[it];  // longest first (k_seg_class_scan)
    int sm, kx, ky, kz;
    ts_unpack_key(g.block_key[item.blk], sm, kx, ky, kz);
    const int ox = kx << TS_BSHIFT, oy = ky << TS_BSHIFT, oz = kz << TS_BSHIFT;
    const float fox = (float)ox, foy = (float)oy, foz = (float)oz;
    // blocks cut by the volume boundary (N not a multiple of 16) need the per-sample bounds test
    const bool partial = ox < -g.hN || ox + TS_B > g.N - g.hN || oy < -g.hN || oy + TS_B > g.N - g.hN || oz < -g.hNz || oz + TS_B > g.Nz - g.hNz;
    const int nseg = (int)item.nseg;
    const TsSeg* const segs = w.seg + item.seg0;
    // ---- 32 segments per warp, one per lane; the next batch's records are fetched while this one is marched ----
    TsSeg nx = TsSeg{0u, 0u};
    float4 na = make_float4(0.f, 0.f, 0.f, 0.f), nb = na;
    {
      const int i0 = (int)wid * 32 + (int)lane;
      if (i0 < nseg) {
        nx = segs[i0];
        const float4* src = reinterpret_cast<const float4*>(&w.rays[nx.ray]);
        na = __ldg(src); nb = __ldg(src + 1);
      }
    }
    constexpr int MB_WARPS = MB_THREADS / 32;
    for (int sb = (int)wid * 32; sb < nseg; sb += MB_WARPS * 32) {
      const TsSeg sg = nx;
      const float4 a = na, b = nb;
      {
        const int i1 = sb + MB_WARPS * 32 + (int)lane;
        nx = TsSeg{0u, 0u};
        if (i1 < nseg) {
          nx = segs[i1];
          const float4* src = reinterpret_cast<const float4*>(&w.rays[nx.ray]);
          na = __ldg(src); nb = __ldg(src + 1);
        }
      }
      const int cnt = (int)(sg.jc & 255u);  // 0 for lanes past the end of the item
      const int j0 = (int)((sg.jc >> 8) & 0xFFFFu);
      const uint32_t frame = sg.jc >> 24;
      const int maxc = __reduce_max_sync(FULL, cnt);
      const float jf = (float)j0;
      const float ux = a.x, uy = a.y, uz = a.z;
      // first sample of the segment in block-local voxel units: one rounding at magnitude <= ~20
      const float x0 = __fmaf_rn(a.x, jf, b.x - fox), y0 = __fmaf_rn(a.y, jf, b.y - foy), z0 = __fmaf_rn(a.z, jf, b.z - foz);
      const float L0 = __fmaf_rn(-jf, vs, a.w);
      const float wf = b.w * fix;  // w in fixed-point units (exact: power of two)
      const int wq = __float2int_rn(wf);
      const int wqh = wq >> 16;
      // weight far below the launch's largest (f32 reductions keep its relative precision), blocks cut by the volume
      // boundary, VERIFY: every sample of the segment takes the exact path below
      const bool all_slow = wq < MB_MIN_WQ || partial || VERIFY;
      const float cntf = (float)cnt;
      int k0 = 0;
      if (cnt > 1) k0 = (int)(lane * 7u) % cnt;  // staggered start
      float kf = (float)k0;
      my_upd += (unsigned)cnt;
      // ---- fast loop: branch-free.  Iteration i of a lane handles step (k0 + i) mod cnt of its segment.  A sample
      // whose rounding is not certain (|fraction - .5| < near_eps) or whose voxel is not in this block only sets bit i
      // of slow_mask; those are redone exactly after the loop.
      unsigned slow_mask = 0u;
      if (all_slow) slow_mask = cnt >= 32 ? 0xffffffffu : ((1u << cnt) - 1u);
      else {
        for (int i = 0; i < maxc; ++i) {
          const float gx = __fmaf_rn(ux, kf, x0), gy = __fmaf_rn(uy, kf, y0), gz = __fmaf_rn(uz, kf, z0);
          // round to nearest + distance of the fraction from .5 (magic-number rounding: |g| < 2^22): the low mantissa
          // bits of t hold the block-local voxel coordinate
          const float tx = gx + 12582912.0f, ty = gy + 12582912.0f, tz = gz + 12582912.0f;
          const float rx = gx - (tx - 12582912.0f), ry = gy - (ty - 12582912.0f), rz = gz - (tz - 12582912.0f);
          const unsigned qx = __float_as_uint(tx), qy = __float_as_uint(ty), qz = __float_as_uint(tz);
          const bool inb = ((qx | qy | qz) - 0x4B400000u) <= 15u;  // all three coordinates in [0, 16)
          const bool sure = fmaxf(fmaxf(fabsf(rx), fabsf(ry)), fabsf(rz)) <= eps_hi;
          const bool pred = i < cnt;
          const float avq = __fmaf_rn(-kf, vs, L0) * wf;  // w * ds, ds = L - j*vs (:258-264), in fixed-point units
          if (pred && inb && sure) {
            const unsigned e = qx * (unsigned)MB_SX + qy * (unsigned)MB_SY + qz - 0x4B400000u * (unsigned)(MB_SX + MB_SY + 1);
            const int xq = __float2int_rn(avq);
            atomicAdd(&a_lo[e], (unsigned int)xq);
            atomicAdd(&a_hi[e], xq >> 16);
            atomicAdd(&b_lo[e], (unsigned int)wq);
            atomicAdd(&b_hi[e], wqh);
          } else if (pred) {
            slow_mask |= 1u << i;
          }
          kf += 1.0f;
          if (kf >= cntf) kf = 0.0f;
        }
      }
      // ---- exact path (:253-254) for the flagged samples; a sample that really lies in another block, is out of
      // bounds or carries a tiny weight goes through the global path
      if (__any_sync(FULL, slow_mask != 0u)) {
        const bool tiny = wq < MB_MIN_WQ;
        while (slow_mask) {
          const int i = __ffs(slow_mask) - 1;
          slow_mask &= slow_mask - 1u;
          int k = k0 + i;
          if (k >= cnt) k -= cnt;
          const float kk = (float)k;
          const float avq = __fmaf_rn(-kk, vs, L0) * wf;
          int xi, yi, zi;
          exact_index(ux, uy, uz, batch.f[frame].T, j0 + k, vs, rvs, xi, yi, zi);
          const int lx = xi - ox, ly = yi - oy, lz = zi - oz;
          if (VERIFY || !all_slow) {
            const float gx = __fmaf_rn(ux, kk, x0), gy = __fmaf_rn(uy, kk, y0), gz = __fmaf_rn(uz, kk, z0);
            const float tx = gx + 12582912.0f, ty = gy + 12582912.0f, tz = gz + 12582912.0f;
            const float rx = gx - (tx - 12582912.0f), ry = gy - (ty - 12582912.0f), rz = gz - (tz - 12582912.0f);
            const bool near = fmaxf(fmaxf(fabsf(rx), fabsf(ry)), fabsf(rz)) > eps_hi;
            if (near) my_slow++;
            if (VERIFY && !near && (lx != __float_as_int(tx) - 0x4B400000 || ly != __float_as_int(ty) - 0x4B400000 || lz != __float_as_int(tz) - 0x4B400000)) my_bad++;
          }
          bool local = !tiny && ((unsigned)(lx | ly | lz)) <= 15u;
          if (!local) my_fb++;
          if (local && partial &&
              !((unsigned)(xi + g.hN) < (unsigned)g.N && (unsigned)(yi + g.hN) < (unsigned)g.N && (unsigned)(zi + g.hNz) < (unsigned)g.Nz)) {
            local = false;  // global_sample counts it as out of bounds
          }
          if (local) {
            const int e = lx * MB_SX + ly * MB_SY + lz;
            const int xq = __float2int_rn(avq);
            atomicAdd(&a_lo[e], (unsigned int)xq);
            atomicAdd(&a_hi[e], xq >> 16);
            atomicAdd(&b_lo[e], (unsigned int)wq);
            atomicAdd(&b_hi[e], wqh);
          } else {
            my_upd--;
            global_sample(g, sm, xi, yi, zi, (float)((double)avq * unfix), (float)((double)wf * unfix), my_upd, my_oob);
          }
        }
      }
    }
    __syncthreads();
    // ---- flush: one coalesced reduction per touched voxel, accumulators back to zero ----
    float2* const acc = g.acc + (size_t)item.blk * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += MB_THREADS) {
      const int e = (v >> 8) * MB_SX + ((v >> 4) & 15) * MB_SY + (v & 15);
      const unsigned int blo = b_lo[e];
      const int bhi = b_hi[e];
      if (blo == 0u && bhi == 0) continue;  // sum w > 0 for every touched voxel
      const unsigned int alo = a_lo[e];
      const int ahi = a_hi[e];
      a_lo[e] = 0u; a_hi[e] = 0; b_lo[e] = 0u; b_hi[e] = 0;
      red_add_f32x2(&acc[v], (float)(mb_sum(alo, ahi) * unfix), (float)(mb_sum(blo, bhi) * unfix));
    }
  }
  // ---- tail of the launch, once the item cursor has run out: the generic path, the fill counters, the control block ----
  // generic path: exact index and one global reduction per sample, for the segments k_seg_count and k_seg_scatter listed
  // (next to the volume boundary, over-long rays, overflow), MB_THREADS records per claim
  const int n_gen = min(w.ctl->n_gen, (int)w.gen_cap);
  unsigned int my_gen = 0;
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) s_item = atomicAdd(&w.ctl->gen_cursor, MB_THREADS);
    __syncthreads();
    const int i = s_item + (int)threadIdx.x;
    if (s_item >= n_gen) break;
    if (i < n_gen) {
      const TsSeg sg = w.gen[i];
      const float4* src = reinterpret_cast<const float4*>(&w.rays[sg.ray]);
      const float4 a = src[0], b = src[1];
      const TsFrame& fr = batch.f[(w.aux[sg.ray] >> 8) & 255u];
      const int j0 = (int)(sg.jc >> 12), cnt = (int)(sg.jc & 4095u);
      for (int q = 0; q < cnt; q++) {
        const int j = j0 + q;
        int xi, yi, zi;
        exact_index(a.x, a.y, a.z, fr.T, j, vs, rvs, xi, yi, zi);
        const float ds = __fmaf_rn(-(float)j, vs, a.w);
        global_sample(g, fr.submap, xi, yi, zi, b.w * ds, b.w, my_upd, my_oob);
        my_gen++;
      }
    }
  }
  // No early trigger (cudaTriggerProgrammaticLaunchCompletion) in this kernel: what its tail writes - seg_count back to
  // zero, the cleared control block and ray count - is read by the next launch's bucket kernel and counting walk, which
  // reach this grid through a chain of programmatic launches (k_collect_dirty, k_commit_tma, k_bucket_depth), and a
  // write after a trigger is not ordered before the dependent's cudaGridDependencySynchronize.
  // fill counters back to zero.  k_seg_scatter counted every run down to 0 unless the launch overflowed; a count left
  // above 0 is a slot of a run that no segment filled (n_seg_guard, must stay 0)
  unsigned int my_left = 0;
  {
    const int nt = w.ctl->n_touched;
    const bool check = w.ctl->overflow == 0;
    for (int q = blockIdx.x * MB_THREADS + threadIdx.x; q < nt * (SEG_KEYS / 4); q += gridDim.x * MB_THREADS) {
      int4* c4 = reinterpret_cast<int4*>(w.seg_count + (size_t)w.touched[q / (SEG_KEYS / 4)] * SEG_KEYS) + q % (SEG_KEYS / 4);
      if (check) {
        const int4 c = *c4;
        my_left += (unsigned)(max(c.x, 0) + max(c.y, 0) + max(c.z, 0) + max(c.w, 0));
      }
      *c4 = make_int4(0, 0, 0, 0);
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    my_upd += __shfl_xor_sync(FULL, my_upd, o);
    my_oob += __shfl_xor_sync(FULL, my_oob, o);
    my_slow += __shfl_xor_sync(FULL, my_slow, o);
    my_fb += __shfl_xor_sync(FULL, my_fb, o);
    my_bad += __shfl_xor_sync(FULL, my_bad, o);
    my_gen += __shfl_xor_sync(FULL, my_gen, o);
    my_left += __shfl_xor_sync(FULL, my_left, o);
  }
  // one global reduction per CTA and counter (same-address atomics serialise in L2)
  __shared__ unsigned int s_stat[7];
  __shared__ int s_last;
  if (threadIdx.x < 7) s_stat[threadIdx.x] = 0u;
  __syncthreads();
  if (lane == 0) {
    if (my_upd) atomicAdd(&s_stat[0], my_upd);
    if (my_oob) atomicAdd(&s_stat[1], my_oob);
    if (my_slow) atomicAdd(&s_stat[2], my_slow);
    if (my_fb) atomicAdd(&s_stat[3], my_fb);
    if (my_bad) atomicAdd(&s_stat[4], my_bad);
    if (my_gen) atomicAdd(&s_stat[5], my_gen);
    if (my_left) atomicAdd(&s_stat[6], my_left);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_stat[0]) atomicAdd(&ctr->n_updates, (unsigned long long)s_stat[0]);
    if (s_stat[1]) atomicAdd(&ctr->n_oob, (unsigned long long)s_stat[1]);
    if (s_stat[2]) atomicAdd(&ctr->n_slow, (unsigned long long)s_stat[2]);
    if (s_stat[3]) atomicAdd(&ctr->n_fallback, (unsigned long long)s_stat[3]);
    if (s_stat[4]) atomicAdd(&ctr->n_verify_bad, (unsigned long long)s_stat[4]);
    if (s_stat[5]) atomicAdd(&ctr->n_generic, (unsigned long long)s_stat[5]);
    if (s_stat[6]) atomicAdd(&ctr->n_seg_guard, (unsigned long long)s_stat[6]);
    __threadfence();
    s_last = atomicAdd(&w.ctl->ticket, 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  // the last CTA to finish (every other one is past its last read of the control block) clears it and the ray count
  // of the launch
  if (s_last) {
    if (threadIdx.x < sizeof(TsMarchCtl) / 4) reinterpret_cast<int*>(w.ctl)[threadIdx.x] = 0;
    if (threadIdx.x == 0) {
      *n_rays = 0;
      ts_stamp_end_thread(prof, TS_K_MARCH);
    }
  }
}

// ---------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------
int ts_march_alloc(tslam_tsdf* m) {
  TsMarchWs& w = m->mw;
  const size_t nr = m->ray_list_cap;
  const size_t nb = (size_t)m->g.max_blocks;
  TS_CUDA(cudaMalloc(&w.rays, nr * sizeof(TsRay)));
  TS_CUDA(cudaMalloc(&w.aux, nr * 4));
  size_t sc = nr * 16;  // ~8 segments per 90-step ray on the bench stream, 15 on 8 m rays
  if (sc < (8u << 20)) sc = 8u << 20;
  if (sc > (128u << 20)) sc = 128u << 20;
  const char* e = getenv("TSLAM_SEG_CAP");  // tests: force the overflow path
  if (e && atoll(e) > 0) sc = (size_t)atoll(e);
  w.seg_cap = (uint32_t)sc;
  TS_CUDA(cudaMalloc(&w.seg, sc * sizeof(TsSeg)));
  TS_CUDA(cudaMalloc(&w.seg_count, nb * SEG_KEYS * 4));
  TS_CUDA(cudaMemset(w.seg_count, 0, nb * SEG_KEYS * 4));
  TS_CUDA(cudaMalloc(&w.seg_rel, nb * SEG_KEYS * 4));
  TS_CUDA(cudaMalloc(&w.seg_off, nb * 4));
  TS_CUDA(cudaMalloc(&w.touched, nb * 4));
  TS_CUDA(cudaMalloc(&w.blk_total, nb * 4));
  TS_CUDA(cudaMalloc(&w.blk_cost, nb * 4));
  w.item_cap = (uint32_t)(sc / MR_CHUNK + nb + 16);
  TS_CUDA(cudaMalloc(&w.items, (size_t)w.item_cap * sizeof(TsItem)));
  w.gen_cap = (uint32_t)(nr > (1u << 20) ? nr : (1u << 20));
  TS_CUDA(cudaMalloc(&w.gen, (size_t)w.gen_cap * sizeof(TsSeg)));
  TS_CUDA(cudaMalloc(&w.ctl, sizeof(TsMarchCtl)));
  TS_CUDA(cudaMemset(w.ctl, 0, sizeof(TsMarchCtl)));
  // |fast index - exact index| bound in voxel units (DESIGN.md "exact indices from a one-FMA fast path"):
  // 2^-24 * (4*max_steps + 2*|T/vs|) for the reference's own rounding chain + 2^-24 * (|T/vs| + max_steps + 100)
  // for ours, with |T/vs| <= N; doubled.
  const double ms = m->cfg.max_ray_length / m->cfg.voxel_scale;
  const double nmax = m->cfg.N > m->cfg.Nz ? m->cfg.N : m->cfg.Nz;
  double eps = 2.0 * 5.9604644775390625e-8 * (5.0 * ms + 3.0 * nmax + 100.0);
  if (eps < 1e-5) eps = 1e-5;
  if (eps > 0.25) eps = 1.0;  // absurd geometry: every sample takes the exact path
  const char* ee = getenv("TSLAM_NEAR_EPS");
  if (ee) eps = atof(ee);
  w.near_eps = (float)eps;
  TS_CUDA(cudaFuncSetAttribute(k_march_blocks<false, 320, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, MB_SMEM));
  TS_CUDA(cudaFuncSetAttribute(k_march_blocks<true, 320, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, MB_SMEM));
  return TSLAM_OK;
}

void ts_march_free(tslam_tsdf* m) {
  TsMarchWs& w = m->mw;
  cudaFree(w.rays); cudaFree(w.aux); cudaFree(w.seg); cudaFree(w.seg_count); cudaFree(w.seg_rel); cudaFree(w.seg_off); cudaFree(w.touched);
  cudaFree(w.blk_total); cudaFree(w.blk_cost); cudaFree(w.items); cudaFree(w.gen); cudaFree(w.ctl);
}

// prof (profiling, may be null): the launch's row of kernel stamps.  Every kernel is launched with programmatic dependent
// launch: each waits (cudaGridDependencySynchronize) only where it first reads its predecessor's output, so its launch
// and prologue overlap the predecessor's tail.
int ts_march_launch(tslam_tsdf* m, cudaStream_t st, const TsBatch& batch, uint32_t bucket_shift, const TsBucketLaunch& bl, unsigned long long* prof) {
  if (!m->mw.rays) { int rca = ts_march_alloc(m); if (rca) return rca; }  // the workspace, at the first launch that needs it
  const int sms = m->sm_count;
  TS_CUDA(ts_launch_pdl(k_seg_count, sms * WC_MINB, MS_THREADS, 0, st, batch, m->in, m->g, (const TsBucket*)m->buckets, m->bidx, bucket_shift, bl,
                        (const uint32_t*)m->ray_list, (const int*)m->n_rays, (uint32_t)m->ray_list_cap, m->mw, m->counters, prof));
  TS_LAUNCH_CHECK(m);
  const int nsc = (m->g.max_blocks + SC_THREADS - 1) / SC_THREADS;
  TS_CUDA(ts_launch_pdl(k_seg_class_scan, nsc < sms ? nsc : sms, SC_THREADS, 0, st, m->g, m->mw, m->counters, prof));
  TS_LAUNCH_CHECK(m);
  TS_CUDA(ts_launch_pdl(k_seg_scatter, sms * WS_MINB, MS_THREADS, 0, st, batch, m->g, (const int*)m->n_rays, (uint32_t)m->ray_list_cap, m->mw,
                        m->counters, prof));
  TS_LAUNCH_CHECK(m);
  const int grid = (sms - m->rm_reserve) * 3;
  if (m->march_verify) TS_CUDA(ts_launch_pdl(k_march_blocks<true, 320, 3>, grid, 320, MB_SMEM, st, batch, m->in, m->g, m->mw, m->counters, m->n_rays, prof));
  else TS_CUDA(ts_launch_pdl(k_march_blocks<false, 320, 3>, grid, 320, MB_SMEM, st, batch, m->in, m->g, m->mw, m->counters, m->n_rays, prof));
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
