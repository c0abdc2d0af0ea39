// libtslam.so - Octomap: per-voxel hit counter on a hash grid of 8^3 u32 blocks.
// Reference: taichi_slam/mapping/taichi_octomap.py.  The reference "Octomap" has no
// log-odds / ray casting: occupy[ijk] += 1 per point (:116-119) and a threshold
// test (:86-88); counts are exact integers, compared bit-for-bit with the oracle.
#include <cstring>
#include <string>
#include "tslam_internal.cuh"
#include "tslam_fuse_plan.cuh"

__device__ __forceinline__ int oc_iroundf(float x) { return (int)roundf(x); }

// cw != 0: colour word of the hit (textured maps): color[ijk] = rgb (:120-124), largest word wins
__device__ __forceinline__ void oc_hit(const OcGrid& g, int s, int i, int j, int k, unsigned int add, unsigned long long cw = 0ull) {
  if (!ts_in_bounds(g, i, j, k)) return;
  const int blk = ts_get_or_alloc(g, ts_pack_key(s, i >> OC_BSHIFT, j >> OC_BSHIFT, k >> OC_BSHIFT));
  if (blk < 0) return;
  const size_t o = (size_t)blk * OC_B3 + oc_voxel_off(i, j, k);
  atomicAdd(&g.cnt[o], add);  // occupy[ijk] += 1 (:119)
  if (cw) ts_red_max_u64(&g.cw[o], cw);
}
// "Stupid OpenCV is BGR" (:121): colour channel 0 <- rgb[2], 2 <- rgb[0]
__device__ __forceinline__ unsigned long long oc_color_word(unsigned int seq, const uint8_t* p) {
  return ((unsigned long long)seq << 24) | ((unsigned long long)p[2] << 16) | ((unsigned long long)p[1] << 8) | (unsigned long long)p[0];
}
__device__ __forceinline__ void oc_word_to_rgb(unsigned long long w, float* out) {
  out[0] = (float)((w >> 16) & 255) / 255.0f; out[1] = (float)((w >> 8) & 255) / 255.0f; out[2] = (float)(w & 255) / 255.0f;
}

// recast_pcl_to_map_kernel (taichi_octomap.py:134-145)
__global__ void __launch_bounds__(256) k_octo_points(OcGrid g, const float* __restrict__ xyz, int n, TsFrame fr, float vs,
                                                      const uint8_t* __restrict__ rgb) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float x = xyz[3 * (size_t)t], y = xyz[3 * (size_t)t + 1], z = xyz[3 * (size_t)t + 2];
  const float px = ((fr.R[0] * x + fr.R[1] * y) + fr.R[2] * z) + fr.T[0];  // :141
  const float py = ((fr.R[3] * x + fr.R[4] * y) + fr.R[5] * z) + fr.T[1];
  const float pz = ((fr.R[6] * x + fr.R[7] * y) + fr.R[8] * z) + fr.T[2];
  const unsigned long long cw = rgb ? oc_color_word(fr.seq, rgb + 3 * (size_t)t) : 0ull;
  oc_hit(g, fr.submap, oc_iroundf(px / vs), oc_iroundf(py / vs), oc_iroundf(pz / vs), 1u, cw);  // xyz_to_sijk mapping_common.py:251-255
}

// recast_depth_to_map_kernel (taichi_octomap.py:147-169)
__global__ void __launch_bounds__(256) k_octo_depth(OcGrid g, const uint16_t* __restrict__ depth, int h, int w, int hh, int ww,
                                                     TsFrame fr, TsIntrin in, const uint8_t* __restrict__ tex, int th, int tw) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= hh * ww) return;
  const int jj = t / ww, ii = t - jj * ww;
  const int j = jj * in.step, i = ii * in.step;
  const uint16_t d = depth[(size_t)j * w + i];
  const float df = (float)d;
  if (d == 0 || df > in.dmax_mm || df < in.dmin_mm) return;  // :155
  const float dep = df / 1000.0f;                              // :157
  const float x = ((float)i - in.cx) * dep / in.fx;
  const float y = ((float)j - in.cy) * dep / in.fy;
  const float px = ((fr.R[0] * x + fr.R[1] * y) + fr.R[2] * dep) + fr.T[0];  // :159
  const float py = ((fr.R[3] * x + fr.R[4] * y) + fr.R[5] * dep) + fr.T[1];
  const float pz = ((fr.R[6] * x + fr.R[7] * y) + fr.R[8] * dep) + fr.T[2];
  unsigned long long cw = 0ull;
  if (tex) {  // :160-167
    int ti, tj;
    const uint8_t zero3[3] = {0, 0, 0};
    cw = oc_color_word(fr.seq, ts_color_pixel(in, i, j, th, tw, ti, tj) ? tex + ((size_t)tj * tw + ti) * 3 : zero3);
  }
  oc_hit(g, fr.submap, oc_iroundf(px / in.vs), oc_iroundf(py / in.vs), oc_iroundf(pz / in.vs), 1u, cw);
}

// the voxels of submap `submap` the rule keeps (OcHits: a hit, OcLogodds: known), with their count (OcLogodds: L)
template <class Rule>
__global__ void __launch_bounds__(256) k_octo_gather(OcGrid g, int submap, long long cap, int32_t* idx, unsigned int* count,
                                                      float* color, unsigned long long* counter) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  const long long total = (long long)nb * OC_B3;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long iters = (total + stride - 1) / stride;
  for (long long it = 0; it < iters; ++it) {  // uniform trip count: the warp ballot below needs all lanes
    const long long e = it * stride + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool want = false;
    unsigned int c = 0;
    int s = 0, bx = 0, by = 0, bz = 0, v = 0;
    if (e < total) {
      const int b = (int)(e >> 9);
      v = (int)(e & 511);
      ts_unpack_key(g.block_key[b], s, bx, by, bz);
      c = g.cnt[e];
      want = (s == submap) && Rule::gather_keep(c);
    }
    const long long row = warp_append_u64(want, counter);
    if (want && row < cap) {
      idx[3 * row] = bx * OC_B + (v >> 6);
      idx[3 * row + 1] = by * OC_B + ((v >> 3) & 7);
      idx[3 * row + 2] = bz * OC_B + (v & 7);
      count[row] = Rule::gather_val(c);
      if (color) {
        if (g.cw) oc_word_to_rgb(g.cw[e], color + 3 * row);
        else color[3 * row] = color[3 * row + 1] = color[3 * row + 2] = 0.0f;
      }
    }
  }
}

// cvt_occupy_to_voxels(level) / cvt_occupy_voxels_to (taichi_octomap.py:90-114).
// occupy.parent(level) visits the active ancestor cells, reported at the group's base
// coordinate, and is_occupy (:86-88) is evaluated AT that coordinate: a group is
// exported iff its corner voxel passes rule.export_occ (hits: exists and has count > min_occupy_thres; log-odds: known
// and L > l_occ).
template <class Rule>
__global__ void __launch_bounds__(256) k_octo_extract(OcGrid g, int submap, int group, Rule rule, const float* pR, const float* pT,
                                                       float vs, long long cap, float* xyz, float* rgb, int* counter) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  const long long total = (long long)nb * OC_B3;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long iters = (total + stride - 1) / stride;
  for (long long it = 0; it < iters; ++it) {  // uniform trip count: the warp ballot below needs all lanes
    const long long e = it * stride + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    bool want = false;
    int i = 0, j = 0, k = 0, s = 0;
    if (e < total) {
      const int b = (int)(e >> 9);
      const int v = (int)(e & 511);
      int bx, by, bz;
      ts_unpack_key(g.block_key[b], s, bx, by, bz);
      i = bx * OC_B + (v >> 6); j = by * OC_B + ((v >> 3) & 7); k = bz * OC_B + (v & 7);
      // tree offset is -N/2 (taichi_octomap.py:72): groups are aligned in offset coordinates
      const bool aligned = ((i + g.hN) % group == 0) && ((j + g.hN) % group == 0) && ((k + g.hNz) % group == 0);
      want = (s == submap) && aligned && rule.export_occ(g.cnt[e]);
    }
    const int row = warp_append_i32(want, counter);
    if (want && row < cap) {
      // sijk_to_xyz mapping_common.py:234-238
      pose_apply(pR + 9 * s, pT + 3 * s, (float)i * vs, (float)j * vs, (float)k * vs, xyz[3 * (size_t)row], xyz[3 * (size_t)row + 1],
                 xyz[3 * (size_t)row + 2]);
      if (rgb && g.cw) oc_word_to_rgb(g.cw[e], rgb + 3 * (size_t)row);  // export_color[index] = color[sijk] (:101-102)
    }
  }
}

// fuse_submaps_kernel (taichi_octomap.py:171-189): every source voxel the rule carries over (rule.fuse_src) is placed at
// the nearest target voxel of its submap's pose and added there (rule.fuse_add); the largest colour word wins.
template <class Rule>
__global__ void __launch_bounds__(256) k_octo_fuse(OcGrid dst, OcGrid src, Rule rule, const float* pR, const float* pT, float vs) {
  const int nb = min(*src.n_blocks, src.max_blocks);
  const long long total = (long long)nb * OC_B3;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const unsigned int c = src.cnt[e];
    if (!rule.fuse_src(c)) continue;  // :181
    const int b = (int)(e >> 9), v = (int)(e & 511);
    int s, bx, by, bz;
    ts_unpack_key(src.block_key[b], s, bx, by, bz);
    int i, j, k;
    oc_fuse_cell(pR + 9 * s, pT + 3 * s, bx, by, bz, v, vs, i, j, k);  // :182-186
    if (!ts_in_bounds(dst, i, j, k)) continue;
    const int blk = ts_get_or_alloc(dst, ts_pack_key(0, i >> OC_BSHIFT, j >> OC_BSHIFT, k >> OC_BSHIFT));
    if (blk < 0) continue;
    const size_t o = (size_t)blk * OC_B3 + oc_voxel_off(i, j, k);
    rule.fuse_add(&dst.cnt[o], c);
    const unsigned long long cw = (dst.cw && src.cw) ? src.cw[e] : 0ull;  // color[ijk_] = submap_color[s,i,j,k] (:189)
    if (cw) ts_red_max_u64(&dst.cw[o], cw);
  }
}

// ---------------------------------------------------------------------------
// Log-odds occupancy (DESIGN.md section 7, "Log-odds Octomap").  One integrate call = one frame = four steps:
//   1. k_octo_lo_depth / k_octo_lo_points: one thread per sampled pixel / point.  Unproject, filter, clip at
//      max_ray_length, append a ray record, set the hit bit of the end cell (unless clipped) and raise its colour word.
//   2. k_octo_lo_walk: one lane per ray walks the 6-connected voxel path origin cell -> end cell and sets the miss bit
//      of every in-volume cell before the end cell (and of the end cell of a clipped ray).
//   3. k_octo_lo_apply: one CTA per block the frame touched: L <- clamp(L + (hit ? l_hit : l_miss)) for every marked
//      voxel, so a voxel is updated once per frame and a hit wins over a miss; the marks are cleared.
// ---------------------------------------------------------------------------

// first touch of a block in this frame: put it on the touched list
__device__ __forceinline__ void lo_touch(const OcLo& lo, int blk) {
  if (lo.touched_flag[blk] == 0 && atomicExch(&lo.touched_flag[blk], 1) == 0) lo.touched[atomicAdd(&lo.ctr[1], 1)] = blk;
}
// test-then-set: every ray starts in the few cells around the sensor, an unconditional atomic would serialise on them
__device__ __forceinline__ void lo_mark(const OcLo& lo, int blk, int v, bool hit) {
  uint32_t* w = lo.mark + (size_t)blk * OC_MARK_WORDS + (hit ? 0 : 16) + (v >> 5);
  const uint32_t bit = 1u << (v & 31);
  if (!(*(volatile uint32_t*)w & bit)) atomicOr(w, bit);
}

// append the ray record of a valid sample; an endpoint that is not clipped marks its cell as a hit
__device__ __forceinline__ void lo_emit(const OcGrid& g, const OcLo& lo, int s, float vs, bool valid, bool clipped, float px, float py,
                                        float pz, unsigned long long cw) {
  const int row = warp_append_i32(valid, &lo.ctr[0]);
  if (!valid) return;
  lo.rays[row] = make_float4(px, py, pz, clipped ? 1.0f : 0.0f);
  if (clipped) return;
  const int i = oc_iroundf(px / vs), j = oc_iroundf(py / vs), k = oc_iroundf(pz / vs);
  if (!ts_in_bounds(g, i, j, k)) return;
  const int blk = ts_get_or_alloc(g, ts_pack_key(s, i >> OC_BSHIFT, j >> OC_BSHIFT, k >> OC_BSHIFT));
  if (blk < 0) return;
  lo_touch(lo, blk);
  const int v = oc_voxel_off(i, j, k);
  lo_mark(lo, blk, v, true);
  if (cw) ts_red_max_u64(&g.cw[(size_t)blk * OC_B3 + v], cw);
}

__global__ void __launch_bounds__(256) k_octo_lo_depth(OcGrid g, OcLo lo, const uint16_t* __restrict__ depth, int h, int w, int hh, int ww,
                                                        TsFrame fr, TsIntrin in, const uint8_t* __restrict__ tex, int th, int tw) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false, clipped = false;
  float px = 0.0f, py = 0.0f, pz = 0.0f;
  unsigned long long cw = 0ull;
  if (t < hh * ww) {
    const int jj = t / ww, ii = t - jj * ww;
    const int j = jj * in.step, i = ii * in.step;
    const uint16_t d = depth[(size_t)j * w + i];
    const float df = (float)d;
    if (d != 0 && !(df < in.dmin_mm)) {
      valid = true;
      clipped = df > in.dmax_mm;
      const float dep = clipped ? lo.max_ray : df / 1000.0f;  // a far pixel is cut at depth max_ray_length
      const float x = ((float)i - in.cx) * dep / in.fx;
      const float y = ((float)j - in.cy) * dep / in.fy;
      px = ((fr.R[0] * x + fr.R[1] * y) + fr.R[2] * dep) + fr.T[0];
      py = ((fr.R[3] * x + fr.R[4] * y) + fr.R[5] * dep) + fr.T[1];
      pz = ((fr.R[6] * x + fr.R[7] * y) + fr.R[8] * dep) + fr.T[2];
      if (tex && !clipped) {
        int ti, tj;
        const uint8_t zero3[3] = {0, 0, 0};
        cw = oc_color_word(fr.seq, ts_color_pixel(in, i, j, th, tw, ti, tj) ? tex + ((size_t)tj * tw + ti) * 3 : zero3);
      }
    }
  }
  lo_emit(g, lo, fr.submap, in.vs, valid, clipped, px, py, pz, cw);
}

__global__ void __launch_bounds__(256) k_octo_lo_points(OcGrid g, OcLo lo, const float* __restrict__ xyz, int n, TsFrame fr, float vs,
                                                         const uint8_t* __restrict__ rgb) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false, clipped = false;
  float px = 0.0f, py = 0.0f, pz = 0.0f;
  unsigned long long cw = 0ull;
  if (t < n) {
    const float x = xyz[3 * (size_t)t], y = xyz[3 * (size_t)t + 1], z = xyz[3 * (size_t)t + 2];
    float rx = (fr.R[0] * x + fr.R[1] * y) + fr.R[2] * z;
    float ry = (fr.R[3] * x + fr.R[4] * y) + fr.R[5] * z;
    float rz = (fr.R[6] * x + fr.R[7] * y) + fr.R[8] * z;
    const float r = sqrtf((rx * rx + ry * ry) + rz * rz);  // range from the sensor
    valid = r >= lo.min_ray && r < INFINITY;
    clipped = r > lo.max_ray;
    if (clipped) {
      const float sc = lo.max_ray / r;
      rx = rx * sc; ry = ry * sc; rz = rz * sc;
    }
    px = rx + fr.T[0]; py = ry + fr.T[1]; pz = rz + fr.T[2];
    if (rgb && valid && !clipped) cw = oc_color_word(fr.seq, rgb + 3 * (size_t)t);
  }
  lo_emit(g, lo, fr.submap, vs, valid, clipped, px, py, pz, cw);
}

// Amanatides-Woo in voxel units: p0 = origin / vs, p1 = endpoint / vs, cells c = round_half_away(p).  The k-th boundary
// crossing of axis a is at t = ((c_a + 0.5 s_a) - p0_a) * (1 / (p1_a - p0_a)), recomputed from the current cell (no
// accumulated increments); each step takes the axis with the smallest t among those with steps left, ties to the
// lower axis.  The step counts |c1 - c0| per axis are integers, so the path always has |c1 - c0|_1 + 1 cells.
// The viewpoint-gain kernels walk the same path through oc_walk_begin / oc_walk_step (tslam_internal.cuh); this kernel
// keeps its own copy because the helper changes its SASS (a jump table for the step), checked bit for bit instead.
__global__ void __launch_bounds__(256) k_octo_lo_walk(OcGrid g, OcLo lo, int s, float vs, float ox, float oy, float oz) {
  const int n = lo.ctr[0];
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0) atomicAdd(&lo.stats[0], (unsigned long long)n);
  unsigned int visits = 0;
  if (t < n) {
    const float4 r = lo.rays[t];
    const float p0x = ox / vs, p0y = oy / vs, p0z = oz / vs;
    const float p1x = r.x / vs, p1y = r.y / vs, p1z = r.z / vs;
    int cx = oc_iroundf(p0x), cy = oc_iroundf(p0y), cz = oc_iroundf(p0z);
    const int ex = oc_iroundf(p1x), ey = oc_iroundf(p1y), ez = oc_iroundf(p1z);
    int lx = abs(ex - cx), ly = abs(ey - cy), lz = abs(ez - cz);
    const int sx = ex > cx ? 1 : -1, sy = ey > cy ? 1 : -1, sz = ez > cz ? 1 : -1;
    const float hx = 0.5f * (float)sx, hy = 0.5f * (float)sy, hz = 0.5f * (float)sz;
    const float ix = lx ? 1.0f / (p1x - p0x) : 0.0f, iy = ly ? 1.0f / (p1y - p0y) : 0.0f, iz = lz ? 1.0f / (p1z - p0z) : 0.0f;
    float tx = (((float)cx + hx) - p0x) * ix, ty = (((float)cy + hy) - p0y) * iy, tz = (((float)cz + hz) - p0z) * iz;
    const bool clipped = r.w != 0.0f;
    unsigned long long ckey = ~0ull;
    int cblk = -1;
    for (int left = lx + ly + lz;; --left) {
      if ((left > 0 || clipped) && ts_in_bounds(g, cx, cy, cz)) {
        ++visits;
        const unsigned long long key = ts_pack_key(s, cx >> OC_BSHIFT, cy >> OC_BSHIFT, cz >> OC_BSHIFT);
        if (key != ckey) {  // hash probe only when the walk enters another block
          ckey = key;
          cblk = ts_get_or_alloc(g, key);
          if (cblk >= 0) lo_touch(lo, cblk);
        }
        if (cblk >= 0) lo_mark(lo, cblk, oc_voxel_off(cx, cy, cz), false);
      }
      if (left == 0) break;
      int a = 3;
      float tb = 0.0f;
      if (lx > 0) { a = 0; tb = tx; }
      if (ly > 0 && (a == 3 || ty < tb)) { a = 1; tb = ty; }
      if (lz > 0 && (a == 3 || tz < tb)) a = 2;
      if (a == 0) { cx += sx; --lx; tx = (((float)cx + hx) - p0x) * ix; }
      else if (a == 1) { cy += sy; --ly; ty = (((float)cy + hy) - p0y) * iy; }
      else { cz += sz; --lz; tz = (((float)cz + hz) - p0z) * iz; }
    }
  }
  for (int o = 16; o > 0; o >>= 1) visits += __shfl_xor_sync(0xffffffffu, visits, o);
  if ((threadIdx.x & 31) == 0 && visits) atomicAdd(&lo.stats[1], (unsigned long long)visits);
}

// one CTA (128 threads, 4 voxels each) per touched block.  TRACK names the change trackers that exist (OC_TRACK_ESDF:
// an occupancy ESDF, OC_TRACK_FRONTIER: a frontier tracker); the block is flagged for the next incremental update of
// each (esdf_dirty, fr_dirty).  Without a tracker nothing is marked.
template <unsigned TRACK>
__global__ void __launch_bounds__(128) k_octo_lo_apply(OcGrid g, OcLo lo, int* esdf_dirty, int* fr_dirty) {
  __shared__ uint32_t mk[OC_MARK_WORDS];
  __shared__ unsigned int n_hit, n_upd;
  const int nt = lo.ctr[1];
  if (threadIdx.x == 0) { n_hit = 0; n_upd = 0; }
  for (int q = blockIdx.x; q < nt; q += gridDim.x) {
    const int blk = lo.touched[q];
    __syncthreads();  // the previous block's marks are consumed
    if (threadIdx.x < OC_MARK_WORDS) {
      uint32_t* w = lo.mark + (size_t)blk * OC_MARK_WORDS + threadIdx.x;
      mk[threadIdx.x] = *w;
      *w = 0u;
    }
    if (threadIdx.x == 0) lo.touched_flag[blk] = 0;
    if ((TRACK & OC_TRACK_ESDF) && threadIdx.x == 0) esdf_dirty[blk] = 1;
    if ((TRACK & OC_TRACK_FRONTIER) && threadIdx.x == 0) fr_dirty[blk] = 1;
    __syncthreads();
    unsigned int h = 0, u = 0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int v = threadIdx.x + 128 * r;
      const bool hit = (mk[v >> 5] >> (v & 31)) & 1u;
      const bool miss = (mk[16 + (v >> 5)] >> (v & 31)) & 1u;
      if (!(hit || miss)) continue;
      unsigned int* p = g.cnt + (size_t)blk * OC_B3 + v;
      const unsigned int w = *p;
      const int L = (lo_known(w) ? lo_val(w) : 0) + (hit ? lo.l_hit : lo.l_miss);
      *p = lo_word(min(max(L, lo.l_min), lo.l_max));
      h += hit;
      ++u;
    }
    if (h) atomicAdd(&n_hit, h);
    if (u) atomicAdd(&n_upd, u);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (n_hit) atomicAdd(&lo.stats[2], (unsigned long long)n_hit);
    if (n_upd) atomicAdd(&lo.stats[3], (unsigned long long)n_upd);
  }
}

// after k_octo_fuse<OcLogodds>: clamps every known target voxel once, when all sums are in
__global__ void __launch_bounds__(256) k_octo_lo_clamp(OcGrid g, int l_min, int l_max) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  const long long total = (long long)nb * OC_B3;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const unsigned int c = g.cnt[e];
    if (lo_known(c)) g.cnt[e] = lo_word(min(max(lo_val(c), l_min), l_max));
  }
}

// ---------------------------------------------------------------------------
static size_t oc_next_pow2(size_t v) {
  size_t p = 1;
  while (p < v) p <<= 1;
  return p;
}

static int oc_create(const tslam_octo_config_t* cfg, const tslam_octo_logodds_t* lp, tslam_octo_t** out) {
  if (!cfg || !out) return TSLAM_E_INVALID;
  *out = nullptr;
  if (cfg->voxel_scale <= 0 || cfg->N <= 0 || cfg->Nz <= 0 || cfg->N > 8192 || cfg->Nz > 8192 || cfg->recast_step <= 0) {
    ts_set_error("invalid octomap config");
    return TSLAM_E_INVALID;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    ts_set_error("no CUDA device visible: libtslam has no CPU fallback");
    return TSLAM_E_NOGPU;
  }
  tslam_octo* m = new tslam_octo();
  memset(m, 0, sizeof(*m));
  m->cfg = *cfg;
  int dev = 0;
  TS_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  TS_CUDA(cudaGetDeviceProperties(&prop, dev));
  m->sm_count = prop.multiProcessorCount;
  if (m->cfg.max_submaps <= 0 || m->cfg.max_submaps > 1024) m->cfg.max_submaps = 1024;
  if (m->cfg.max_image_pixels <= 0) m->cfg.max_image_pixels = 640 * 480;
  if (m->cfg.max_points <= 0) m->cfg.max_points = 1 << 20;
  if (m->cfg.max_blocks <= 0) m->cfg.max_blocks = 1 << 18;  // 262144 blocks x 2 KB = 512 MB
  if (m->cfg.max_blocks > TS_MAX_BLOCKS) m->cfg.max_blocks = TS_MAX_BLOCKS;
  fz_ver_init(m->ver, m->cfg.max_submaps);
  m->in.fx = (float)cfg->fx; m->in.fy = (float)cfg->fy; m->in.cx = (float)cfg->cx; m->in.cy = (float)cfg->cy;
  m->in.dmin_mm = (float)(cfg->min_ray_length * 1000.0);
  m->in.dmax_mm = (float)(cfg->max_ray_length * 1000.0);
  m->in.vs = (float)cfg->voxel_scale;
  m->in.step = cfg->recast_step;
  OcGrid& g = m->g;
  g.max_blocks = m->cfg.max_blocks;
  g.N = cfg->N; g.Nz = cfg->Nz; g.hN = cfg->N / 2; g.hNz = cfg->Nz / 2;
  m->table_cap = oc_next_pow2((size_t)g.max_blocks * 2 + 64);
  g.table_mask = (uint32_t)(m->table_cap - 1);
  TS_CUDA(cudaMalloc(&g.table, m->table_cap * 8));
  TS_CUDA(cudaMemset(g.table, 0xFF, m->table_cap * 8));
  TS_CUDA(cudaMalloc(&g.block_key, (size_t)g.max_blocks * 8));
  TS_CUDA(cudaMalloc(&g.cnt, (size_t)g.max_blocks * OC_B3 * 4));
  TS_CUDA(cudaMemset(g.cnt, 0, (size_t)g.max_blocks * OC_B3 * 4));
  g.cw = nullptr;
  if (cfg->texture_enabled) {
    TS_CUDA(cudaMalloc(&g.cw, (size_t)g.max_blocks * OC_B3 * 8));
    TS_CUDA(cudaMemset(g.cw, 0, (size_t)g.max_blocks * OC_B3 * 8));
    const size_t tb = (size_t)m->cfg.max_image_pixels > (size_t)m->cfg.max_points ? (size_t)m->cfg.max_image_pixels : (size_t)m->cfg.max_points;
    TS_CUDA(cudaMalloc(&m->tex_stage, tb * 3));
  }
  m->in.same_proj = 1;
  TS_CUDA(cudaMalloc(&m->scratch_i, 64 * 4));
  TS_CUDA(cudaMemset(m->scratch_i, 0, 64 * 4));
  g.n_blocks = m->scratch_i + 0;
  g.err = m->scratch_i + 2;
  TS_CUDA(cudaMalloc(&m->depth_stage, (size_t)m->cfg.max_image_pixels * 2));
  TS_CUDA(cudaMalloc(&m->points_stage, (size_t)m->cfg.max_points * 12));
  TS_CUDA(cudaMalloc(&m->pose_R, (size_t)m->cfg.max_submaps * 36));
  TS_CUDA(cudaMalloc(&m->pose_T, (size_t)m->cfg.max_submaps * 12));
  TS_CUDA(cudaMemset(m->pose_R, 0, (size_t)m->cfg.max_submaps * 36));
  TS_CUDA(cudaMemset(m->pose_T, 0, (size_t)m->cfg.max_submaps * 12));
  if (lp) {  // log-odds workspace: mark plane 128 B + touched flag / list 8 B per pool block, 16 B per ray record
    m->logodds = 1;
    OcLo& lo = m->lo;
    lo.l_hit = lp->l_hit; lo.l_miss = lp->l_miss; lo.l_min = lp->l_min; lo.l_max = lp->l_max; lo.l_occ = lp->l_occ;
    lo.min_ray = (float)cfg->min_ray_length;
    lo.max_ray = (float)cfg->max_ray_length;
    m->ray_cap = m->cfg.max_image_pixels > m->cfg.max_points ? m->cfg.max_image_pixels : m->cfg.max_points;
    TS_CUDA(cudaMalloc(&lo.mark, (size_t)g.max_blocks * OC_MARK_WORDS * 4));
    TS_CUDA(cudaMemset(lo.mark, 0, (size_t)g.max_blocks * OC_MARK_WORDS * 4));
    TS_CUDA(cudaMalloc(&lo.touched_flag, (size_t)g.max_blocks * 4));
    TS_CUDA(cudaMemset(lo.touched_flag, 0, (size_t)g.max_blocks * 4));
    TS_CUDA(cudaMalloc(&lo.touched, (size_t)g.max_blocks * 4));
    TS_CUDA(cudaMalloc(&lo.rays, (size_t)m->ray_cap * 16));
    lo.ctr = m->scratch_i + 16;
    TS_CUDA(cudaMalloc(&lo.stats, 4 * 8));
    TS_CUDA(cudaMemset(lo.stats, 0, 4 * 8));
  }
  TS_CUDA(cudaDeviceSynchronize());
  *out = m;
  return TSLAM_OK;
}

extern "C" int tslam_octo_create(const tslam_octo_config_t* cfg, tslam_octo_t** out) { return oc_create(cfg, nullptr, out); }

extern "C" int tslam_octo_create_logodds(const tslam_octo_config_t* cfg, const tslam_octo_logodds_t* lp, tslam_octo_t** out) {
  if (!lp || !out) return TSLAM_E_INVALID;
  *out = nullptr;
  if (!(lp->l_min <= 0 && 0 <= lp->l_max && lp->l_min < lp->l_max && lp->l_miss < 0 && lp->l_hit > 0 && lp->l_min >= -(1 << 24) &&
        lp->l_max <= (1 << 24) && lp->l_occ >= lp->l_min && lp->l_occ <= lp->l_max)) {
    ts_set_error("invalid log-odds parameters: need l_miss < 0 < l_hit, l_min <= 0 <= l_max within +-2^24, l_occ in [l_min, l_max]");
    return TSLAM_E_INVALID;
  }
  return oc_create(cfg, lp, out);
}

extern "C" int tslam_octo_destroy(tslam_octo_t* m) {
  if (!m) return TSLAM_OK;
  cudaDeviceSynchronize();
  cudaFree(m->g.table); cudaFree(m->g.block_key); cudaFree(m->g.cnt); cudaFree(m->scratch_i);
  if (m->g.cw) cudaFree(m->g.cw);
  if (m->tex_stage) cudaFree(m->tex_stage);
  cudaFree(m->depth_stage); cudaFree(m->points_stage); cudaFree(m->pose_R); cudaFree(m->pose_T);
  if (m->logodds) {
    cudaFree(m->lo.mark); cudaFree(m->lo.touched_flag); cudaFree(m->lo.touched); cudaFree(m->lo.rays); cudaFree(m->lo.stats);
  }
  oc_esdf_free(m);
  oc_frontier_free(m);
  oc_view_free(m);
  oc_travel_free(m);
  if (m->traj_mem) cudaFree(m->traj_mem);
  fz_free(m->fz);
  fz_ver_free(m->ver);
  delete m;
  return TSLAM_OK;
}

extern "C" int tslam_octo_reset(tslam_octo_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int nb = 0;
  TS_CUDA(cudaMemcpyAsync(&nb, m->g.n_blocks, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (nb > m->g.max_blocks) nb = m->g.max_blocks;
  TS_CUDA(cudaMemsetAsync(m->g.table, 0xFF, m->table_cap * 8, st));
  if (nb) TS_CUDA(cudaMemsetAsync(m->g.cnt, 0, (size_t)nb * OC_B3 * 4, st));
  if (nb && m->g.cw) TS_CUDA(cudaMemsetAsync(m->g.cw, 0, (size_t)nb * OC_B3 * 8, st));
  TS_CUDA(cudaMemsetAsync(m->scratch_i, 0, 4 * 4, st));
  oc_track_invalidate_all(m);
  fz_written(m->ver, -1);
  return TSLAM_OK;
}

void oc_track_invalidate_all(tslam_octo* m) {
  for (OcTrack* t : {&m->esdf_track, &m->fr_track, &m->tr.track, &m->trm.track}) t->ready = 0;
}

int oc_logodds_submap(tslam_octo* m, int32_t submap, const char* what, const char* feature) {
  if (!m->logodds) {
    ts_set_error("%s: the map is a hit counter; %s needs a log-odds map (tslam_octo_create_logodds)", what, feature);
    return TSLAM_E_INVALID;
  }
  if (submap < 0 || submap >= m->cfg.max_submaps) { ts_set_error("%s: submap %d out of range", what, submap); return TSLAM_E_INVALID; }
  return TSLAM_OK;
}

int oc_track_readable(tslam_octo* m, const OcTrack& t, int32_t submap, const char* what, const char* update) {
  int rc = oc_logodds_submap(m, submap, what, update);
  if (rc) return rc;
  if (!t.ready) {
    ts_set_error("%s: no completed %s since the map was created, reset or fused, or since the last one failed", what, update);
    return TSLAM_E_INVALID;
  }
  if (t.submap != submap) {
    ts_set_error("%s: the last %s was for submap %d, not %d", what, update, t.submap, submap);
    return TSLAM_E_INVALID;
  }
  return TSLAM_OK;
}

int oc_reserve(void** p, size_t* bytes, size_t need) {
  if (need <= *bytes) return TSLAM_OK;
  if (*p) cudaFree(*p);
  *p = nullptr;
  *bytes = 0;
  TS_CUDA(cudaMalloc(p, need));
  *bytes = need;
  return TSLAM_OK;
}

extern "C" int tslam_octo_set_submap_pose(tslam_octo_t* m, int32_t s, const float* R9, const float* T3) {
  if (!m || !R9 || !T3 || s < 0 || s >= m->cfg.max_submaps) return TSLAM_E_INVALID;
  TS_CUDA(cudaMemcpy(m->pose_R + 9 * (size_t)s, R9, 36, cudaMemcpyHostToDevice));
  TS_CUDA(cudaMemcpy(m->pose_T + 3 * (size_t)s, T3, 12, cudaMemcpyHostToDevice));
  return TSLAM_OK;
}

extern "C" int tslam_octo_set_intrinsics(tslam_octo_t* m, double fx, double fy, double cx, double cy) {
  if (!m) return TSLAM_E_INVALID;
  m->cfg.fx = fx; m->cfg.fy = fy; m->cfg.cx = cx; m->cfg.cy = cy;
  m->in.fx = (float)fx; m->in.fy = (float)fy; m->in.cx = (float)cx; m->in.cy = (float)cy;
  return TSLAM_OK;
}

extern "C" int tslam_octo_set_color_intrinsics(tslam_octo_t* m, double fx, double fy, double cx, double cy, int color_same_proj) {
  if (!m) return TSLAM_E_INVALID;
  m->in.fxc = (float)fx; m->in.fyc = (float)fy; m->in.cxc = (float)cx; m->in.cyc = (float)cy;
  m->in.same_proj = color_same_proj ? 1 : 0;
  return TSLAM_OK;
}

static void oc_fill_frame(tslam_octo* m, TsFrame& fr, const float* R9, const float* T3, int submap) {
  memcpy(fr.R, R9, 36); memcpy(fr.T, T3, 12); fr.submap = submap;
  if (m->frame_seq < 0xFFFFFFFEu) m->frame_seq++;  // the colour word keeps 40 bits for it (seq << 24 | rgb): no practical limit
  fr.seq = m->frame_seq;
}

// steps 2 and 3 of a log-odds frame; n_max bounds the ray records the endpoint kernel wrote
static int oc_lo_finish(tslam_octo* m, const TsFrame& fr, int n_max, cudaStream_t st) {
  k_octo_lo_walk<<<(n_max + 255) / 256, 256, 0, st>>>(m->g, m->lo, fr.submap, m->in.vs, fr.T[0], fr.T[1], fr.T[2]);
  TS_LAUNCH_CHECK(m);
  const unsigned track = (m->esdf_dirty ? OC_TRACK_ESDF : 0u) | (m->fr_dirty ? OC_TRACK_FRONTIER : 0u);
  const int grid = m->sm_count * 16;
  if (track == 0u)
    k_octo_lo_apply<0u><<<grid, 128, 0, st>>>(m->g, m->lo, nullptr, nullptr);
  else if (track == OC_TRACK_ESDF)
    k_octo_lo_apply<OC_TRACK_ESDF><<<grid, 128, 0, st>>>(m->g, m->lo, m->esdf_dirty, nullptr);
  else if (track == OC_TRACK_FRONTIER)
    k_octo_lo_apply<OC_TRACK_FRONTIER><<<grid, 128, 0, st>>>(m->g, m->lo, nullptr, m->fr_dirty);
  else
    k_octo_lo_apply<OC_TRACK_ESDF | OC_TRACK_FRONTIER><<<grid, 128, 0, st>>>(m->g, m->lo, m->esdf_dirty, m->fr_dirty);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

// Reads and clears the device error flags.  A pool or table bit means hits were dropped: TSLAM_E_POOL_FULL.  Otherwise
// one message names every tracker bit that is set: TSLAM_E_INVALID.
int oc_deferred(tslam_octo* m) {
  int err = 0;
  TS_CUDA(cudaMemcpy(&err, m->g.err, 4, cudaMemcpyDeviceToHost));
  if (!err) return TSLAM_OK;
  int zero = 0;
  cudaMemcpy(m->g.err, &zero, 4, cudaMemcpyHostToDevice);
  static const struct { int bit; const char* msg; } flags[] = {
      {OC_ERR_VIEW_WINDOW, "octo view gain: a walk left its view's bitmap window (is every view's R a rotation?): gains are invalid"},
      {OC_ERR_TRAVEL_PATH, "octo travel path: a cell of the field had no predecessor: paths are invalid"},
      {OC_ERR_TRAVEL_SOURCE, "octo travel multi path: a source index was outside [0, n_starts): those paths have len 0"},
      {OC_ERR_FUSE_MISSING, "octo fuse_update: a removal found no block of dst (the map and its fusion record disagree): the next update is a "
                            "full one"}};
  int tracker = 0;
  for (const auto& f : flags) tracker |= f.bit;
  if (err & ~tracker) {
    ts_set_error("octomap block pool / table exhausted (max_blocks=%d, flags 0x%x): hits were dropped", m->g.max_blocks, err);
    return TSLAM_E_POOL_FULL;
  }
  std::string msg;
  for (const auto& f : flags)
    if (err & f.bit) msg += (msg.empty() ? "" : "; ") + std::string(f.msg);
  ts_set_error("%s", msg.c_str());
  return TSLAM_E_INVALID;
}

extern "C" int tslam_octo_integrate_points(tslam_octo_t* m, const float* xyz, int mem, int32_t n, const float* R9, const float* T3,
                                           int32_t submap, void* stream) {
  return tslam_octo_integrate_points_rgb(m, xyz, nullptr, mem, n, R9, T3, submap, stream);
}
extern "C" int tslam_octo_integrate_points_rgb(tslam_octo_t* m, const float* xyz, const uint8_t* rgb, int mem, int32_t n, const float* R9,
                                               const float* T3, int32_t submap, void* stream) {
  if (m && rgb && !m->g.cw) { ts_set_error("point colours given but the octomap was created with texture_enabled=0"); return TSLAM_E_INVALID; }
  if (!m || (!xyz && n > 0) || !R9 || !T3 || n < 0 || submap < 0 || submap >= m->cfg.max_submaps) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  if (n > m->cfg.max_points && mem == TSLAM_MEM_HOST) { ts_set_error("n=%d exceeds max_points=%d", n, m->cfg.max_points); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const float* src = xyz;
  if (mem == TSLAM_MEM_HOST) {
    TS_CUDA(cudaMemcpyAsync(m->points_stage, xyz, (size_t)n * 12, cudaMemcpyHostToDevice, st));
    src = m->points_stage;
  }
  const uint8_t* csrc = rgb;
  if (rgb && mem == TSLAM_MEM_HOST) {
    TS_CUDA(cudaMemcpyAsync(m->tex_stage, rgb, (size_t)n * 3, cudaMemcpyHostToDevice, st));
    csrc = m->tex_stage;
  }
  TsFrame fr;
  oc_fill_frame(m, fr, R9, T3, submap);
  if (m->logodds) {
    if (n > m->ray_cap) { ts_set_error("n=%d exceeds the ray records of a log-odds map (%d)", n, m->ray_cap); return TSLAM_E_INVALID; }
    fz_written(m->ver, submap);
    TS_CUDA(cudaMemsetAsync(m->lo.ctr, 0, 8, st));
    k_octo_lo_points<<<(n + 255) / 256, 256, 0, st>>>(m->g, m->lo, src, n, fr, m->in.vs, csrc);
    TS_LAUNCH_CHECK(m);
    return oc_lo_finish(m, fr, n, st);
  }
  fz_written(m->ver, submap);
  k_octo_points<<<(n + 255) / 256, 256, 0, st>>>(m->g, src, n, fr, m->in.vs, csrc);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

extern "C" int tslam_octo_integrate_depth(tslam_octo_t* m, const uint16_t* depth, int mem, int32_t h, int32_t w, const float* R9,
                                          const float* T3, int32_t submap, void* stream) {
  return tslam_octo_integrate_depth_tex(m, depth, nullptr, mem, h, w, 0, 0, R9, T3, submap, stream);
}
extern "C" int tslam_octo_integrate_depth_tex(tslam_octo_t* m, const uint16_t* depth, const uint8_t* tex, int mem, int32_t h, int32_t w,
                                              int32_t th, int32_t tw, const float* R9, const float* T3, int32_t submap, void* stream) {
  if (m && tex) {
    if (!m->g.cw) { ts_set_error("colour image given but the octomap was created with texture_enabled=0"); return TSLAM_E_INVALID; }
    if (th <= 0 || tw <= 0 || (long long)th * tw > m->cfg.max_image_pixels) { ts_set_error("texture exceeds max_image_pixels"); return TSLAM_E_INVALID; }
  }
  if (!m || !depth || !R9 || !T3 || h <= 0 || w <= 0 || submap < 0 || submap >= m->cfg.max_submaps) return TSLAM_E_INVALID;
  if ((long long)h * w > m->cfg.max_image_pixels) { ts_set_error("frame exceeds max_image_pixels"); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const uint16_t* src = depth;
  if (mem == TSLAM_MEM_HOST) {
    TS_CUDA(cudaMemcpyAsync(m->depth_stage, depth, (size_t)h * w * 2, cudaMemcpyHostToDevice, st));
    src = m->depth_stage;
  }
  const int step = m->cfg.recast_step;
  const int hh = (int)((double)h / step), ww = (int)((double)w / step);
  if (hh <= 0 || ww <= 0) return TSLAM_OK;
  const uint8_t* tsrc = tex;
  if (tex && mem == TSLAM_MEM_HOST) {
    TS_CUDA(cudaMemcpyAsync(m->tex_stage, tex, (size_t)th * tw * 3, cudaMemcpyHostToDevice, st));
    tsrc = m->tex_stage;
  }
  TsFrame fr;
  oc_fill_frame(m, fr, R9, T3, submap);
  fz_written(m->ver, submap);
  if (m->logodds) {
    TS_CUDA(cudaMemsetAsync(m->lo.ctr, 0, 8, st));
    k_octo_lo_depth<<<(hh * ww + 255) / 256, 256, 0, st>>>(m->g, m->lo, src, h, w, hh, ww, fr, m->in, tsrc, th, tw);
    TS_LAUNCH_CHECK(m);
    return oc_lo_finish(m, fr, hh * ww, st);
  }
  k_octo_depth<<<(hh * ww + 255) / 256, 256, 0, st>>>(m->g, src, h, w, hh, ww, fr, m->in, tsrc, th, tw);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

static int oc_gather(tslam_octo* m, int32_t submap, int64_t cap, int32_t* idx, uint32_t* count, float* color, int64_t* n_out,
                     cudaStream_t st) {
  const int rc = oc_counted_gather(m, st, [&](unsigned long long* ctr) {
    oc_with_rule(m, [&](auto rule) {
      k_octo_gather<decltype(rule)><<<m->sm_count * 8, 256, 0, st>>>(m->g, submap, cap, idx, count, color, ctr);
    });
  }, cap, n_out, m->logodds ? "tslam_octo_gather_logodds" : "tslam_octo_gather");
  if (rc && rc != TSLAM_E_CAPACITY) return rc;
  const int drc = oc_deferred(m);  // dropped hits are reported before a short buffer
  return drc ? drc : rc;
}

extern "C" int tslam_octo_gather(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, uint32_t* count, int64_t* n_out,
                                 void* stream) {
  return tslam_octo_gather2(m, submap, cap, idx, count, nullptr, n_out, stream);
}
extern "C" int tslam_octo_gather2(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, uint32_t* count, float* color,
                                  int64_t* n_out, void* stream) {
  if (!m || !n_out) return TSLAM_E_INVALID;
  if (m->logodds) { ts_set_error("tslam_octo_gather*: the map holds log-odds, read it with tslam_octo_gather_logodds"); return TSLAM_E_INVALID; }
  return oc_gather(m, submap, cap, idx, count, color, n_out, (cudaStream_t)stream);
}
extern "C" int tslam_octo_gather_logodds(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, int32_t* L, float* color,
                                         int64_t* n_out, void* stream) {
  if (!m || !n_out) return TSLAM_E_INVALID;
  if (!m->logodds) { ts_set_error("tslam_octo_gather_logodds: the map is a hit counter"); return TSLAM_E_INVALID; }
  return oc_gather(m, submap, cap, idx, (uint32_t*)L, color, n_out, (cudaStream_t)stream);
}

extern "C" int tslam_octo_extract(tslam_octo_t* m, int32_t submap, int32_t level, int64_t cap, float* xyz, int32_t* count_dev,
                                  void* stream) {
  return tslam_octo_extract2(m, submap, level, cap, xyz, nullptr, count_dev, stream);
}
extern "C" int tslam_octo_extract2(tslam_octo_t* m, int32_t submap, int32_t level, int64_t cap, float* xyz, float* rgb,
                                   int32_t* count_dev, void* stream) {
  if (!m || !xyz || !count_dev || level < 1) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  long long group = 1;
  for (int l = 1; l < level; l++) group *= m->cfg.K;
  if (group > (1 << 20)) group = 1 << 20;
  oc_with_rule(m, [&](auto rule) {
    k_octo_extract<<<m->sm_count * 8, 256, 0, st>>>(m->g, submap, (int)group, rule, m->pose_R, m->pose_T, m->in.vs, cap, xyz, rgb, count_dev);
  });
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

extern "C" int tslam_octo_fuse(tslam_octo_t* dst, tslam_octo_t* src, void* stream) {
  if (!dst || !src || dst == src) return TSLAM_E_INVALID;
  if (dst->logodds != src->logodds) { ts_set_error("tslam_octo_fuse: a log-odds map and a hit counter cannot be fused"); return TSLAM_E_INVALID; }
  int rc = tslam_octo_reset(dst, stream);  // taichi_octomap.py:195-196
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  oc_with_rule(dst, [&](auto rule) {
    k_octo_fuse<<<dst->sm_count * 8, 256, 0, st>>>(dst->g, src->g, rule, dst->pose_R, dst->pose_T, dst->in.vs);
  });
  TS_LAUNCH_CHECK(dst);
  if (dst->logodds) {
    k_octo_lo_clamp<<<dst->sm_count * 8, 256, 0, st>>>(dst->g, dst->lo.l_min, dst->lo.l_max);
    TS_LAUNCH_CHECK(dst);
  }
  return TSLAM_OK;
}

extern "C" int tslam_octo_sync(tslam_octo_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  TS_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return oc_deferred(m);
}
extern "C" int64_t tslam_octo_launch_count(tslam_octo_t* m) { return m ? m->launches : 0; }

extern "C" int tslam_octo_get_stats(tslam_octo_t* m, int64_t* out4, int clear) {
  if (!m || !out4) return TSLAM_E_INVALID;
  if (!m->logodds) { for (int q = 0; q < 4; q++) out4[q] = 0; return TSLAM_OK; }
  TS_CUDA(cudaDeviceSynchronize());
  TS_CUDA(cudaMemcpy(out4, m->lo.stats, 32, cudaMemcpyDeviceToHost));
  if (clear) TS_CUDA(cudaMemset(m->lo.stats, 0, 32));
  return TSLAM_OK;
}
