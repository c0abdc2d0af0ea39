// libtslam.so - viewpoint gain of a log-odds Octomap (DESIGN.md section 7, "Viewpoint gain of the log-odds Octomap").
//
// Per submap, classes as the occupancy ESDF and the frontiers define them: OCC = known and L > l_occ, FREE = known and
// L <= l_occ, UNKNOWN = not known (every cell of an absent block).  A view is a position p and a rotation R (row-major)
// in the submap's map frame; it is valid iff its 12 numbers are finite and its cell c0 = rha(p / vs) is in the volume
// and FREE.
//   unknown gain   one lane per (view, ray): the ray of an all-far pixel (k_octo_lo_depth's clipped endpoint at depth
//                  max_range) walks k_octo_lo_walk's path, end cell included, up to its first OCC cell; every UNKNOWN
//                  cell it sees sets a bit in the view's bitmap, and the lane that sets a bit counts it.  The bitmap
//                  covers the view's window, the cube of half-extent ceil(r_max / vs) + 2 around c0 clipped to the
//                  volume; views run in chunks whose bitmaps fit the scratch budget.
//   frontier gain  one lane per (view, frontier voxel): frustum test, then the line-of-sight walk from p to the voxel
//                  centre, which must cross FREE cells only; counts per (view, cluster ordinal) by warp-aggregated
//                  integer atomics.
// Neither writes the map: blocks are looked up with ts_find (no allocation) and no mark, touched list, dirty flag or
// stats counter is touched.  Every output is an integer count, so the result does not depend on the thread schedule.
#include <cmath>
#include <cstdlib>
#include "tslam_internal.cuh"

#define OV_SCRATCH_BYTES (256ull << 20)  // bitmap budget per chunk of views (TSLAM_VIEW_SCRATCH overrides); >= 1 view
#define OV_MAX_HALF (1 << 22)            // largest window half-extent in cells: cell indices stay far from int overflow

struct OvCam {
  float fx, fy, cx, cy, max_range, wmax, hmax;  // wmax / hmax = f32(width - 1), f32(height - 1)
  int ww, hh, step;                             // rays per row / column, pixel stride
  int half;                                     // window half-extent in cells
};

// oc_class of cell (i, j, k) in pool block blk; an absent block (blk < 0) reads UNKNOWN.  The rule is spelled out here
// because calling oc_class changes the SASS of the three kernels that use it (k_octo_lo_walk keeps its walk for the
// same reason).
__device__ __forceinline__ int ov_cell_class(const OcGrid& g, int blk, int i, int j, int k, int l_occ) {
  if (blk < 0) return OC_UNK;
  const unsigned int w = g.cnt[(size_t)blk * OC_B3 + oc_voxel_off(i, j, k)];
  return !lo_known(w) ? OC_UNK : (lo_val(w) > l_occ ? OC_OCC : OC_FREE);
}

// valid[v] for every view
__global__ void __launch_bounds__(256) k_octo_view_valid(OcGrid g, int s, float vs, int l_occ, const float* __restrict__ pos,
                                                          const float* __restrict__ R9, long long n, uint8_t* valid) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x) {
    bool ok = true;
    for (int q = 0; q < 3; ++q) ok = ok && isfinite(pos[3 * v + q]);
    for (int q = 0; q < 9; ++q) ok = ok && isfinite(R9[9 * v + q]);
    if (ok) {
      const float u0 = pos[3 * v] / vs, u1 = pos[3 * v + 1] / vs, u2 = pos[3 * v + 2] / vs;
      ok = fabsf(u0) < 1e9f && fabsf(u1) < 1e9f && fabsf(u2) < 1e9f;  // no out-of-range float -> int conversion below
      if (ok) {
        const int i = (int)roundf(u0), j = (int)roundf(u1), k = (int)roundf(u2);
        ok = ts_in_bounds(g, i, j, k) &&
             ov_cell_class(g, ts_find(g, ts_pack_key(s, i >> OC_BSHIFT, j >> OC_BSHIFT, k >> OC_BSHIFT)), i, j, k, l_occ) == OC_FREE;
      }
    }
    valid[v] = ok ? 1 : 0;
  }
}

// Unknown gain of the chunk of views [v0, v0 + nv).  bits: nv bitmaps of `words` u32 each, zeroed.  The walk stops at
// the first OCC cell, and when it leaves the volume: every axis moves monotonically from c0 (inside) to c1, so no later
// cell of the path is inside again.
__global__ void __launch_bounds__(256) k_octo_view_unknown(OcGrid g, OvCam cam, int s, float vs, int l_occ, const float* __restrict__ pos,
                                                            const float* __restrict__ R9, const uint8_t* __restrict__ valid, long long v0,
                                                            int nv, long long words, uint32_t* bits, unsigned long long* gain) {
  const int nrays = cam.ww * cam.hh;
  const long long total = (long long)nv * nrays;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  for (long long base = (long long)blockIdx.x * blockDim.x; base < total; base += stride) {  // uniform per warp
    const long long t = base + threadIdx.x;
    long long v = -1;
    unsigned int cnt = 0;
    if (t < total) {
      const int vl = (int)(t / nrays), r = (int)(t - (long long)vl * nrays);
      v = v0 + vl;
      if (valid[v]) {
        const float* p = pos + 3 * v;
        const float* R = R9 + 9 * v;
        const float px = p[0], py = p[1], pz = p[2];
        const int jj = r / cam.ww, ii = r - jj * cam.ww;
        const int i = ii * cam.step, j = jj * cam.step;
        const float dep = cam.max_range;
        const float x = ((float)i - cam.cx) * dep / cam.fx;
        const float y = ((float)j - cam.cy) * dep / cam.fy;
        const float ex = ((R[0] * x + R[1] * y) + R[2] * dep) + px;
        const float ey = ((R[3] * x + R[4] * y) + R[5] * dep) + py;
        const float ez = ((R[6] * x + R[7] * y) + R[8] * dep) + pz;
        OcWalk w;
        oc_walk_begin(w, px / vs, py / vs, pz / vs, ex / vs, ey / vs, ez / vs);
        // the view's window, clipped to the volume
        const int lox = max(w.cx - cam.half, -g.hN), loy = max(w.cy - cam.half, -g.hN), loz = max(w.cz - cam.half, -g.hNz);
        const int nx = min(w.cx + cam.half, g.N - g.hN - 1) - lox + 1, ny = min(w.cy + cam.half, g.N - g.hN - 1) - loy + 1,
                  nz = min(w.cz + cam.half, g.Nz - g.hNz - 1) - loz + 1;
        uint32_t* bv = bits + (long long)vl * words;
        unsigned long long ckey = ~0ull;
        int cblk = -1;
        for (int left = w.lx + w.ly + w.lz;; --left) {
          if (!ts_in_bounds(g, w.cx, w.cy, w.cz)) break;
          const unsigned long long key = ts_pack_key(s, w.cx >> OC_BSHIFT, w.cy >> OC_BSHIFT, w.cz >> OC_BSHIFT);
          if (key != ckey) {  // hash probe only when the walk enters another block
            ckey = key;
            cblk = ts_find(g, key);
          }
          const int cl = ov_cell_class(g, cblk, w.cx, w.cy, w.cz, l_occ);
          if (cl == OC_OCC) break;
          if (cl == OC_UNK) {
            const int dx = w.cx - lox, dy = w.cy - loy, dz = w.cz - loz;
            if ((unsigned)dx >= (unsigned)nx || (unsigned)dy >= (unsigned)ny || (unsigned)dz >= (unsigned)nz) {
              atomicOr(g.err, OC_ERR_VIEW_WINDOW);  // never dropped silently: the next synchronising call reports it
            } else {
              const long long b = ((long long)dx * ny + dy) * nz + dz;
              uint32_t* wp = bv + (b >> 5);
              const uint32_t bit = 1u << (b & 31);
              // test-then-set: the rays of a view start in the same cell and fan out from it
              if (!(*(volatile uint32_t*)wp & bit) && !(atomicOr(wp, bit) & bit)) ++cnt;
            }
          }
          if (left == 0) break;
          oc_walk_step(w);
        }
      }
    }
    // the lanes of a warp that share a view add their counts first (a view's rays are consecutive lanes)
    unsigned todo = __ballot_sync(0xffffffffu, cnt > 0);
    while (todo) {
      const int leader = __ffs(todo) - 1;
      const long long lv = __shfl_sync(0xffffffffu, v, leader);
      const unsigned peers = __ballot_sync(0xffffffffu, cnt > 0 && v == lv);
      const unsigned sum = __reduce_add_sync(0xffffffffu, ((peers >> lane) & 1u) ? cnt : 0u);
      if (lane == leader) atomicAdd(&gain[lv], (unsigned long long)sum);
      todo &= ~peers;
    }
  }
}

// Frontier gain: one lane per (view, frontier row); rows of one view are consecutive lanes and mostly share a cluster
__global__ void __launch_bounds__(256) k_octo_view_frontier(OcGrid g, OvCam cam, int s, float vs, int l_occ, const float* __restrict__ pos,
                                                             const float* __restrict__ R9, const uint8_t* __restrict__ valid, long long n,
                                                             const int32_t* __restrict__ fidx, const int32_t* __restrict__ fcl, int nf,
                                                             int nc, int32_t* total, int32_t* per_cluster) {
  const long long pairs = n * nf;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  for (long long base = (long long)blockIdx.x * blockDim.x; base < pairs; base += stride) {  // uniform per warp
    const long long t = base + threadIdx.x;
    long long v = -1;
    int cl = -1;
    bool vis = false;
    if (t < pairs) {
      v = t / nf;
      const int r = (int)(t - v * nf);
      if (valid[v]) {
        const float* p = pos + 3 * v;
        const float* R = R9 + 9 * v;
        const float px = p[0], py = p[1], pz = p[2];
        const int ci = fidx[3 * (size_t)r], cj = fidx[3 * (size_t)r + 1], ck = fidx[3 * (size_t)r + 2];
        cl = fcl[r];
        const float xx = (float)ci * vs, xy = (float)cj * vs, xz = (float)ck * vs;
        const float dx = xx - px, dy = xy - py, dz = xz - pz;
        const float qx = (R[0] * dx + R[3] * dy) + R[6] * dz;  // q = R^T d
        const float qy = (R[1] * dx + R[4] * dy) + R[7] * dz;
        const float qz = (R[2] * dx + R[5] * dy) + R[8] * dz;
        if (qz > 0.0f && qz <= cam.max_range) {
          const float u = ((qx * cam.fx) / qz) + cam.cx, uv = ((qy * cam.fy) / qz) + cam.cy;
          if (u >= 0.0f && u <= cam.wmax && uv >= 0.0f && uv <= cam.hmax) {
            // line of sight: every cell of the path before the voxel's own cell must be FREE
            OcWalk w;
        oc_walk_begin(w, px / vs, py / vs, pz / vs, xx / vs, xy / vs, xz / vs);
            unsigned long long ckey = ~0ull;
            int cblk = -1;
            vis = true;
            for (int left = w.lx + w.ly + w.lz; left > 0; --left) {
              const unsigned long long key = ts_pack_key(s, w.cx >> OC_BSHIFT, w.cy >> OC_BSHIFT, w.cz >> OC_BSHIFT);
              if (key != ckey) {
                ckey = key;
                cblk = ts_find(g, key);
              }
              if (!ts_in_bounds(g, w.cx, w.cy, w.cz) || ov_cell_class(g, cblk, w.cx, w.cy, w.cz, l_occ) != OC_FREE) {
                vis = false;
                break;
              }
              oc_walk_step(w);
            }
          }
        }
      }
    }
    unsigned todo = __ballot_sync(0xffffffffu, vis);
    while (todo) {
      const int leader = __ffs(todo) - 1;
      const long long lv = __shfl_sync(0xffffffffu, v, leader);
      const int lc = __shfl_sync(0xffffffffu, cl, leader);
      const unsigned peers = __ballot_sync(0xffffffffu, vis && v == lv && cl == lc);
      if (lane == leader) {
        atomicAdd(&total[lv], __popc(peers));
        if (per_cluster) atomicAdd(&per_cluster[lv * nc + lc], __popc(peers));
      }
      todo &= ~peers;
    }
  }
}

// ---- host side -----------------------------------------------------------------------------------------------------
int oc_view_free(tslam_octo* m) {
  if (m->vw_mem) cudaFree(m->vw_mem);
  m->vw_mem = nullptr;
  m->vw_bytes = 0;
  return TSLAM_OK;
}

// The checks both calls share; fills the kernel's camera.  The window half-extent is ceil(r_max / vs) + 2 with r_max the
// largest |(x, y, dep)| over the image corners at dep = max_range (f64; a rotation keeps the length).
static int ov_check(tslam_octo* m, int32_t submap, int64_t n, const void* pos, const void* R9, const tslam_view_camera_t* cam,
                    const void* valid, const void* out, const char* what, OvCam& c) {
  if (!m || !cam || n < 0 || (n > 0 && (!pos || !R9 || !valid || !out))) return TSLAM_E_INVALID;
  const int rc = oc_logodds_submap(m, submap, what, "a viewpoint gain");
  if (rc) return rc;
  if (!(std::isfinite(cam->fx) && cam->fx > 0.0f && std::isfinite(cam->fy) && cam->fy > 0.0f && std::isfinite(cam->max_range) &&
        cam->max_range > 0.0f && std::isfinite(cam->cx) && std::isfinite(cam->cy))) {
    ts_set_error("%s: the camera needs finite fx, fy, max_range > 0 and finite cx, cy", what);
    return TSLAM_E_INVALID;
  }
  if (cam->width <= 0 || cam->height <= 0 || cam->step <= 0 || cam->width / cam->step == 0 || cam->height / cam->step == 0) {
    ts_set_error("%s: the camera needs width, height, step > 0 and at least one ray per row and column (got %d x %d, step %d)", what,
                 cam->width, cam->height, cam->step);
    return TSLAM_E_INVALID;
  }
  c.fx = cam->fx; c.fy = cam->fy; c.cx = cam->cx; c.cy = cam->cy; c.max_range = cam->max_range;
  c.wmax = (float)(cam->width - 1); c.hmax = (float)(cam->height - 1);
  c.ww = cam->width / cam->step; c.hh = cam->height / cam->step; c.step = cam->step;
  if ((long long)c.ww * c.hh > (1ll << 30)) { ts_set_error("%s: more than 2^30 rays per view", what); return TSLAM_E_INVALID; }
  const double dep = cam->max_range;
  double r2 = 0.0;
  for (int q = 0; q < 4; ++q) {
    const double x = ((double)((q & 1) ? (c.ww - 1) * c.step : 0) - cam->cx) * dep / cam->fx;
    const double y = ((double)((q & 2) ? (c.hh - 1) * c.step : 0) - cam->cy) * dep / cam->fy;
    r2 = std::fmax(r2, x * x + y * y + dep * dep);
  }
  const double half = std::ceil(std::sqrt(r2) / (double)m->in.vs) + 2.0;
  if (!(half <= (double)OV_MAX_HALF)) {
    ts_set_error("%s: the camera's farthest ray spans %.3g cells, more than 2^22", what, half);
    return TSLAM_E_INVALID;
  }
  c.half = (int)half;
  return TSLAM_OK;
}

// u32 words of one view's bitmap: the window's extent per axis is 2 * half + 1, at most the volume's
static long long ov_words(const tslam_octo* m, int half) {
  const long long e = 2ll * half + 1;
  const long long ex = e < m->g.N ? e : m->g.N, ez = e < m->g.Nz ? e : m->g.Nz;
  return (ex * ex * ez + 31) / 32;
}

extern "C" int tslam_octo_view_gain_unknown(tslam_octo_t* m, int32_t submap, int64_t n, const float* pos, const float* R9,
                                            const tslam_view_camera_t* cam, uint8_t* valid, int64_t* gain, void* stream) {
  OvCam c;
  int rc = ov_check(m, submap, n, pos, R9, cam, valid, gain, "tslam_octo_view_gain_unknown", c);
  if (rc || n == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const long long words = ov_words(m, c.half);
  unsigned long long budget = OV_SCRATCH_BYTES;
  if (const char* e = getenv("TSLAM_VIEW_SCRATCH")) budget = strtoull(e, nullptr, 10);
  long long chunk = (long long)(budget / ((unsigned long long)words * 4));
  if (chunk < 1) chunk = 1;
  if (chunk > n) chunk = n;
  rc = oc_reserve(&m->vw_mem, &m->vw_bytes, (size_t)(chunk * words * 4));
  if (rc) return rc;
  uint32_t* bits = (uint32_t*)m->vw_mem;
  TS_CUDA(cudaMemsetAsync(gain, 0, (size_t)n * 8, st));
  const int cap = m->sm_count * 16;
  k_octo_view_valid<<<oc_grid(n, 256, cap), 256, 0, st>>>(m->g, submap, m->in.vs, m->lo.l_occ, pos, R9, n, valid);
  TS_LAUNCH_CHECK(m);
  for (long long v0 = 0; v0 < n; v0 += chunk) {
    const int nv = (int)(n - v0 < chunk ? n - v0 : chunk);
    TS_CUDA(cudaMemsetAsync(bits, 0, (size_t)nv * words * 4, st));
    k_octo_view_unknown<<<oc_grid((long long)nv * c.ww * c.hh, 256, m->sm_count * 64), 256, 0, st>>>(
        m->g, c, submap, m->in.vs, m->lo.l_occ, pos, R9, valid, v0, nv, words, bits, (unsigned long long*)gain);
    TS_LAUNCH_CHECK(m);
  }
  return TSLAM_OK;
}

extern "C" int tslam_octo_view_gain_frontier(tslam_octo_t* m, int32_t submap, int64_t n, const float* pos, const float* R9,
                                             const tslam_view_camera_t* cam, int64_t n_clusters, uint8_t* valid, int32_t* total,
                                             int32_t* per_cluster, void* stream) {
  const char* what = "tslam_octo_view_gain_frontier";
  OvCam c;
  int rc = ov_check(m, submap, n, pos, R9, cam, valid, total, what, c);
  if (rc) return rc;
  rc = oc_track_readable(m, m->fr_track, submap, what, "tslam_octo_frontier_update");
  if (rc) return rc;
  if (n_clusters != m->fr_nc) {
    ts_set_error("%s: n_clusters = %lld, but the last tslam_octo_frontier_update found %d clusters", what, (long long)n_clusters, m->fr_nc);
    return TSLAM_E_INVALID;
  }
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  TS_CUDA(cudaMemsetAsync(total, 0, (size_t)n * 4, st));
  if (per_cluster && n_clusters > 0) TS_CUDA(cudaMemsetAsync(per_cluster, 0, (size_t)n * n_clusters * 4, st));
  const int cap = m->sm_count * 16;
  k_octo_view_valid<<<oc_grid(n, 256, cap), 256, 0, st>>>(m->g, submap, m->in.vs, m->lo.l_occ, pos, R9, n, valid);
  TS_LAUNCH_CHECK(m);
  const int nf = m->fr_n;
  if (nf == 0) return TSLAM_OK;
  rc = oc_reserve(&m->vw_mem, &m->vw_bytes, (size_t)nf * 16);
  if (rc) return rc;
  int32_t* fidx = (int32_t*)m->vw_mem;
  int32_t* fcl = fidx + 3 * (size_t)nf;
  rc = oc_frontier_rows(m, fidx, fcl, st);
  if (rc) return rc;
  k_octo_view_frontier<<<oc_grid(n * nf, 256, m->sm_count * 64), 256, 0, st>>>(m->g, c, submap, m->in.vs, m->lo.l_occ, pos, R9, valid, n,
                                                                          fidx, fcl, nf, (int)n_clusters, total, per_cluster);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
