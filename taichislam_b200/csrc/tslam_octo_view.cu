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
//   frontier viewpoints  (DESIGN.md section 7, "Frontier viewpoints") candidate (c, s) = cluster c's f32 centroid plus
//                  offset s, a level camera facing the centroid; valid iff finite, off the centroid's vertical and on a
//                  traversable cell (oc_traversable); scored by the frontier gain's test (ov_sees) against cluster c's
//                  own rows (grouped by cluster with a counting scatter), one warp per chunk of 64 rows of a valid
//                  candidate; the top_k per cluster by (score desc, s asc).
// None writes the map: blocks are looked up with ts_find (no allocation) and no mark, touched list, dirty flag or
// stats counter is touched.  Every output is an integer count, so the result does not depend on the thread schedule.
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cub/device/device_scan.cuh>
#include "tslam_internal.cuh"

#define OV_SCRATCH_BYTES (256ull << 20)  // bitmap budget per chunk of views (TSLAM_VIEW_SCRATCH overrides); >= 1 view
#define OV_MAX_HALF (1 << 22)            // largest window half-extent in cells: cell indices stay far from int overflow
#define OVP_CHUNK 64                     // frontier rows per scoring item of a frontier viewpoint (two per lane)

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

// Whether the view (p, R) sees frontier voxel (ci, cj, ck): its centre x = f32(c) * vs lies in the frustum (q = R^T (x - p)
// with 0 < q_z <= max_range, projected inside the image), and every cell of the walk from p to x before the voxel's own
// cell is inside the volume and FREE.  The frontier gain and the frontier viewpoints count with it.
__device__ __forceinline__ bool ov_sees(const OcGrid& g, const OvCam& cam, int s, float vs, int l_occ, float px, float py, float pz,
                                        const float* R, int ci, int cj, int ck) {
  const float xx = (float)ci * vs, xy = (float)cj * vs, xz = (float)ck * vs;
  const float dx = xx - px, dy = xy - py, dz = xz - pz;
  const float qx = (R[0] * dx + R[3] * dy) + R[6] * dz;  // q = R^T d
  const float qy = (R[1] * dx + R[4] * dy) + R[7] * dz;
  const float qz = (R[2] * dx + R[5] * dy) + R[8] * dz;
  if (!(qz > 0.0f && qz <= cam.max_range)) return false;
  const float u = ((qx * cam.fx) / qz) + cam.cx, uv = ((qy * cam.fy) / qz) + cam.cy;
  if (!(u >= 0.0f && u <= cam.wmax && uv >= 0.0f && uv <= cam.hmax)) return false;
  // line of sight: every cell of the path before the voxel's own cell must be FREE
  OcWalk w;
  oc_walk_begin(w, px / vs, py / vs, pz / vs, xx / vs, xy / vs, xz / vs);
  unsigned long long ckey = ~0ull;
  int cblk = -1;
  for (int left = w.lx + w.ly + w.lz; left > 0; --left) {
    const unsigned long long key = ts_pack_key(s, w.cx >> OC_BSHIFT, w.cy >> OC_BSHIFT, w.cz >> OC_BSHIFT);
    if (key != ckey) {
      ckey = key;
      cblk = ts_find(g, key);
    }
    if (!ts_in_bounds(g, w.cx, w.cy, w.cz) || ov_cell_class(g, cblk, w.cx, w.cy, w.cz, l_occ) != OC_FREE) return false;
    oc_walk_step(w);
  }
  return true;
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
        const float px = p[0], py = p[1], pz = p[2];
        const int ci = fidx[3 * (size_t)r], cj = fidx[3 * (size_t)r + 1], ck = fidx[3 * (size_t)r + 2];
        cl = fcl[r];
        vis = ov_sees(g, cam, s, vs, l_occ, px, py, pz, R9 + 9 * v, ci, cj, ck);
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

// ---- frontier viewpoints -------------------------------------------------------------------------------------------
// Candidate (c, s) of the frontier viewpoints: p = m_c + off[s] (f32 adds) with m_c the cluster's f32 centroid, and the
// level camera facing m_c: with (dx, dy) = m - p, h = sqrtf(dx^2 + dy^2), u = (dx, dy) / h, R = [[uy, 0, ux], [-ux, 0,
// uy], [0, -1, 0]] (camera z = (ux, uy, 0), x = (uy, -ux, 0), y = (0, 0, -1)).  False when p is not finite or h == 0.
__device__ __forceinline__ bool ovp_pose(const float* __restrict__ cen, const float* __restrict__ off, int c, int s, float p[3], float R[9]) {
  const float mx = cen[3 * c], my = cen[3 * c + 1], mz = cen[3 * c + 2];
  p[0] = mx + off[3 * s]; p[1] = my + off[3 * s + 1]; p[2] = mz + off[3 * s + 2];
  const float dx = mx - p[0], dy = my - p[1];
  const float h = sqrtf(dx * dx + dy * dy);
  const float ux = dx / h, uy = dy / h;
  R[0] = uy;  R[1] = 0.0f;  R[2] = ux;
  R[3] = -ux; R[4] = 0.0f;  R[5] = uy;
  R[6] = 0.0f; R[7] = -1.0f; R[8] = 0.0f;
  return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]) && h > 0.0f;
}

// Per cluster ordinal c: its voxel count cnt[c] (cnt[nc] = 0, for the exclusive scan) and its f32 centroid
// m_a = (float)((double)sum_a / (double)n * (double)vs), the f32 rounding of get_frontier_clusters' centroid
__global__ void __launch_bounds__(256) k_octo_viewpoint_clusters(const int64_t* __restrict__ rec, int nc, float vs, int* cnt, float* cen) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c <= nc; c += gridDim.x * blockDim.x) {
    if (c == nc) { cnt[c] = 0; continue; }
    const int64_t* r = rec + 16 * (size_t)c;
    cnt[c] = (int)r[1];
    for (int a = 0; a < 3; ++a) cen[3 * c + a] = (float)((double)r[2 + a] / (double)r[1] * (double)vs);
  }
}

// The frontier rows grouped by cluster ordinal: row r goes to [coff[cl], coff[cl + 1]) (any order within a cluster; the
// scores are counts)
__global__ void __launch_bounds__(256) k_octo_viewpoint_scatter(const int32_t* __restrict__ fidx, const int32_t* __restrict__ fcl, int nf,
                                                                 const int* __restrict__ coff, int* cur, int32_t* sidx) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nf; r += gridDim.x * blockDim.x) {
    const int cl = fcl[r];
    const int q = coff[cl] + atomicAdd(&cur[cl], 1);
    sidx[3 * (size_t)q] = fidx[3 * (size_t)r];
    sidx[3 * (size_t)q + 1] = fidx[3 * (size_t)r + 1];
    sidx[3 * (size_t)q + 2] = fidx[3 * (size_t)r + 2];
  }
}

// One thread per candidate id = c * S + s: when it is valid (ovp_pose, and its cell rha(p / vs) traversable under
// oc_traversable), vis[id] = 0 and the items (id, q) for the chunks q of OVP_CHUNK rows of cluster c go to `items`;
// else vis[id] = -1
__global__ void __launch_bounds__(256) k_octo_viewpoint_candidates(OcGrid g, OcEsdfField ef, int submap, float vs, int l_occ, float clearance,
                                                                    const float* __restrict__ cen, const float* __restrict__ off, int S, int n,
                                                                    const int* __restrict__ coff, int* vis, int2* items, int* ctr) {
  const bool clear = clearance > 0.0f;
  const int enb = clear ? *ef.nb_seen : 0;
  for (int id = blockIdx.x * blockDim.x + threadIdx.x; id < n; id += gridDim.x * blockDim.x) {
    float p[3], R[9];
    bool ok = ovp_pose(cen, off, id / S, id % S, p, R);
    if (ok) {
      const float u0 = p[0] / vs, u1 = p[1] / vs, u2 = p[2] / vs;
      ok = fabsf(u0) < 1e9f && fabsf(u1) < 1e9f && fabsf(u2) < 1e9f;  // no out-of-range float -> int conversion below
      if (ok) {
        const int i = (int)roundf(u0), j = (int)roundf(u1), k = (int)roundf(u2);
        ok = ts_in_bounds(g, i, j, k);
        if (ok) {
          const int b = ts_find(g, ts_pack_key(submap, i >> OC_BSHIFT, j >> OC_BSHIFT, k >> OC_BSHIFT));
          const size_t o = (size_t)(b < 0 ? 0 : b) * OC_B3 + oc_voxel_off(i, j, k);
          ok = b >= 0 && oc_traversable(g, ef, l_occ, clearance, clear, enb, b, o, g.cnt[o], i, j, k);
        }
      }
    }
    vis[id] = ok ? 0 : -1;
    if (ok) {
      const int c = id / S, nq = (coff[c + 1] - coff[c] + OVP_CHUNK - 1) / OVP_CHUNK;
      const int at = atomicAdd(ctr, nq);
      for (int q = 0; q < nq; ++q) items[at + q] = make_int2(id, q);
    }
  }
}

// One warp per item (candidate, chunk): its lanes test the chunk's rows of the candidate's own cluster with ov_sees, and
// the warp adds its count to vis[id].  A candidate of a large cluster spreads over many warps; the sum of integer
// additions does not depend on their order.
__global__ void __launch_bounds__(256) k_octo_viewpoint_score(OcGrid g, OvCam cam, int submap, float vs, int l_occ, const float* __restrict__ cen,
                                                               const float* __restrict__ off, int S, const int2* __restrict__ items,
                                                               const int* __restrict__ ctr, const int* __restrict__ coff,
                                                               const int32_t* __restrict__ sidx, int* vis) {
  const int lane = threadIdx.x & 31;
  const int n = *ctr;
  for (int wi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; wi < n; wi += (gridDim.x * blockDim.x) >> 5) {
    const int2 it = items[wi];
    const int c = it.x / S;
    float p[3], R[9];
    ovp_pose(cen, off, c, it.x - c * S, p, R);
    const int r0 = coff[c] + it.y * OVP_CHUNK, r1 = min(r0 + OVP_CHUNK, coff[c + 1]);
    unsigned cnt = 0;
    for (int r = r0 + lane; r < r1; r += 32)
      cnt += ov_sees(g, cam, submap, vs, l_occ, p[0], p[1], p[2], R, sidx[3 * (size_t)r], sidx[3 * (size_t)r + 1], sidx[3 * (size_t)r + 2]) ? 1u : 0u;
    const unsigned sum = __reduce_add_sync(0xffffffffu, cnt);
    if (lane == 0 && sum) atomicAdd(&vis[it.x], (int)sum);
  }
}

// One CTA per cluster: the kept candidates (vis >= min_visible) ranked by (vis descending, s ascending); rank q < top_k
// goes to slot q, and slots [min(top_k, kept), top_k) are cleared (sample -1, visible 0, zero pose)
__global__ void __launch_bounds__(256) k_octo_viewpoint_select(const float* __restrict__ cen, const float* __restrict__ off, int S, int nc,
                                                                int min_visible, int top_k, const int* __restrict__ vis, int32_t* count,
                                                                int32_t* sample, int32_t* visible, float* pos, float* R9) {
  __shared__ int key[TSLAM_OCTO_VIEWPOINT_MAX_SAMPLES];
  __shared__ int kept;
  for (int c = blockIdx.x; c < nc; c += gridDim.x) {
    __syncthreads();  // the previous cluster's keys are read
    if (threadIdx.x == 0) kept = 0;
    int mine = 0;
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
      const int v = vis[(size_t)c * S + s];
      key[s] = v >= min_visible ? v : -1;
      mine += v >= min_visible ? 1 : 0;
    }
    __syncthreads();
    if (mine) atomicAdd(&kept, mine);
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
      const int ks = key[s];
      if (ks < 0) continue;
      int rank = 0;
      for (int t = 0; t < S && rank < top_k; ++t) {
        const int kt = key[t];
        rank += (kt > ks || (kt == ks && t < s)) ? 1 : 0;
      }
      if (rank >= top_k) continue;
      const size_t q = (size_t)c * top_k + rank;
      float p[3], R[9];
      ovp_pose(cen, off, c, s, p, R);
      sample[q] = s;
      visible[q] = ks;
      for (int a = 0; a < 3; ++a) pos[3 * q + a] = p[a];
      for (int a = 0; a < 9; ++a) R9[9 * q + a] = R[a];
    }
    __syncthreads();
    const int n_out = min(kept, top_k);
    if (threadIdx.x == 0) count[c] = n_out;
    for (int j = n_out + threadIdx.x; j < top_k; j += blockDim.x) {
      const size_t q = (size_t)c * top_k + j;
      sample[q] = -1;
      visible[q] = 0;
      for (int a = 0; a < 3; ++a) pos[3 * q + a] = 0.0f;
      for (int a = 0; a < 9; ++a) R9[9 * q + a] = 0.0f;
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

static int ov_camera(tslam_octo* m, const tslam_view_camera_t* cam, const char* what, OvCam& c);

// The checks both calls share; fills the kernel's camera
static int ov_check(tslam_octo* m, int32_t submap, int64_t n, const void* pos, const void* R9, const tslam_view_camera_t* cam,
                    const void* valid, const void* out, const char* what, OvCam& c) {
  if (!m || !cam || n < 0 || (n > 0 && (!pos || !R9 || !valid || !out))) return TSLAM_E_INVALID;
  const int rc = oc_logodds_submap(m, submap, what, "a viewpoint gain");
  if (rc) return rc;
  return ov_camera(m, cam, what, c);
}

// The camera checks of every view call; fills the kernel's camera.  The window half-extent is ceil(r_max / vs) + 2 with
// r_max the largest |(x, y, dep)| over the image corners at dep = max_range (f64; a rotation keeps the length).
static int ov_camera(tslam_octo* m, const tslam_view_camera_t* cam, const char* what, OvCam& c) {
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

// 256-byte aligned carving of the frontier-viewpoint scratch
static size_t ovp_align(size_t b) { return (b + 255) & ~(size_t)255; }

extern "C" int tslam_octo_frontier_viewpoints(tslam_octo_t* m, int32_t submap, const tslam_view_camera_t* cam, int32_t n_samples,
                                              const float* offsets, float clearance, int32_t min_visible, int32_t top_k, int64_t n_clusters,
                                              int32_t* count, int32_t* sample, int32_t* visible, float* pos, float* R9, void* stream) {
  const char* what = "tslam_octo_frontier_viewpoints";
  if (!m || !cam || !offsets || (n_clusters > 0 && (!count || !sample || !visible || !pos || !R9))) return TSLAM_E_INVALID;
  int rc = oc_logodds_submap(m, submap, what, "frontier viewpoints");
  if (rc) return rc;
  if (n_samples < 1 || n_samples > TSLAM_OCTO_VIEWPOINT_MAX_SAMPLES || top_k < 1 || top_k > TSLAM_OCTO_VIEWPOINT_MAX_SAMPLES) {
    ts_set_error("%s: n_samples and top_k must be in [1, %d] (got %d, %d)", what, TSLAM_OCTO_VIEWPOINT_MAX_SAMPLES, n_samples, top_k);
    return TSLAM_E_INVALID;
  }
  if (min_visible < 1) { ts_set_error("%s: min_visible must be >= 1 (got %d)", what, min_visible); return TSLAM_E_INVALID; }
  OvCam c;
  rc = ov_camera(m, cam, what, c);
  if (rc) return rc;
  OcEsdfField ef;
  rc = oc_clearance_field(m, submap, clearance, what, &ef);
  if (rc) return rc;
  rc = oc_track_readable(m, m->fr_track, submap, what, "tslam_octo_frontier_update");
  if (rc) return rc;
  if (n_clusters != m->fr_nc) {
    ts_set_error("%s: n_clusters = %lld, but the last tslam_octo_frontier_update found %d clusters", what, (long long)n_clusters, m->fr_nc);
    return TSLAM_E_INVALID;
  }
  if (n_clusters == 0) return TSLAM_OK;
  const int nc = (int)n_clusters, S = n_samples, nf = m->fr_n;
  const long long n = (long long)nc * S;
  const long long n_items = (long long)S * ((nf + OVP_CHUNK - 1) / OVP_CHUNK + nc);  // >= the sum over candidates of their chunks
  if (n_items > INT_MAX) {
    ts_set_error("%s: %d clusters x %d samples exceed 2^31 candidates or scoring items", what, nc, S);
    return TSLAM_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  size_t tb = 0;
  TS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, (int*)nullptr, (int*)nullptr, nc + 1, st));
  // scratch: records, centroids, counts, offsets, cursors, item counter, frontier rows, grouped rows, scores, items, CUB
  const size_t sz[] = {(size_t)nc * 16 * 8, (size_t)nc * 3 * 4, (size_t)(nc + 1) * 4, (size_t)(nc + 1) * 4, (size_t)nc * 4, 16,
                       (size_t)nf * 16, (size_t)nf * 12, (size_t)n * 4, (size_t)n_items * 8, tb};
  size_t at[sizeof(sz) / sizeof(sz[0]) + 1] = {0};
  for (size_t q = 0; q < sizeof(sz) / sizeof(sz[0]); ++q) at[q + 1] = at[q] + ovp_align(sz[q]);
  rc = oc_reserve(&m->vw_mem, &m->vw_bytes, at[sizeof(sz) / sizeof(sz[0])]);
  if (rc) return rc;
  char* base = (char*)m->vw_mem;
  int64_t* rec = (int64_t*)(base + at[0]);
  float* cen = (float*)(base + at[1]);
  int* cnt = (int*)(base + at[2]);
  int* coff = (int*)(base + at[3]);
  int* cur = (int*)(base + at[4]);
  int* ctr = (int*)(base + at[5]);
  int32_t* fidx = (int32_t*)(base + at[6]);
  int32_t* fcl = fidx + 3 * (size_t)nf;
  int32_t* sidx = (int32_t*)(base + at[7]);
  int* vis = (int*)(base + at[8]);
  int2* items = (int2*)(base + at[9]);
  void* tmp = base + at[10];
  TS_CUDA(cudaMemsetAsync(cur, 0, at[6] - at[4], st));  // cursors and the item counter
  rc = oc_frontier_records(m, rec, st);
  if (rc) return rc;
  rc = oc_frontier_rows(m, fidx, fcl, st);
  if (rc) return rc;
  const int cap = m->sm_count * 16;
  k_octo_viewpoint_clusters<<<oc_grid(nc + 1, 256, cap), 256, 0, st>>>(rec, nc, m->in.vs, cnt, cen);
  TS_LAUNCH_CHECK(m);
  TS_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, coff, nc + 1, st));
  k_octo_viewpoint_scatter<<<oc_grid(nf, 256, cap), 256, 0, st>>>(fidx, fcl, nf, coff, cur, sidx);
  TS_LAUNCH_CHECK(m);
  k_octo_viewpoint_candidates<<<oc_grid(n, 256, cap), 256, 0, st>>>(m->g, ef, submap, m->in.vs, m->lo.l_occ, clearance, cen, offsets, S,
                                                                     (int)n, coff, vis, items, ctr);
  TS_LAUNCH_CHECK(m);
  k_octo_viewpoint_score<<<oc_grid(n_items * 32, 256, m->sm_count * 64), 256, 0, st>>>(m->g, c, submap, m->in.vs, m->lo.l_occ, cen, offsets,
                                                                                        S, items, ctr, coff, sidx, vis);
  TS_LAUNCH_CHECK(m);
  k_octo_viewpoint_select<<<oc_grid(nc, 1, cap), 256, 0, st>>>(cen, offsets, S, nc, min_visible, top_k, vis, count, sample, visible, pos, R9);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
