// libtslam.so - batched map queries for planners: the reference exposes these as @ti.func helpers that
// TopoGraphGen calls from inside its own kernels (mapping_common.py:165-204, topo_graph.py:444-507);
// here they are stand-alone kernels over arrays of query points / rays.
#include "tslam_internal.cuh"

__device__ __forceinline__ int q_iround(float x) { return (int)roundf(x); }

// The planner queries are written once over a probe P of the map kind, which answers for a point (x, y, z):
//   flags(x, y, z)    bit0 occupied, bit1 unknown (TSDF: unobserved);
//   occ(x, y, z)      occupied (BaseMap.raycast's is_pos_occupy);
//   occ_cell(i, j, k) occupied, for cell (i, j, k) of the near-occupancy window.
// A kernel takes the probe's parts (grid, submap, voxel size, and its Param: the TSDF's surface threshold or the
// Octomap's occupancy rule) as parameters and builds the probe itself: the probe passed as one parameter costs up to 3
// registers more.

// DenseTSDF.is_occupy (dense_tsdf.py:152-155): TSDF[sijk] < tsdf_surface_thres - no observed test, and an
// inactive cell reads 0, so unobserved space counts as occupied.  is_unobserved (:148-150): observed == 0.
// Ghost blocks read as inactive unless Ghosts (the near-occupancy query of a tiled map, whose ghosts are current).
template <bool Ghosts = false>
struct TsdfProbe {
  using Grid = TsGrid;
  using Param = float;  // tsdf_surface_thres
  TsGrid g;
  int s;
  float vs, thres;
  __device__ __forceinline__ void read(float x, float y, float z, float& t, int& o) const {
    int c[3];
    t = 0.0f;
    o = 0;
    if (ts_query_cell(g, x, y, z, vs, c)) ts_query_read<Ghosts>(g, s, c, t, o);  // sxyz_to_ijk mapping_common.py:257-261
  }
  __device__ __forceinline__ unsigned flags(float x, float y, float z) const {
    float t;
    int o;
    read(x, y, z, t, o);
    return (t < thres ? 1u : 0u) | (o == 0 ? 2u : 0u);
  }
  __device__ __forceinline__ bool occ(float x, float y, float z) const {
    float t;
    int o;
    read(x, y, z, t, o);
    return t < thres;
  }
  // re-probes the cell's centre: (i * vs) / vs re-rounds to i, exact for |i| < 2^22
  __device__ __forceinline__ bool occ_cell(int i, int j, int k) const { return occ((float)i * vs, (float)j * vs, (float)k * vs); }
};

// Word of cell (i, j, k) of submap s of an Octomap: 0 (no hits / unknown) outside the volume and in absent blocks
__device__ __forceinline__ unsigned int oc_cell_word(const OcGrid& g, int s, int i, int j, int k) {
  unsigned int c = 0;
  if (ts_in_bounds(g, i, j, k)) {
    const int blk = ts_find(g, ts_pack_key(s, i >> OC_BSHIFT, j >> OC_BSHIFT, k >> OC_BSHIFT));
    if (blk >= 0) c = g.cnt[(size_t)blk * OC_B3 + oc_voxel_off(i, j, k)];
  }
  return c;
}
// Octomap.is_occupy (taichi_octomap.py:86-88) under the map's occupancy rule (OcHits / OcLogodds).  On a log-odds map
// unknown space is not occupied, so a ray passes through it.
template <class R>
struct OcProbe {
  using Grid = OcGrid;
  using Param = R;
  OcGrid g;
  int s;
  float vs;
  R rule;
  __device__ __forceinline__ unsigned int word(float x, float y, float z) const {
    return oc_cell_word(g, s, q_iround(x / vs), q_iround(y / vs), q_iround(z / vs));
  }
  __device__ __forceinline__ unsigned flags(float x, float y, float z) const {
    const unsigned int c = word(x, y, z);
    return (rule.occ(c) ? 1u : 0u) | (rule.unknown(c) ? 2u : 0u);
  }
  __device__ __forceinline__ bool occ(float x, float y, float z) const { return rule.occ(word(x, y, z)); }
  __device__ __forceinline__ bool occ_cell(int i, int j, int k) const { return rule.occ(oc_cell_word(g, s, i, j, k)); }
};

template <class P>
__global__ void __launch_bounds__(256) k_query_points(typename P::Grid g, int s, long long n, const float* __restrict__ xyz, float vs,
                                                      typename P::Param param, uint8_t* flags) {
  const P p{g, s, vs, param};
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x)
    flags[q] = (uint8_t)p.flags(xyz[3 * q], xyz[3 * q + 1], xyz[3 * q + 2]);
}

// is_near_pos_occupy (mapping_common.py:193-204): any occupied cell (i0 + a, j0 + b, k0 + c), a, b, c in [-voxel, voxel),
// around the point's cell.  TsdfProbe<true>: ghost blocks are read like owned ones (a tiled map after a halo exchange,
// voxel <= 16: the window stays in the 3^3 blocks around the centre cell's block, and the halo carries every one of them
// that lies in a foreign tile).
template <class P>
__global__ void __launch_bounds__(256) k_query_near(typename P::Grid g, int s, long long n, const float* __restrict__ xyz, float vs,
                                                    typename P::Param param, int voxel, uint8_t* out) {
  const P p{g, s, vs, param};
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const int i0 = q_iround(xyz[3 * q] / vs), j0 = q_iround(xyz[3 * q + 1] / vs), k0 = q_iround(xyz[3 * q + 2] / vs);
    bool any = false;
    for (int i = -voxel; i < voxel && !any; i++)
      for (int j = -voxel; j < voxel && !any; j++)
        for (int k = -voxel; k < voxel && !any; k++) any = p.occ_cell(i0 + i, j0 + j, k0 + k);
    out[q] = any ? 1 : 0;
  }
}

// BaseMap.raycast (mapping_common.py:165-178): march in voxel_scale steps until is_pos_occupy.  A miss reports the last
// sample's position and length.
template <class P>
__global__ void __launch_bounds__(256) k_raycast(typename P::Grid g, int s, long long n, const float* __restrict__ pos,
                                                 const float* __restrict__ dir, float max_dist, float vs, typename P::Param param, uint8_t* hit,
                                                 float* xyz_out, float* len_out) {
  const P p{g, s, vs, param};
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const float3 org = make_float3(pos[3 * q], pos[3 * q + 1], pos[3 * q + 2]);
    const float3 dr = make_float3(dir[3 * q], dir[3 * q + 1], dir[3 * q + 2]);
    const int steps = raycast_steps(max_dist, vs);
    float x = 0.f, y = 0.f, z = 0.f, len = 0.f;
    bool succ = false;
    for (int j = 0; j < steps; j++) {
      raycast_sample(org, dr, j, vs, x, y, z, len);
      if (p.occ(x, y, z)) { succ = true; break; }  // :175-177
    }
    hit[q] = succ ? 1 : 0;
    xyz_out[3 * q] = x; xyz_out[3 * q + 1] = y; xyz_out[3 * q + 2] = z;
    len_out[q] = len;
  }
}

static int grid_for(long long n, int sm) {
  long long b = (n + 255) / 256;
  return (int)(b < (long long)sm * 16 ? (b > 0 ? b : 1) : (long long)sm * 16);
}

// tsdf_surface_thres (dense_tsdf.py:39)
static float tsdf_thres(const tslam_tsdf* m) { return (float)(m->cfg.voxel_scale * 1.8); }

extern "C" int tslam_tsdf_query_points(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* xyz, uint8_t* flags, void* stream) {
  if (!m || n < 0 || (n && (!xyz || !flags))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  k_query_points<TsdfProbe<>><<<grid_for(n, m->sm_count), 256, 0, st>>>(m->g, submap, n, xyz, m->in.vs, tsdf_thres(m), flags);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
extern "C" int tslam_tsdf_query_near_occupy(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* xyz, int32_t voxel, uint8_t* out, void* stream) {
  if (!m || n < 0 || voxel < 0 || (n && (!xyz || !out))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  k_query_near<TsdfProbe<false>><<<grid_for(n, m->sm_count), 256, 0, st>>>(m->g, submap, n, xyz, m->in.vs, tsdf_thres(m), voxel, out);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
extern "C" int tslam_tsdf_query_near_occupy_tiled(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* xyz, int32_t voxel, uint8_t* out,
                                                  void* stream) {
  if (!m || n < 0 || (n && (!xyz || !out))) return TSLAM_E_INVALID;
  if (voxel < 0 || voxel > TS_B) {
    ts_set_error("tslam_tsdf_query_near_occupy_tiled: voxel %d outside [0, %d] (the halo holds one block)", voxel, TS_B);
    return TSLAM_E_INVALID;
  }
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  k_query_near<TsdfProbe<true>><<<grid_for(n, m->sm_count), 256, 0, st>>>(m->g, submap, n, xyz, m->in.vs, tsdf_thres(m), voxel, out);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
extern "C" int tslam_tsdf_raycast(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* pos, const float* dir, float max_dist,
                                  uint8_t* hit, float* xyz_out, float* len_out, void* stream) {
  if (!m || n < 0 || (n && (!pos || !dir || !hit || !xyz_out || !len_out))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  k_raycast<TsdfProbe<>><<<grid_for(n, m->sm_count), 256, 0, st>>>(m->g, submap, n, pos, dir, max_dist, m->in.vs, tsdf_thres(m), hit,
                                                                 xyz_out, len_out);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
extern "C" int tslam_octo_query_points(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, uint8_t* flags, void* stream) {
  if (!m || n < 0 || (n && (!xyz || !flags))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  oc_with_rule(m, [&](auto rule) {
    k_query_points<OcProbe<decltype(rule)>><<<grid_for(n, m->sm_count), 256, 0, (cudaStream_t)stream>>>(m->g, submap, n, xyz, m->in.vs, rule, flags);
  });
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
extern "C" int tslam_octo_raycast(tslam_octo_t* m, int32_t submap, int64_t n, const float* pos, const float* dir, float max_dist, uint8_t* hit,
                                  float* xyz_out, float* len_out, void* stream) {
  if (!m || n < 0 || (n && (!pos || !dir || !hit || !xyz_out || !len_out))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  oc_with_rule(m, [&](auto rule) {
    k_raycast<OcProbe<decltype(rule)>><<<grid_for(n, m->sm_count), 256, 0, (cudaStream_t)stream>>>(m->g, submap, n, pos, dir, max_dist, m->in.vs,
                                                                                                   rule, hit, xyz_out, len_out);
  });
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
extern "C" int tslam_octo_query_near_occupy(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, int32_t voxel, uint8_t* out, void* stream) {
  if (!m || n < 0 || voxel < 0 || (n && (!xyz || !out))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  oc_with_rule(m, [&](auto rule) {
    k_query_near<OcProbe<decltype(rule)>><<<grid_for(n, m->sm_count), 256, 0, (cudaStream_t)stream>>>(m->g, submap, n, xyz, m->in.vs, rule, voxel,
                                                                                                      out);
  });
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
