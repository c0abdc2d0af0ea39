// libtslam.so - batched map queries for planners: the reference exposes these as @ti.func helpers that
// TopoGraphGen calls from inside its own kernels (mapping_common.py:165-204, topo_graph.py:444-507);
// here they are stand-alone kernels over arrays of query points / rays.
#include "tslam_internal.cuh"

__device__ __forceinline__ int q_iround(float x) { return (int)roundf(x); }

// DenseTSDF.is_occupy (dense_tsdf.py:152-155): TSDF[sijk] < tsdf_surface_thres - no observed test, and an
// inactive cell reads 0, so unobserved space counts as occupied.  is_unobserved (:148-150): observed == 0.
// Ghost blocks read as inactive unless Ghosts (the near-occupancy query of a tiled map, whose ghosts are current).
template <bool Ghosts = false>
__device__ __forceinline__ void tsdf_probe(const TsGrid& g, int s, float x, float y, float z, float vs, float thres, bool& occ, bool& unobs) {
  int c[3];
  float t = 0.0f;
  int o = 0;
  if (ts_query_cell(g, x, y, z, vs, c)) ts_query_read<Ghosts>(g, s, c, t, o);  // sxyz_to_ijk mapping_common.py:257-261
  occ = t < thres;
  unobs = o == 0;
}

__global__ void __launch_bounds__(256) k_tsdf_query_points(TsGrid g, int s, long long n, const float* __restrict__ xyz, float vs, float thres,
                                                            uint8_t* flags) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    bool occ, un;
    tsdf_probe(g, s, xyz[3 * q], xyz[3 * q + 1], xyz[3 * q + 2], vs, thres, occ, un);
    flags[q] = (uint8_t)((occ ? 1 : 0) | (un ? 2 : 0));
  }
}

// is_near_pos_occupy (mapping_common.py:193-204): any occupied cell in [-voxel, voxel)^3 around the point's cell.
// Ghosts: ghost blocks are read like owned ones (a tiled map after a halo exchange, voxel <= 16: the window stays in
// the 3^3 blocks around the centre cell's block, and the halo carries every one of them that lies in a foreign tile).
template <bool Ghosts>
__global__ void __launch_bounds__(256) k_tsdf_query_near(TsGrid g, int s, long long n, const float* __restrict__ xyz, float vs, float thres,
                                                          int voxel, uint8_t* out) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const int i0 = q_iround(xyz[3 * q] / vs), j0 = q_iround(xyz[3 * q + 1] / vs), k0 = q_iround(xyz[3 * q + 2] / vs);
    bool any = false;
    for (int i = -voxel; i < voxel && !any; i++)
      for (int j = -voxel; j < voxel && !any; j++)
        for (int k = -voxel; k < voxel && !any; k++) {
          bool occ, un;
          tsdf_probe<Ghosts>(g, s, (float)(i0 + i) * vs, (float)(j0 + j) * vs, (float)(k0 + k) * vs, vs, thres, occ, un);
          // (probe re-rounds (i0+i)*vs/vs; exact for |index| < 2^22)
          any = occ;
        }
    out[q] = any ? 1 : 0;
  }
}

// BaseMap.raycast (mapping_common.py:165-178): march in voxel_scale steps until is_pos_occupy.
__global__ void __launch_bounds__(256) k_tsdf_raycast(TsGrid g, int s, long long n, const float* __restrict__ pos, const float* __restrict__ dir,
                                                       float max_dist, float vs, float thres, uint8_t* hit, float* xyz_out, float* len_out) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const float px = pos[3 * q], py = pos[3 * q + 1], pz = pos[3 * q + 2];
    const float dx = dir[3 * q], dy = dir[3 * q + 1], dz = dir[3 * q + 2];
    const int steps = (int)(max_dist / vs);  // :167, range(float) truncates
    float x = 0.f, y = 0.f, z = 0.f, len = 0.f;
    bool succ = false;
    for (int j = 0; j < steps; j++) {
      len = (float)j * vs;                       // :173
      x = dx * len + px; y = dy * len + py; z = dz * len + pz;  // :174
      bool occ, un;
      tsdf_probe(g, s, x, y, z, vs, thres, occ, un);
      if (occ) { succ = true; break; }           // :175-177
    }
    hit[q] = succ ? 1 : 0;
    xyz_out[3 * q] = x; xyz_out[3 * q + 1] = y; xyz_out[3 * q + 2] = z;
    len_out[q] = len;
  }
}

// Octomap.is_occupy (taichi_octomap.py:86-88): occupy > min_occupy_thres
__device__ __forceinline__ bool octo_probe(const OcGrid& g, int s, float x, float y, float z, float vs, float thres) {
  const int i = q_iround(x / vs), j = q_iround(y / vs), k = q_iround(z / vs);
  unsigned int c = 0;
  if (ts_in_bounds(g, i, j, k)) {
    const int blk = ts_find(g, ts_pack_key(s, i >> OC_BSHIFT, j >> OC_BSHIFT, k >> OC_BSHIFT));
    if (blk >= 0) c = g.cnt[(size_t)blk * OC_B3 + oc_voxel_off(i, j, k)];
  }
  return (float)c > thres;
}
__global__ void __launch_bounds__(256) k_octo_query_points(OcGrid g, int s, long long n, const float* __restrict__ xyz, float vs, float thres,
                                                            uint8_t* flags) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x)
    flags[q] = octo_probe(g, s, xyz[3 * q], xyz[3 * q + 1], xyz[3 * q + 2], vs, thres) ? 1 : 0;
}
__global__ void __launch_bounds__(256) k_octo_raycast(OcGrid g, int s, long long n, const float* __restrict__ pos, const float* __restrict__ dir,
                                                       float max_dist, float vs, float thres, uint8_t* hit, float* xyz_out, float* len_out) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const float px = pos[3 * q], py = pos[3 * q + 1], pz = pos[3 * q + 2];
    const float dx = dir[3 * q], dy = dir[3 * q + 1], dz = dir[3 * q + 2];
    const int steps = (int)(max_dist / vs);
    float x = 0.f, y = 0.f, z = 0.f, len = 0.f;
    bool succ = false;
    for (int j = 0; j < steps; j++) {
      len = (float)j * vs;
      x = dx * len + px; y = dy * len + py; z = dz * len + pz;
      if (octo_probe(g, s, x, y, z, vs, thres)) { succ = true; break; }
    }
    hit[q] = succ ? 1 : 0;
    xyz_out[3 * q] = x; xyz_out[3 * q + 1] = y; xyz_out[3 * q + 2] = z;
    len_out[q] = len;
  }
}

// Word of cell (i, j, k) of submap s of a log-odds map: 0 (unknown) outside the volume and in absent blocks
__device__ __forceinline__ unsigned int octo_lo_word(const OcGrid& g, int s, int i, int j, int k) {
  unsigned int c = 0;
  if (ts_in_bounds(g, i, j, k)) {
    const int blk = ts_find(g, ts_pack_key(s, i >> OC_BSHIFT, j >> OC_BSHIFT, k >> OC_BSHIFT));
    if (blk >= 0) c = g.cnt[(size_t)blk * OC_B3 + oc_voxel_off(i, j, k)];
  }
  return c;
}
// occupied: known and L > l_occ
__device__ __forceinline__ bool octo_lo_occ(unsigned int c, int l_occ) { return lo_known(c) && lo_val(c) > l_occ; }
__device__ __forceinline__ unsigned int octo_lo_probe(const OcGrid& g, int s, float x, float y, float z, float vs) {
  return octo_lo_word(g, s, q_iround(x / vs), q_iround(y / vs), q_iround(z / vs));
}
// flags: bit0 occupied, bit1 unknown
__global__ void __launch_bounds__(256) k_octo_lo_query_points(OcGrid g, int s, long long n, const float* __restrict__ xyz, float vs, int l_occ,
                                                               uint8_t* flags) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const unsigned int c = octo_lo_probe(g, s, xyz[3 * q], xyz[3 * q + 1], xyz[3 * q + 2], vs);
    flags[q] = (uint8_t)((octo_lo_occ(c, l_occ) ? 1 : 0) | (lo_known(c) ? 0 : 2));
  }
}
// BaseMap.raycast on a log-odds map: stops at the first occupied sample (unknown space is not occupied)
__global__ void __launch_bounds__(256) k_octo_lo_raycast(OcGrid g, int s, long long n, const float* __restrict__ pos, const float* __restrict__ dir,
                                                          float max_dist, float vs, int l_occ, uint8_t* hit, float* xyz_out, float* len_out) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const float px = pos[3 * q], py = pos[3 * q + 1], pz = pos[3 * q + 2];
    const float dx = dir[3 * q], dy = dir[3 * q + 1], dz = dir[3 * q + 2];
    const int steps = (int)(max_dist / vs);
    float x = 0.f, y = 0.f, z = 0.f, len = 0.f;
    bool succ = false;
    for (int j = 0; j < steps; j++) {
      len = (float)j * vs;
      x = dx * len + px; y = dy * len + py; z = dz * len + pz;
      if (octo_lo_occ(octo_lo_probe(g, s, x, y, z, vs), l_occ)) { succ = true; break; }
    }
    hit[q] = succ ? 1 : 0;
    xyz_out[3 * q] = x; xyz_out[3 * q + 1] = y; xyz_out[3 * q + 2] = z;
    len_out[q] = len;
  }
}
// is_near_pos_occupy (mapping_common.py:193-204) on an Octomap: any occupied cell (i0 + a, j0 + b, k0 + c), a, b, c in
// [-voxel, voxel), around the point's cell.  LO: log-odds predicate with thres = l_occ; else count > min_occupy_thres.
template <bool LO>
__global__ void __launch_bounds__(256) k_octo_query_near(OcGrid g, int s, long long n, const float* __restrict__ xyz, float vs, int thres,
                                                          int voxel, uint8_t* out) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    const int i0 = q_iround(xyz[3 * q] / vs), j0 = q_iround(xyz[3 * q + 1] / vs), k0 = q_iround(xyz[3 * q + 2] / vs);
    bool any = false;
    for (int i = -voxel; i < voxel && !any; i++)
      for (int j = -voxel; j < voxel && !any; j++)
        for (int k = -voxel; k < voxel && !any; k++) {
          const unsigned int c = octo_lo_word(g, s, i0 + i, j0 + j, k0 + k);
          any = LO ? octo_lo_occ(c, thres) : (float)c > (float)thres;
        }
    out[q] = any ? 1 : 0;
  }
}

static int grid_for(long long n, int sm) {
  long long b = (n + 255) / 256;
  return (int)(b < (long long)sm * 16 ? (b > 0 ? b : 1) : (long long)sm * 16);
}

extern "C" int tslam_tsdf_query_points(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* xyz, uint8_t* flags, void* stream) {
  if (!m || n < 0 || (n && (!xyz || !flags))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  k_tsdf_query_points<<<grid_for(n, m->sm_count), 256, 0, st>>>(m->g, submap, n, xyz, m->in.vs, (float)(m->cfg.voxel_scale * 1.8), flags);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
extern "C" int tslam_tsdf_query_near_occupy(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* xyz, int32_t voxel, uint8_t* out, void* stream) {
  if (!m || n < 0 || voxel < 0 || (n && (!xyz || !out))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  k_tsdf_query_near<false><<<grid_for(n, m->sm_count), 256, 0, st>>>(m->g, submap, n, xyz, m->in.vs, (float)(m->cfg.voxel_scale * 1.8), voxel, out);
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
  k_tsdf_query_near<true><<<grid_for(n, m->sm_count), 256, 0, st>>>(m->g, submap, n, xyz, m->in.vs, (float)(m->cfg.voxel_scale * 1.8), voxel, out);
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
  k_tsdf_raycast<<<grid_for(n, m->sm_count), 256, 0, st>>>(m->g, submap, n, pos, dir, max_dist, m->in.vs, (float)(m->cfg.voxel_scale * 1.8), hit,
                                                         xyz_out, len_out);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
extern "C" int tslam_octo_query_points(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, uint8_t* flags, void* stream) {
  if (!m || n < 0 || (n && (!xyz || !flags))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  if (m->logodds)
    k_octo_lo_query_points<<<grid_for(n, m->sm_count), 256, 0, (cudaStream_t)stream>>>(m->g, submap, n, xyz, m->in.vs, m->lo.l_occ, flags);
  else
    k_octo_query_points<<<grid_for(n, m->sm_count), 256, 0, (cudaStream_t)stream>>>(m->g, submap, n, xyz, m->in.vs, (float)m->cfg.min_occupy_thres, flags);
  m->launches++;
  TS_CUDA(cudaGetLastError());
  return TSLAM_OK;
}
extern "C" int tslam_octo_raycast(tslam_octo_t* m, int32_t submap, int64_t n, const float* pos, const float* dir, float max_dist, uint8_t* hit,
                                  float* xyz_out, float* len_out, void* stream) {
  if (!m || n < 0 || (n && (!pos || !dir || !hit || !xyz_out || !len_out))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  if (m->logodds)
    k_octo_lo_raycast<<<grid_for(n, m->sm_count), 256, 0, (cudaStream_t)stream>>>(m->g, submap, n, pos, dir, max_dist, m->in.vs, m->lo.l_occ,
                                                                                hit, xyz_out, len_out);
  else
    k_octo_raycast<<<grid_for(n, m->sm_count), 256, 0, (cudaStream_t)stream>>>(m->g, submap, n, pos, dir, max_dist, m->in.vs,
                                                                             (float)m->cfg.min_occupy_thres, hit, xyz_out, len_out);
  m->launches++;
  TS_CUDA(cudaGetLastError());
  return TSLAM_OK;
}
extern "C" int tslam_octo_query_near_occupy(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, int32_t voxel, uint8_t* out, void* stream) {
  if (!m || n < 0 || voxel < 0 || (n && (!xyz || !out))) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  if (m->logodds)
    k_octo_query_near<true><<<grid_for(n, m->sm_count), 256, 0, (cudaStream_t)stream>>>(m->g, submap, n, xyz, m->in.vs, m->lo.l_occ, voxel, out);
  else
    k_octo_query_near<false><<<grid_for(n, m->sm_count), 256, 0, (cudaStream_t)stream>>>(m->g, submap, n, xyz, m->in.vs, m->cfg.min_occupy_thres,
                                                                                         voxel, out);
  m->launches++;
  TS_CUDA(cudaGetLastError());
  return TSLAM_OK;
}
