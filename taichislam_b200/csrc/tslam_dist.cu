// libtslam.so - multi-GPU support for a spatially TILED global TSDF map (SURVEY.md section 8e, BASELINE
// config 5).  One process per GPU; the global volume is cut into tx*ty*tz tiles of whole 16^3 blocks,
// tile t is owned by rank t.  The library only PACKS and UNPACKS voxel blocks; the exchange itself is a
// torch.distributed all_to_all over NCCL/NVLink done by the host layer (taichislam_b200/distributed.py):
//
//   fusion   every rank splats ITS submaps (k_fuse, sums left pending); blocks that fall into a foreign tile
//            are packed (key + pending-sum plane + observed/occupy planes), removed locally, sent to their
//            owner and added there (k_unpack_add); then every rank commits its own tile.
//   meshing  the one-block-thick boundary layer of every tile is copied to the (up to 26) neighbouring
//            tiles as GHOST blocks: marching cubes reads them for the +1 corner / +-1 normal stencil but
//            emits triangles only for owned blocks; the triangle soups are all-gathered by the host layer.
#include <cstring>
#include "tslam_internal.cuh"

// Tile boundaries (TsTiling, tile_owner: tslam_internal.cuh): the cuts set by tslam_tiling_set_cuts when they match
// `tiles3` (data-driven: the host layer puts them at the quantiles of the occupied blocks' marginal histograms, so a
// flat flight volume does not leave half the ranks empty), else equal slices of the volume.
int fill_tiling(tslam_tsdf* m, const int32_t* tiles3, int rank, int world, TsTiling* t) {
  if (!tiles3 || tiles3[0] < 1 || tiles3[1] < 1 || tiles3[2] < 1 || tiles3[0] * tiles3[1] * tiles3[2] != world || rank < 0 || rank >= world ||
      tiles3[0] > TS_MAX_TILES_AXIS || tiles3[1] > TS_MAX_TILES_AXIS || tiles3[2] > TS_MAX_TILES_AXIS) {
    ts_set_error("bad tiling: %d x %d x %d tiles for world size %d", tiles3 ? tiles3[0] : -1, tiles3 ? tiles3[1] : -1, tiles3 ? tiles3[2] : -1, world);
    return TSLAM_E_INVALID;
  }
  const int n[3] = {m->g.N, m->g.N, m->g.Nz}, h[3] = {m->g.hN, m->g.hN, m->g.hNz};
  const bool custom = m->tile_cuts_set && m->tile_cuts_tiles[0] == tiles3[0] && m->tile_cuts_tiles[1] == tiles3[1] && m->tile_cuts_tiles[2] == tiles3[2];
  for (int a = 0; a < 3; a++) {
    t->tiles[a] = tiles3[a];
    const int lo = (-h[a]) >> TS_BSHIFT, hi = (n[a] - h[a] - 1) >> TS_BSHIFT;  // block range of the volume
    const int ext = (hi - lo + 1 + tiles3[a] - 1) / tiles3[a];
    for (int k = 0; k <= tiles3[a]; k++) t->cuts[a][k] = custom ? m->tile_cuts[a][k] : lo + k * ext;
  }
  t->rank = rank;
  t->world = world;
  return TSLAM_OK;
}

// per-axis histograms of the block coordinates of the dirty blocks (coordinate + 512 in [0, 1024))
__global__ void __launch_bounds__(256) k_dirty_hist(TsGrid g, int* hist) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    if (!g.dirty_flag[b]) continue;
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    atomicAdd(&hist[(bx + 512) & 1023], 1);
    atomicAdd(&hist[1024 + ((by + 512) & 1023)], 1);
    atomicAdd(&hist[2048 + ((bz + 512) & 1023)], 1);
  }
}

// ---- fusion exchange -------------------------------------------------------------------------------------------
// pass 1: per destination rank, how many dirty blocks does it own?   pass 2: pack them, grouped by destination.
__global__ void __launch_bounds__(256) k_foreign_count(TsGrid g, TsTiling t, int* counts) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    if (!g.dirty_flag[b]) continue;
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    const int o = tile_owner(t, bx, by, bz);
    if (o != t.rank) atomicAdd(&counts[o], 1);
  }
}

// one CTA per block of the pool; foreign dirty blocks copy their planes into the slot group of their owner
__global__ void __launch_bounds__(256) k_foreign_pack(TsGrid g, TsTiling t, const int* offsets, int* cursor, long long cap,
                                                       long long* keys, float2* acc_out, uint8_t* obs_out, int8_t* occ_out, float4* col_out) {
  __shared__ long long s_slot;
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (!g.dirty_flag[b]) continue;  // uniform per CTA
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    const int o = tile_owner(t, bx, by, bz);
    if (o == t.rank) continue;
    __syncthreads();
    if (threadIdx.x == 0) {
      s_slot = (long long)offsets[o] + atomicAdd(&cursor[o], 1);
      if (s_slot < cap) keys[s_slot] = (long long)g.block_key[b];
      g.dirty_flag[b] = 0;  // not ours: never committed here
    }
    __syncthreads();
    const long long slot = s_slot;
    const size_t base = (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      if (slot < cap) {
        acc_out[slot * TS_B3 + v] = g.acc[base + v];
        obs_out[slot * TS_B3 + v] = g.obs[base + v];
        occ_out[slot * TS_B3 + v] = g.occ[base + v];
        if (col_out) col_out[slot * TS_B3 + v] = g.col[base + v];  // textured maps: pending sum of w * colour (dense_tsdf.py:277)
      }
      g.acc[base + v] = make_float2(0.f, 0.f);  // the block stays allocated but empty on this rank
      g.obs[base + v] = 0;
      g.occ[base + v] = 0;
      if (col_out) g.col[base + v] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

__global__ void __launch_bounds__(256) k_unpack_add(TsGrid g, long long n, const long long* keys, const float2* acc_in,
                                                     const uint8_t* obs_in, const int8_t* occ_in, const float4* col_in) {
  __shared__ int s_blk;
  for (long long q = blockIdx.x; q < n; q += gridDim.x) {
    __syncthreads();
    if (threadIdx.x == 0) {
      s_blk = ts_get_or_alloc(g, (unsigned long long)keys[q]);
      if (s_blk >= 0) ts_mark_dirty(g, s_blk);
    }
    __syncthreads();
    const int blk = s_blk;
    if (blk < 0) continue;
    const size_t base = (size_t)blk * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const float2 a = acc_in[q * TS_B3 + v];
      const uint8_t o = obs_in[q * TS_B3 + v];
      const int oc = occ_in[q * TS_B3 + v];
      if (a.x != 0.f || a.y != 0.f) atomicAdd(&g.acc[base + v], a);  // several ranks may send the same block
      if (col_in) {
        const float4 c = col_in[q * TS_B3 + v];
        if (c.x != 0.f || c.y != 0.f || c.z != 0.f) {
          float* cp = reinterpret_cast<float*>(&g.col[base + v]);
          atomicAdd(cp, c.x); atomicAdd(cp + 1, c.y); atomicAdd(cp + 2, c.z);
        }
      }
      if (o && g.obs[base + v] == 0) g.obs[base + v] = 2;            // observed, value pending (2 -> 1 at commit)
      if (oc) {
        // blocks with the same key (from different senders) are processed by different CTAs: go through a word CAS
        unsigned int* wp = (unsigned int*)((uintptr_t)&g.occ[base + v] & ~(uintptr_t)3);
        const int sh = (int)((uintptr_t)&g.occ[base + v] & 3) * 8;
        unsigned int old = *wp, assumed;
        do {
          assumed = old;
          int nv = (int)(int8_t)((assumed >> sh) & 0xFF) + oc;
          nv = nv > 127 ? 127 : (nv < -128 ? -128 : nv);
          old = atomicCAS(wp, assumed, (assumed & ~(0xFFu << sh)) | (((unsigned int)(nv & 0xFF)) << sh));
        } while (old != assumed);
      }
    }
  }
}

// ---- halo (ghost) exchange ---------------------------------------------------------------------------------------
// A block on the boundary layer of its tile goes to every neighbouring tile that touches it.  dests of a block =
// product over axes of {0} U {-1 if on the low face} U {+1 if on the high face}, minus the all-zero choice.
__device__ __forceinline__ int halo_dests(const TsTiling& t, int bx, int by, int bz, int* out /*<=26*/) {
  const int b[3] = {bx, by, bz};
  int tc[3], lo[3], hi[3];
  for (int a = 0; a < 3; a++) {
    tc[a] = tile_coord(t, a, b[a]);
    lo[a] = (b[a] == t.cuts[a][tc[a]]) && tc[a] > 0;
    hi[a] = (b[a] == t.cuts[a][tc[a] + 1] - 1) && tc[a] < t.tiles[a] - 1;
  }
  int n = 0;
  for (int dx = -1; dx <= 1; dx++)
    for (int dy = -1; dy <= 1; dy++)
      for (int dz = -1; dz <= 1; dz++) {
        if (!dx && !dy && !dz) continue;
        if ((dx == -1 && !lo[0]) || (dx == 1 && !hi[0]) || (dy == -1 && !lo[1]) || (dy == 1 && !hi[1]) || (dz == -1 && !lo[2]) ||
            (dz == 1 && !hi[2]))
          continue;
        out[n++] = ((tc[0] + dx) * t.tiles[1] + (tc[1] + dy)) * t.tiles[2] + (tc[2] + dz);
      }
  return n;
}

__global__ void __launch_bounds__(256) k_halo_count(TsGrid g, TsTiling t, int* counts) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    if (g.ghost[b]) continue;
    int s, bx, by, bz, d[26];
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (tile_owner(t, bx, by, bz) != t.rank) continue;
    const int n = halo_dests(t, bx, by, bz, d);
    for (int q = 0; q < n; q++) atomicAdd(&counts[d[q]], 1);
  }
}

__global__ void __launch_bounds__(256) k_halo_pack(TsGrid g, TsTiling t, const int* offsets, int* cursor, long long cap, long long* keys,
                                                    float2* tw_out, uint8_t* obs_out, float4* col_out) {
  __shared__ long long s_slot[26];
  __shared__ int s_n;
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (g.ghost[b]) continue;
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (tile_owner(t, bx, by, bz) != t.rank) continue;
    __syncthreads();
    if (threadIdx.x == 0) {
      int d[26];
      s_n = halo_dests(t, bx, by, bz, d);
      for (int q = 0; q < s_n; q++) {
        s_slot[q] = (long long)offsets[d[q]] + atomicAdd(&cursor[d[q]], 1);
        if (s_slot[q] < cap) keys[s_slot[q]] = (long long)g.block_key[b];
      }
    }
    __syncthreads();
    const int n = s_n;
    const size_t base = (size_t)b * TS_B3;
    for (int q = 0; q < n; q++) {
      const long long slot = s_slot[q];
      if (slot >= cap) continue;
      for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
        tw_out[slot * TS_B3 + v] = g.tw[base + v];
        obs_out[slot * TS_B3 + v] = g.obs[base + v];
        if (col_out) col_out[slot * TS_B3 + v] = g.col[base + v];
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_ghost_unpack(TsGrid g, long long n, const long long* keys, const float2* tw_in,
                                                       const uint8_t* obs_in, const float4* col_in, unsigned long long* stamp,
                                                       unsigned long long seq) {
  __shared__ int s_blk;
  for (long long q = blockIdx.x; q < n; q += gridDim.x) {
    __syncthreads();
    if (threadIdx.x == 0) {
      s_blk = ts_get_or_alloc(g, (unsigned long long)keys[q]);
      if (s_blk >= 0) { g.ghost[s_blk] = 1; stamp[s_blk] = seq; }
    }
    __syncthreads();
    const int blk = s_blk;
    if (blk < 0) continue;
    const size_t base = (size_t)blk * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      g.tw[base + v] = tw_in[q * TS_B3 + v];
      g.obs[base + v] = obs_in[q * TS_B3 + v];
      if (col_in) g.col[base + v] = col_in[q * TS_B3 + v];
    }
  }
}

// ---- ESDF halo (tiled ESDF, tslam_esdf.cu) ------------------------------------------------------------------------
// The same boundary blocks as the TSDF halo (halo_dests), those marked as changed since they were last packed.
__global__ void __launch_bounds__(256) k_esdf_halo_count(TsGrid g, TsTiling t, const int* xmark, int* counts) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    if (g.ghost[b] || !xmark[b]) continue;
    int s, bx, by, bz, d[26];
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (tile_owner(t, bx, by, bz) != t.rank) continue;
    const int n = halo_dests(t, bx, by, bz, d);
    for (int q = 0; q < n; q++) atomicAdd(&counts[d[q]], 1);
  }
}

struct EsHaloGroups { int off[24], cnt[24]; };  // slot group of every destination rank (from the caller's counts)

// One CTA per block.  A block whose every copy found a slot inside its group and below cap loses its mark; the others
// keep it (the host reports TSLAM_E_CAPACITY).
__global__ void __launch_bounds__(256) k_esdf_halo_pack(TsGrid g, TsTiling t, int* xmark, EsHaloGroups grp, int* cursor, long long cap,
                                                         long long* keys, float4* esdf_out) {
  __shared__ long long s_slot[26];
  __shared__ int s_n;
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    if (g.ghost[b] || !xmark[b]) continue;  // (uniform per CTA)
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (tile_owner(t, bx, by, bz) != t.rank) continue;
    __syncthreads();
    if (threadIdx.x == 0) {
      int d[26];
      bool all = true;
      s_n = halo_dests(t, bx, by, bz, d);
      for (int q = 0; q < s_n; q++) {
        const int k = atomicAdd(&cursor[d[q]], 1);
        long long slot = (long long)grp.off[d[q]] + k;
        if (k >= grp.cnt[d[q]] || slot >= cap) slot = -1;
        if (slot >= 0) keys[slot] = (long long)g.block_key[b];
        all &= slot >= 0;
        s_slot[q] = slot;
      }
      if (all) xmark[b] = 0;
    }
    __syncthreads();
    const int n = s_n;
    const float4* src = reinterpret_cast<const float4*>(g.esdf + (size_t)b * TS_B3);
    for (int q = 0; q < n; q++) {
      const long long slot = s_slot[q];
      if (slot < 0) continue;
      for (int v = threadIdx.x; v < TS_B3 / 4; v += blockDim.x) esdf_out[slot * (TS_B3 / 4) + v] = src[v];
    }
  }
}

// owner rank of the block holding each point's low interpolation corner (the corner k_esdf_query starts from), -1 for
// a point that is not finite or whose low corner lies outside the volume
__global__ void __launch_bounds__(256) k_owner_points(TsGrid g, TsTiling t, float vs, long long n, const float* __restrict__ xyz,
                                                       int* __restrict__ owner) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    float u[3];
    int c[3];
    owner[q] = esq_low_corner(g, vs, xyz + 3 * q, u, c) ? tile_owner(t, c[0] >> TS_BSHIFT, c[1] >> TS_BSHIFT, c[2] >> TS_BSHIFT) : -1;
  }
}

// ---- planner queries of a tiled map (tslam_query.cu) ---------------------------------------------------------------
// owner rank of the block holding each point's cell round(x / vs) - the cell TsdfProbe reads, by the same helper -
// or -1 for a cell outside the volume (it reads occupied and unobserved on any rank)
__global__ void __launch_bounds__(256) k_owner_cells(TsGrid g, TsTiling t, float vs, long long n, const float* __restrict__ xyz,
                                                      int* __restrict__ owner) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    int c[3];
    owner[q] = ts_query_cell(g, xyz[3 * q], xyz[3 * q + 1], xyz[3 * q + 2], vs, c) ? tile_owner(t, c[0] >> TS_BSHIFT, c[1] >> TS_BSHIFT, c[2] >> TS_BSHIFT)
                                                                                   : -1;
  }
}

// One round of BaseMap.raycast (mapping_common.py:165-178) on a tiled map, one lane per ray row f32[8] = pos, dir,
// max_dist, next sample j (int32 bits).  The samples and their count come from raycast_steps / raycast_sample, as in
// k_raycast, so a ray that stops at sample j here and continues at j on another rank visits the same cells with the
// same bits as one uninterrupted march.  The march runs while the sample's cell lies in a block this rank owns;
// ghosts are not read.  A sample in a foreign block hands the ray over: dest = its owner, j written back.  A hit, a
// sample outside the volume (occupied on any rank) or the last step ends the ray here: dest = -1 and the answer of
// the TSDF's k_raycast in row i of hit / xyz_out / len_out (for a miss: the last sample's position and length).
__global__ void __launch_bounds__(256) k_tsdf_raycast_tiled(TsGrid g, TsTiling t, int s, long long n, float* __restrict__ ray, float vs,
                                                             float thres, int* __restrict__ dest, uint8_t* hit, float* xyz_out, float* len_out) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
    float* r = ray + 8 * q;
    const float3 org = make_float3(r[0], r[1], r[2]), dr = make_float3(r[3], r[4], r[5]);
    const int steps = raycast_steps(r[6], vs);
    int j = __float_as_int(r[7]), to = -1;
    float x = 0.f, y = 0.f, z = 0.f, len = 0.f;
    bool succ = false;
    for (; j < steps; j++) {
      raycast_sample(org, dr, j, vs, x, y, z, len);
      int c[3];
      if (!ts_query_cell(g, x, y, z, vs, c)) { succ = true; break; }  // outside the volume: TSDF 0 on every rank
      const int o = tile_owner(t, c[0] >> TS_BSHIFT, c[1] >> TS_BSHIFT, c[2] >> TS_BSHIFT);
      if (o != t.rank) { to = o; break; }
      float tv = 0.0f;
      int ob = 0;
      ts_query_read<false>(g, s, c, tv, ob);
      if (tv < thres) { succ = true; break; }
    }
    dest[q] = to;
    if (to >= 0) {
      r[7] = __int_as_float(j);
      continue;
    }
    hit[q] = succ ? 1 : 0;
    xyz_out[3 * q] = x; xyz_out[3 * q + 1] = y; xyz_out[3 * q + 2] = z;
    len_out[q] = len;
  }
}

// ---- C ABI -------------------------------------------------------------------------------------------------------
// defined in tslam_tsdf.cu
extern "C" int tslam_tsdf_fuse_pending(tslam_tsdf_t* dst, tslam_tsdf_t* src, void* stream);

static int scan_counts(const int* h_counts, int world, int* h_offsets) {
  int tot = 0;
  for (int r = 0; r < world; r++) { h_offsets[r] = tot; tot += h_counts[r]; }
  return tot;
}

extern "C" int tslam_tiling_owner(tslam_tsdf_t* m, const int32_t* tiles3, int32_t world, int32_t bx, int32_t by, int32_t bz, int32_t* owner) {
  if (!m || !owner) return TSLAM_E_INVALID;
  TsTiling t;
  int rc = fill_tiling(m, tiles3, 0, world, &t);
  if (rc) return rc;
  *owner = tile_owner(t, bx, by, bz);
  return TSLAM_OK;
}

extern "C" int tslam_tiling_owner_points(tslam_tsdf_t* m, const int32_t* tiles3, int32_t world, int64_t n, const float* xyz, int32_t* owner,
                                         void* stream) {
  if (!m || n < 0 || (n && (!xyz || !owner))) return TSLAM_E_INVALID;
  TsTiling t;
  int rc = fill_tiling(m, tiles3, 0, world, &t);
  if (rc || n == 0) return rc;
  long long blocks = (n + 255) / 256;
  if (blocks > (long long)m->sm_count * 16) blocks = (long long)m->sm_count * 16;
  k_owner_points<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(m->g, t, m->in.vs, n, xyz, owner);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

static int lanes_grid(long long n, int sm) {
  const long long b = (n + 255) / 256;
  return (int)(b < (long long)sm * 16 ? b : (long long)sm * 16);
}

extern "C" int tslam_tiling_owner_cells(tslam_tsdf_t* m, const int32_t* tiles3, int32_t world, int64_t n, const float* xyz, int32_t* owner,
                                        void* stream) {
  if (!m || n < 0 || (n && (!xyz || !owner))) return TSLAM_E_INVALID;
  TsTiling t;
  int rc = fill_tiling(m, tiles3, 0, world, &t);
  if (rc || n == 0) return rc;
  k_owner_cells<<<lanes_grid(n, m->sm_count), 256, 0, (cudaStream_t)stream>>>(m->g, t, m->in.vs, n, xyz, owner);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_raycast_tiled(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, int32_t submap, int64_t n,
                                        float* ray, int32_t* dest, uint8_t* hit, float* xyz_out, float* len_out, void* stream) {
  if (!m || n < 0 || (n && (!ray || !dest || !hit || !xyz_out || !len_out))) return TSLAM_E_INVALID;
  TsTiling t;
  int rc = fill_tiling(m, tiles3, rank, world, &t);
  if (rc || n == 0) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = ts_flush_pending(m, st);
  if (rc) return rc;
  k_tsdf_raycast_tiled<<<lanes_grid(n, m->sm_count), 256, 0, st>>>(m->g, t, submap, n, ray, m->in.vs, (float)(m->cfg.voxel_scale * 1.8), dest,
                                                                   hit, xyz_out, len_out);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

extern "C" int tslam_tiling_set_cuts(tslam_tsdf_t* m, const int32_t* tiles3, const int32_t* cuts_x, const int32_t* cuts_y, const int32_t* cuts_z) {
  if (!m) return TSLAM_E_INVALID;
  if (!tiles3) { m->tile_cuts_set = 0; return TSLAM_OK; }  // back to equal slices of the volume
  const int32_t* cu[3] = {cuts_x, cuts_y, cuts_z};
  for (int a = 0; a < 3; a++) {
    if (tiles3[a] < 1 || tiles3[a] > TS_MAX_TILES_AXIS || !cu[a]) { ts_set_error("bad tile cuts"); return TSLAM_E_INVALID; }
    for (int k = 0; k < tiles3[a]; k++)
      if (cu[a][k] >= cu[a][k + 1]) { ts_set_error("tile cuts must increase strictly (axis %d)", a); return TSLAM_E_INVALID; }
  }
  for (int a = 0; a < 3; a++) {
    m->tile_cuts_tiles[a] = tiles3[a];
    for (int k = 0; k <= tiles3[a]; k++) m->tile_cuts[a][k] = cu[a][k];
  }
  m->tile_cuts_set = 1;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_dirty_hist(tslam_tsdf_t* m, int32_t* hist3x1024, void* stream) {
  if (!m || !hist3x1024) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  if (!m->tile_hist) TS_CUDA(cudaMalloc(&m->tile_hist, 3 * 1024 * sizeof(int)));
  TS_CUDA(cudaMemsetAsync(m->tile_hist, 0, 3 * 1024 * sizeof(int), st));
  k_dirty_hist<<<m->sm_count * 2, 256, 0, st>>>(m->g, m->tile_hist);
  TS_LAUNCH_CHECK(m);
  TS_CUDA(cudaMemcpyAsync(hist3x1024, m->tile_hist, 3 * 1024 * sizeof(int), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  return TSLAM_OK;
}

// counts_out[world] (host): blocks this rank must send to every other rank.  Synchronises.
extern "C" int tslam_tsdf_foreign_count(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, int32_t* counts_out,
                                        void* stream) {
  if (!m || !counts_out || world > 64) return TSLAM_E_INVALID;
  TsTiling t;
  int rc = fill_tiling(m, tiles3, rank, world, &t);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int* d = m->scratch_i + 16;  // [16..48): per-rank counters (world <= 32 here)
  if (world > 24) { ts_set_error("world size %d > 24 not supported by the scratch counters", world); return TSLAM_E_INVALID; }
  TS_CUDA(cudaMemsetAsync(d, 0, 48 * sizeof(int), st));
  k_foreign_count<<<m->sm_count * 2, 256, 0, st>>>(m->g, t, d);
  TS_LAUNCH_CHECK(m);
  TS_CUDA(cudaMemcpyAsync(counts_out, d, world * sizeof(int), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  return TSLAM_OK;
}

// Pack the foreign dirty blocks grouped by destination (counts from tslam_tsdf_foreign_count), clear them locally.
// keys int64[cap], acc f32[cap,4096,2], obs u8[cap,4096], occ i8[cap,4096] (DEVICE).
extern "C" int tslam_tsdf_foreign_pack(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts,
                                       int64_t cap, int64_t* keys, float* acc, uint8_t* obs, int8_t* occ, void* stream) {
  return tslam_tsdf_foreign_pack2(m, tiles3, rank, world, counts, cap, keys, acc, obs, occ, nullptr, stream);
}
extern "C" int tslam_tsdf_foreign_pack2(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts,
                                        int64_t cap, int64_t* keys, float* acc, uint8_t* obs, int8_t* occ, float* col, void* stream) {
  if (!m || !counts || world > 24) return TSLAM_E_INVALID;
  if (col && !m->g.col) { ts_set_error("colour plane requested from an untextured map"); return TSLAM_E_INVALID; }
  if (!col && m->g.col) { ts_set_error("textured map: the colour plane must travel with the blocks (pass col)"); return TSLAM_E_INVALID; }
  TsTiling t;
  int rc = fill_tiling(m, tiles3, rank, world, &t);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int h_off[24];
  scan_counts(counts, world, h_off);
  int* d_off = m->scratch_i + 16;
  int* d_cur = m->scratch_i + 40;
  TS_CUDA(cudaMemcpyAsync(d_off, h_off, world * sizeof(int), cudaMemcpyHostToDevice, st));
  TS_CUDA(cudaMemsetAsync(d_cur, 0, 24 * sizeof(int), st));
  m->mesh_epoch++;  // the packed blocks' obs / col planes are cleared without a stamp
  fz_written(m->ver, -1);
  k_foreign_pack<<<m->sm_count * 4, 256, 0, st>>>(m->g, t, d_off, d_cur, cap, (long long*)keys, (float2*)acc, obs, occ, (float4*)col);
  TS_LAUNCH_CHECK(m);
  TS_CUDA(cudaStreamSynchronize(st));  // h_off is on the stack
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_unpack_add(tslam_tsdf_t* m, int64_t n, const int64_t* keys, const float* acc, const uint8_t* obs,
                                     const int8_t* occ, void* stream) {
  return tslam_tsdf_unpack_add2(m, n, keys, acc, obs, occ, nullptr, stream);
}
extern "C" int tslam_tsdf_unpack_add2(tslam_tsdf_t* m, int64_t n, const int64_t* keys, const float* acc, const uint8_t* obs,
                                      const int8_t* occ, const float* col, void* stream) {
  if (!m || n < 0) return TSLAM_E_INVALID;
  if (col && !m->g.col) { ts_set_error("colour plane given to an untextured map"); return TSLAM_E_INVALID; }
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  m->mesh_epoch++;  // obs / col change before the fused commit stamps the blocks
  fz_written(m->ver, -1);
  k_unpack_add<<<(int)(n < m->sm_count * 4 ? n : m->sm_count * 4), 256, 0, st>>>(m->g, n, (const long long*)keys, (const float2*)acc, obs, occ, (const float4*)col);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_halo_count(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, int32_t* counts_out,
                                     void* stream) {
  if (!m || !counts_out || world > 24) return TSLAM_E_INVALID;
  TsTiling t;
  int rc = fill_tiling(m, tiles3, rank, world, &t);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = ts_flush_pending(m, st);
  if (rc) return rc;
  int* d = m->scratch_i + 16;
  TS_CUDA(cudaMemsetAsync(d, 0, 48 * sizeof(int), st));
  k_halo_count<<<m->sm_count * 2, 256, 0, st>>>(m->g, t, d);
  TS_LAUNCH_CHECK(m);
  TS_CUDA(cudaMemcpyAsync(counts_out, d, world * sizeof(int), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_halo_pack(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts,
                                    int64_t cap, int64_t* keys, float* tw, uint8_t* obs, void* stream) {
  return tslam_tsdf_halo_pack2(m, tiles3, rank, world, counts, cap, keys, tw, obs, nullptr, stream);
}
extern "C" int tslam_tsdf_halo_pack2(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts,
                                     int64_t cap, int64_t* keys, float* tw, uint8_t* obs, float* col, void* stream) {
  if (!m || !counts || world > 24) return TSLAM_E_INVALID;
  if (col && !m->g.col) { ts_set_error("colour plane requested from an untextured map"); return TSLAM_E_INVALID; }
  TsTiling t;
  int rc = fill_tiling(m, tiles3, rank, world, &t);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int h_off[24];
  scan_counts(counts, world, h_off);
  int* d_off = m->scratch_i + 16;
  int* d_cur = m->scratch_i + 40;
  TS_CUDA(cudaMemcpyAsync(d_off, h_off, world * sizeof(int), cudaMemcpyHostToDevice, st));
  TS_CUDA(cudaMemsetAsync(d_cur, 0, 24 * sizeof(int), st));
  k_halo_pack<<<m->sm_count * 4, 256, 0, st>>>(m->g, t, d_off, d_cur, cap, (long long*)keys, (float2*)tw, obs, (float4*)col);
  TS_LAUNCH_CHECK(m);
  TS_CUDA(cudaStreamSynchronize(st));
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_ghost_unpack(tslam_tsdf_t* m, int64_t n, const int64_t* keys, const float* tw, const uint8_t* obs, void* stream) {
  return tslam_tsdf_ghost_unpack2(m, n, keys, tw, obs, nullptr, stream);
}
extern "C" int tslam_tsdf_ghost_unpack2(tslam_tsdf_t* m, int64_t n, const int64_t* keys, const float* tw, const uint8_t* obs, const float* col,
                                        void* stream) {
  if (!m || n < 0) return TSLAM_E_INVALID;
  if (col && !m->g.col) { ts_set_error("colour plane given to an untextured map"); return TSLAM_E_INVALID; }
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  fz_written(m->ver, -1);
  m->ghost_gen++;
  m->esdf_full_needed = 1;
  const unsigned long long seq = ++m->commit_seq;  // the imported ghosts are stamped like committed blocks (incremental mesh)
  k_ghost_unpack<<<(int)(n < m->sm_count * 4 ? n : m->sm_count * 4), 256, 0, st>>>(m->g, n, (const long long*)keys, (const float2*)tw, obs, (const float4*)col,
                                                                                  m->blk_stamp, seq);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

// ---- ESDF halo of a tiled ESDF (tslam_esdf_tiled_begin .. _end) ----------------------------------------------------
static int esdf_halo_open(tslam_tsdf* m, const char* what) {
  if (!ts_esdf_xmark(m) || m->esdf_tiled != 1 || m->esdf_full_needed) {
    ts_set_error("%s: no tiled ESDF is in progress (tslam_esdf_tiled_begin, then no reset, load, fusion or ghost import)", what);
    return TSLAM_E_INVALID;
  }
  return TSLAM_OK;
}

extern "C" int tslam_esdf_halo_count(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, int32_t* counts_out, void* stream) {
  if (!m || !counts_out || world > 24) return TSLAM_E_INVALID;
  TsTiling t;
  int rc = fill_tiling(m, tiles3, rank, world, &t);
  if (rc) return rc;
  rc = esdf_halo_open(m, "tslam_esdf_halo_count");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  int* d = m->scratch_i + 16;
  TS_CUDA(cudaMemsetAsync(d, 0, 48 * sizeof(int), st));
  k_esdf_halo_count<<<m->sm_count * 2, 256, 0, st>>>(m->g, t, ts_esdf_xmark(m), d);
  TS_LAUNCH_CHECK(m);
  TS_CUDA(cudaMemcpyAsync(counts_out, d, world * sizeof(int), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  return TSLAM_OK;
}

extern "C" int tslam_esdf_halo_pack(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts, int64_t cap,
                                    int64_t* keys, float* esdf, void* stream) {
  if (!m || !counts || world > 24 || cap < 0 || (cap && (!keys || !esdf))) return TSLAM_E_INVALID;
  TsTiling t;
  int rc = fill_tiling(m, tiles3, rank, world, &t);
  if (rc) return rc;
  rc = esdf_halo_open(m, "tslam_esdf_halo_pack");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  EsHaloGroups grp;
  const int tot = scan_counts(counts, world, grp.off);
  for (int r = 0; r < world; r++) grp.cnt[r] = counts[r] < 0 ? 0 : counts[r];
  int* d_cur = m->scratch_i + 40;
  TS_CUDA(cudaMemsetAsync(d_cur, 0, 24 * sizeof(int), st));
  k_esdf_halo_pack<<<m->sm_count * 4, 256, 0, st>>>(m->g, t, ts_esdf_xmark(m), grp, d_cur, cap, (long long*)keys, (float4*)esdf);
  TS_LAUNCH_CHECK(m);
  int h_cur[24];
  TS_CUDA(cudaMemcpyAsync(h_cur, d_cur, world * sizeof(int), cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  bool over = tot > cap;
  for (int r = 0; r < world; r++) over |= h_cur[r] > grp.cnt[r];
  if (over) {
    ts_set_error("esdf halo pack: capacity (buffers saturated; the blocks that did not fit stay marked)");
    return TSLAM_E_CAPACITY;
  }
  return TSLAM_OK;
}
