// libtslam.so - marching cubes over the TSDF hash grid.  Two passes
// (count -> exclusive scan over blocks -> emit) instead of the reference's single
// pass with one global atomic per triangle (marching_cube_mesher.py:114).
// One CTA per 16^3 block; the block plus its halo (-1 .. +17 per axis: +1 for the
// cube corners, and +-1 around round(vertex) for the central-difference normals,
// :84-93) is staged in shared memory once, so every TSDF value is read from HBM
// once per pass instead of 8 + 18 times through a tree walk.
#include <cstring>
#include "tslam_internal.cuh"
#include "../../include/tslam_mc_cases.h"

#define MC_T 19                 // tile edge: block 16 + halo (1 below, 2 above)
#define MC_T3 (MC_T * MC_T * MC_T)
#define MC_EPS 1e-6f            // marching_cube_mesher.py:6

__constant__ unsigned long long c_mc_cases[256];   // packed tri table (marching_cube_mesher.py:244-499)
__constant__ unsigned short c_mc_edges[256];        // derived edge masks (:225-241)
__constant__ unsigned char c_mc_ntri[256];

static const unsigned long long h_mc_cases[256] = TSLAM_MC_CASE_WORDS;
static bool g_tables_uploaded = false;

static int mc_upload_tables() {
  if (g_tables_uploaded) return TSLAM_OK;
  unsigned short edges[256];
  unsigned char ntri[256];
  for (int c = 0; c < 256; c++) {
    unsigned m = 0, n = 0;
    for (int q = 0; q < 16; q++) {
      unsigned e = (unsigned)((h_mc_cases[c] >> (4 * q)) & 0xF);
      if (e != 0xF) { m |= 1u << e; n++; }
    }
    edges[c] = (unsigned short)m;
    ntri[c] = (unsigned char)(n / 3);
  }
  TS_CUDA(cudaMemcpyToSymbol(c_mc_cases, h_mc_cases, sizeof(h_mc_cases)));
  TS_CUDA(cudaMemcpyToSymbol(c_mc_edges, edges, sizeof(edges)));
  TS_CUDA(cudaMemcpyToSymbol(c_mc_ntri, ntri, sizeof(ntri)));
  g_tables_uploaded = true;
  return TSLAM_OK;
}

// corner offsets V0..V7 (marching_cube_mesher.py:196-206) packed x|y<<1|z<<2 per corner
__device__ __forceinline__ void mc_corner(int c, int& dx, int& dy, int& dz) {
  // V0 000, V1 100, V2 110, V3 010, V4 001, V5 101, V6 111, V7 011
  const unsigned X = 0x66u, Y = 0xCCu, Z = 0xF0u;  // bit c of X/Y/Z = dx/dy/dz of corner c
  dx = (X >> c) & 1; dy = (Y >> c) & 1; dz = (Z >> c) & 1;
}
// edge endpoints (:208-221): E0 01, E1 12, E2 23, E3 30, E4 45, E5 56, E6 67, E7 74, E8 04, E9 15, E10 26, E11 37
__device__ __forceinline__ void mc_edge_ends(int e, int& a, int& b) {
  const unsigned long long A = 0x321076543210ull, B = 0x765447650321ull;  // nibble e = endpoint
  a = (int)((A >> (4 * e)) & 0xF);
  b = (int)((B >> (4 * e)) & 0xF);
}

struct McTile {
  float t[MC_T3];
  unsigned char o[MC_T3];
  int nbr[27];
};

__device__ __forceinline__ int mc_tidx(int lx, int ly, int lz) {  // local coords in [-1, 17]
  return ((lx + 1) * MC_T + (ly + 1)) * MC_T + (lz + 1);
}

// stage block b (+halo) of the TSDF / observed planes into shared memory.
// Reads of inactive cells return 0 (pointer-SNode semantics).
__device__ void mc_stage(const TsGrid& g, McTile& tile, int s, int bx, int by, int bz) {
  if (threadIdx.x < 27) {
    const int dx = threadIdx.x / 9 - 1, dy = (threadIdx.x / 3) % 3 - 1, dz = threadIdx.x % 3 - 1;
    tile.nbr[threadIdx.x] = ts_find(g, ts_pack_key(s, bx + dx, by + dy, bz + dz));
  }
  __syncthreads();
  for (int c = threadIdx.x; c < MC_T3; c += blockDim.x) {
    const int lz = c % MC_T - 1, ly = (c / MC_T) % MC_T - 1, lx = c / (MC_T * MC_T) - 1;
    const int nx = (lx + 16) >> 4, ny = (ly + 16) >> 4, nz = (lz + 16) >> 4;  // 0,1,2 -> -1,0,+1 block
    const int nb = tile.nbr[(nx * 3 + ny) * 3 + nz];
    float tv = 0.0f;
    unsigned char ov = 0;
    if (nb >= 0) {
      const size_t off = (size_t)nb * TS_B3 + ((((lx & 15) << 4) | (ly & 15)) << 4 | (lz & 15));
      tv = g.tw[off].x;
      ov = g.obs[off];
    }
    tile.t[c] = tv;
    tile.o[c] = ov;
  }
  __syncthreads();
}

// cube index of the cell at local (lx,ly,lz), or -1 when the cell is skipped
// (marching_cube_mesher.py:184 filter, :133-144 corners).
__device__ __forceinline__ int mc_cube_index(const McTile& tile, int lx, int ly, int lz, float thres, float* val) {
  const int c0 = mc_tidx(lx, ly, lz);
  if (!(tile.o[c0] > 0 && tile.t[c0] < thres)) return -1;  // :184
  bool any_unobs = false;
  int cube = 0;
#pragma unroll
  for (int c = 0; c < 8; c++) {
    int dx, dy, dz;
    mc_corner(c, dx, dy, dz);
    const int ci = mc_tidx(lx + dx, ly + dy, lz + dz);
    const float v = tile.t[ci];
    val[c] = v;
    if (tile.o[ci] == 0) any_unobs = true;  // :137-138
    if (v < 0.0f) cube |= 1 << c;           // :143-144
  }
  return any_unobs ? -1 : cube;
}

// Whether block b holds an observed voxel with TSDF < 0 (NaN and -0 are not < 0, as in mc_cube_index): a cell can only
// emit a triangle when one of its corners is such a voxel.  Read straight from the planes; CTA-uniform result.
__device__ __forceinline__ bool mc_block_neg(const TsGrid& g, int b) {
  const size_t base = (size_t)b * TS_B3;
  int neg = 0;
  for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) neg |= (g.obs[base + v] != 0 && g.tw[base + v].x < 0.0f);
  return __syncthreads_or(neg) != 0;
}

// pass 1: triangles per block.  List = false: every block of the pool (tslam_mc_generate2).  List = true: the blocks
// list[0 .. *n_list) (the incremental mesh), which also stores mc_block_neg of each listed block in neg[].
template <bool List>
__global__ void __launch_bounds__(256) k_mc_count(TsGrid g, float thres, unsigned int* blk_tris, const int* list, const int* n_list,
                                                   uint8_t* neg) {
  __shared__ McTile tile;
  __shared__ unsigned int warp_sum[8];
  const int nb = List ? *n_list : min(*g.n_blocks, g.max_blocks);
  for (int q = blockIdx.x; q < nb; q += gridDim.x) {
    const int b = List ? list[q] : q;
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (g.ghost[b]) {  // halo copy: its cells belong to the owning rank
      if (List) {      // (its voxels are corners of the owned cells next to it)
        const bool ng = mc_block_neg(g, b);
        if (threadIdx.x == 0) neg[b] = ng;
      }
      if (threadIdx.x == 0) blk_tris[b] = 0;
      continue;
    }
    __syncthreads();
    mc_stage(g, tile, s, bx, by, bz);
    unsigned int n = 0;
    int ng = 0;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      float val[8];
      const int cube = mc_cube_index(tile, v >> 8, (v >> 4) & 15, v & 15, thres, val);
      if (cube >= 0) n += c_mc_ntri[cube];
      if (List) {
        const int c = mc_tidx(v >> 8, (v >> 4) & 15, v & 15);
        ng |= (tile.o[c] != 0 && tile.t[c] < 0.0f);
      }
    }
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = n;
    if (List) ng = __syncthreads_or(ng);
    else __syncthreads();
    if (threadIdx.x == 0) {
      unsigned int t = 0;
      for (int w = 0; w < 8; w++) t += warp_sum[w];
      blk_tris[b] = t;
      if (List) neg[b] = ng != 0;
    }
  }
}

// exclusive scan of per-block triangle counts (single CTA, nb <= 2^24)
__global__ void __launch_bounds__(1024) k_mc_scan(const int* n_blocks_p, int max_blocks, const unsigned int* blk_tris,
                                                   unsigned long long* blk_off, unsigned long long* total) {
  __shared__ unsigned long long wsum[32];
  __shared__ unsigned long long carry;
  const int nb = min(*n_blocks_p, max_blocks);
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += 1024) {
    const int i = base + threadIdx.x;
    unsigned long long v = (i < nb) ? blk_tris[i] : 0ull;
    unsigned long long x = v;
    for (int o = 1; o < 32; o <<= 1) {
      unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
      if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      unsigned long long w = wsum[threadIdx.x];
      unsigned long long ws = w;
      for (int o = 1; o < 32; o <<= 1) {
        unsigned long long y = __shfl_up_sync(0xffffffffu, ws, o);
        if (threadIdx.x >= o) ws += y;
      }
      wsum[threadIdx.x] = ws - w;  // exclusive warp offsets
    }
    __syncthreads();
    const unsigned long long excl = carry + wsum[threadIdx.x >> 5] + (x - v);
    if (i < nb) blk_off[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}

// vertexInterp_color (marching_cube_mesher.py:62-82) for the vertex on edge e of the cell at (i,j,k).  Reference
// quirks kept: mu stays 0 in the two snap branches (:66-71), and the "colour is zero" tests look at channel 0 only.
__device__ __forceinline__ float4 mc_read_col(const TsGrid& g, int s, int i, int j, int k) {
  const int blk = ts_find(g, ts_pack_key(s, i >> TS_BSHIFT, j >> TS_BSHIFT, k >> TS_BSHIFT));
  if (blk < 0 || !g.col) return make_float4(0.f, 0.f, 0.f, 0.f);
  return g.col[(size_t)blk * TS_B3 + ts_voxel_off(i, j, k)];
}
__device__ __forceinline__ void mc_vertex_color(const TsGrid& g, int s, int i, int j, int k, int step, int e, const float* val, float* out) {
  int a, bb, ax, ay, az, cx, cy, cz;
  mc_edge_ends(e, a, bb);
  mc_corner(a, ax, ay, az);
  mc_corner(bb, cx, cy, cz);
  const float v1 = val[a], v2 = val[bb];
  float mu = 0.0f;
  if (!(fabsf(0.0f - v1) < MC_EPS) && !(fabsf(0.0f - v2) < MC_EPS)) mu = (0.0f - v1) / (v2 - v1);
  const float4 c1 = mc_read_col(g, s, i + ax * step, j + ay * step, k + az * step);
  const float4 c2 = mc_read_col(g, s, i + cx * step, j + cy * step, k + cz * step);
  if (c1.x == 0.0f) { out[0] = c2.x; out[1] = c2.y; out[2] = c2.z; }
  else if (!(c2.x == 0.0f)) {
    out[0] = c1.x + mu * (c2.x - c1.x); out[1] = c1.y + mu * (c2.y - c1.y); out[2] = c1.z + mu * (c2.z - c1.z);
  } else { out[0] = c1.x; out[1] = c1.y; out[2] = c1.z; }
}

// pass 2: emit.  vertexInterp (:44-60), add_triangle (:95-102), generate_normal (:84-93).
// Per block: (1) every thread classifies its 16 voxels slab by slab, a CTA-wide exclusive scan of the triangle counts
// gives every cell its deterministic output slot (voxel order), cells with triangles go into a shared-memory list;
// (2) the list is worked off one thread per VERTEX (cell x triangle x corner): one edge interpolation, one normal,
// coalescing-friendly stores.  (The first version let the thread that owned a surface cell interpolate all 12 edges
// into a local array and write up to 15 vertices itself: a few per cent of the lanes did all the work, several
// times the count pass's time on the bench map.)
#define MC_LIST 1024
__device__ __forceinline__ void mc_emit_list(const TsGrid& g, const McTile& tile, int s, int bx, int by, int bz, float vs, unsigned long long boff,
                                             long long cap_tri, const unsigned int* cell_vc, const unsigned int* cell_off, int ncell,
                                             float* verts, float* normals, float* colors) {
  for (int idx = threadIdx.x; idx < ncell * 15; idx += blockDim.x) {
    const int c = idx / 15, r = idx - c * 15, t = r / 3, q = r - t * 3;
    const unsigned int vc = cell_vc[c];
    const int cube = (int)(vc & 255u), v = (int)(vc >> 8);
    if (t >= (int)c_mc_ntri[cube]) continue;
    const long long tri = (long long)(boff + cell_off[c] + (unsigned)t);
    if (tri >= cap_tri) continue;  // saturate (the reference writes out of bounds, :175-177)
    const int lx = v >> 8, ly = (v >> 4) & 15, lz = v & 15;
    const int i = bx * TS_B + lx, j = by * TS_B + ly, k = bz * TS_B + lz;
    const int e = (int)((c_mc_cases[cube] >> (4 * (3 * t + q))) & 0xF);  // :173-174, :110-125
    int a, bb, ax, ay, az, cx, cy, cz;
    mc_edge_ends(e, a, bb);
    mc_corner(a, ax, ay, az);
    mc_corner(bb, cx, cy, cz);
    const float p1x = (float)(i + ax), p1y = (float)(j + ay), p1z = (float)(k + az);
    const float p2x = (float)(i + cx), p2y = (float)(j + cy), p2z = (float)(k + cz);
    const float v1 = tile.t[mc_tidx(lx + ax, ly + ay, lz + az)], v2 = tile.t[mc_tidx(lx + cx, ly + cy, lz + cz)];
    float px, py, pz;
    if (fabsf(0.0f - v1) < MC_EPS) { px = p1x; py = p1y; pz = p1z; }        // :49-50
    else if (fabsf(0.0f - v2) < MC_EPS) { px = p2x; py = p2y; pz = p2z; }   // :51-54
    else {
      const float mu = (0.0f - v1) / (v2 - v1);                             // :56
      px = p1x + mu * (p2x - p1x);
      py = p1y + mu * (p2y - p1y);
      pz = p1z + mu * (p2z - p1z);
    }
    float* vo = verts + ((size_t)tri * 3 + q) * 3;
    vo[0] = px * vs; vo[1] = py * vs; vo[2] = pz * vs;  // ijk_to_xyz :40-42 (map-local metres)
    if (colors) {  // :104-108
      float val[8];
#pragma unroll
      for (int cc = 0; cc < 8; cc++) {
        int dx, dy, dz;
        mc_corner(cc, dx, dy, dz);
        val[cc] = tile.t[mc_tidx(lx + dx, ly + dy, lz + dz)];
      }
      mc_vertex_color(g, s, i, j, k, 1, e, val, colors + ((size_t)tri * 3 + q) * 3);
    }
    // generate_normal :84-93 - central differences at round(vertex), from the staged tile
    float* no = normals + ((size_t)tri * 3 + q) * 3;
    if (!(isfinite(px) && isfinite(py) && isfinite(pz))) {  // NaN TSDF corner: round(NaN) is undefined (:86)
      no[0] = no[1] = no[2] = __int_as_float(0x7fc00000);
      continue;
    }
    const int qx = (int)roundf(px) - bx * TS_B, qy = (int)roundf(py) - by * TS_B, qz = (int)roundf(pz) - bz * TS_B;
    const float nx = tile.t[mc_tidx(qx + 1, qy, qz)] - tile.t[mc_tidx(qx - 1, qy, qz)];
    const float ny = tile.t[mc_tidx(qx, qy + 1, qz)] - tile.t[mc_tidx(qx, qy - 1, qz)];
    const float nz = tile.t[mc_tidx(qx, qy, qz + 1)] - tile.t[mc_tidx(qx, qy, qz - 1)];
    const float nn = sqrtf((nx * nx + ny * ny) + nz * nz);
    no[0] = nx / nn; no[1] = ny / nn; no[2] = nz / nn;  // normalized(): NaN when the gradient vanishes
  }
}

// List as k_mc_count: every block of the pool, or the blocks list[0 .. *n_list).
template <bool List>
__global__ void __launch_bounds__(256) k_mc_emit(TsGrid g, float thres, float vs, const unsigned int* blk_tris,
                                                  const unsigned long long* blk_off, long long cap_tri, float* verts, float* normals,
                                                  float* colors, const int* list, const int* n_list) {
  __shared__ McTile tile;
  __shared__ unsigned int warp_sum[8];
  __shared__ unsigned int run_base;
  __shared__ unsigned int cell_vc[MC_LIST], cell_off[MC_LIST];  // voxel << 8 | cube index; first output triangle (relative to the block's)
  __shared__ int n_cell;
  const int nb = List ? *n_list : min(*g.n_blocks, g.max_blocks);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int q = blockIdx.x; q < nb; q += gridDim.x) {
    const int b = List ? list[q] : q;
    if (blk_tris[b] == 0) continue;
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    __syncthreads();
    mc_stage(g, tile, s, bx, by, bz);
    if (threadIdx.x == 0) { run_base = 0; n_cell = 0; }
    __syncthreads();
    const unsigned long long boff = blk_off[b];
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {  // uniform trip count (16)
      const int lx = v >> 8, ly = (v >> 4) & 15, lz = v & 15;
      float val[8];
      const int cube = mc_cube_index(tile, lx, ly, lz, thres, val);
      const unsigned int nt = cube >= 0 ? c_mc_ntri[cube] : 0u;
      // CTA-wide exclusive scan of nt (voxel order within this slab of 256 voxels)
      unsigned int x = nt;
      for (int o = 1; o < 32; o <<= 1) {
        unsigned int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
      }
      if (lane == 31) warp_sum[wid] = x;
      __syncthreads();
      unsigned int woff = 0, slab_total = 0;
#pragma unroll
      for (int w = 0; w < 8; w++) {
        const unsigned int ws = warp_sum[w];
        if (w < wid) woff += ws;
        slab_total += ws;
      }
      const unsigned int my_off = run_base + woff + (x - nt);
      if (nt) {
        const int p = atomicAdd(&n_cell, 1);  // (list order is irrelevant: the output slot rides along)
        cell_vc[p] = ((unsigned)v << 8) | (unsigned)cube;
        cell_off[p] = my_off;
      }
      __syncthreads();
      if (threadIdx.x == 0) run_base += slab_total;
      if (n_cell + 256 > MC_LIST) {  // the next slab might not fit: work the list off now (uniform: n_cell is shared)
        mc_emit_list(g, tile, s, bx, by, bz, vs, boff, cap_tri, cell_vc, cell_off, n_cell, verts, normals, colors);
        __syncthreads();
        if (threadIdx.x == 0) n_cell = 0;
        __syncthreads();
      }
    }
    __syncthreads();
    mc_emit_list(g, tile, s, bx, by, bz, vs, boff, cap_tri, cell_vc, cell_off, n_cell, verts, normals, colors);
  }
}

// generic (step != 1) path: corners and normals read through the hash grid.
__device__ __forceinline__ void mc_read(const TsGrid& g, int s, int i, int j, int k, float& t, int& o) {
  const int blk = ts_find(g, ts_pack_key(s, i >> TS_BSHIFT, j >> TS_BSHIFT, k >> TS_BSHIFT));
  if (blk < 0) { t = 0.0f; o = 0; return; }
  const size_t off = (size_t)blk * TS_B3 + ts_voxel_off(i, j, k);
  t = g.tw[off].x;
  o = g.obs[off];
}

__global__ void __launch_bounds__(256) k_mc_generic(TsGrid g, int step, float thres, float vs, long long cap_tri, float* verts,
                                                     float* normals, float* colors, unsigned long long* counter) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (g.ghost[b]) continue;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const int i = bx * TS_B + (v >> 8), j = by * TS_B + ((v >> 4) & 15), k = bz * TS_B + (v & 15);
      const size_t off = (size_t)b * TS_B3 + v;
      if (!(g.obs[off] > 0 && g.tw[off].x < thres)) continue;
      float val[8];
      bool bad = false;
      int cube = 0;
      for (int c = 0; c < 8; c++) {
        int dx, dy, dz, o;
        mc_corner(c, dx, dy, dz);
        mc_read(g, s, i + dx * step, j + dy * step, k + dz * step, val[c], o);
        if (o == 0) bad = true;
        if (val[c] < 0.0f) cube |= 1 << c;
      }
      if (bad) continue;
      const unsigned nt = c_mc_ntri[cube];
      if (!nt) continue;
      const unsigned mask = c_mc_edges[cube];
      float vl[12][3];
      for (int e = 0; e < 12; e++) {
        if (!(mask & (1u << e))) continue;
        int a, bb, ax, ay, az, cx, cy, cz;
        mc_edge_ends(e, a, bb);
        mc_corner(a, ax, ay, az);
        mc_corner(bb, cx, cy, cz);
        const float p1x = (float)(i + ax * step), p1y = (float)(j + ay * step), p1z = (float)(k + az * step);
        const float p2x = (float)(i + cx * step), p2y = (float)(j + cy * step), p2z = (float)(k + cz * step);
        const float v1 = val[a], v2 = val[bb];
        if (fabsf(0.0f - v1) < MC_EPS) { vl[e][0] = p1x; vl[e][1] = p1y; vl[e][2] = p1z; }
        else if (fabsf(0.0f - v2) < MC_EPS) { vl[e][0] = p2x; vl[e][1] = p2y; vl[e][2] = p2z; }
        else {
          const float mu = (0.0f - v1) / (v2 - v1);
          vl[e][0] = p1x + mu * (p2x - p1x);
          vl[e][1] = p1y + mu * (p2y - p1y);
          vl[e][2] = p1z + mu * (p2z - p1z);
        }
      }
      const unsigned long long base = atomicAdd(counter, (unsigned long long)nt);
      const unsigned long long cw = c_mc_cases[cube];
      for (unsigned t = 0; t < nt; t++) {
        const long long tri = (long long)(base + t);
        if (tri >= cap_tri) break;
        for (int q = 0; q < 3; q++) {
          const int e = (int)((cw >> (4 * (3 * t + q))) & 0xF);
          const float px = vl[e][0], py = vl[e][1], pz = vl[e][2];
          float* vo = verts + ((size_t)tri * 3 + q) * 3;
          vo[0] = px * vs; vo[1] = py * vs; vo[2] = pz * vs;
          if (colors) mc_vertex_color(g, s, i, j, k, step, e, val, colors + ((size_t)tri * 3 + q) * 3);
          float* no = normals + ((size_t)tri * 3 + q) * 3;
          if (!(isfinite(px) && isfinite(py) && isfinite(pz))) {
            no[0] = no[1] = no[2] = __int_as_float(0x7fc00000);
            continue;
          }
          const int qx = (int)roundf(px), qy = (int)roundf(py), qz = (int)roundf(pz);
          float a0, a1;
          int o;
          mc_read(g, s, qx + 1, qy, qz, a0, o); mc_read(g, s, qx - 1, qy, qz, a1, o);
          const float nx = a0 - a1;
          mc_read(g, s, qx, qy + 1, qz, a0, o); mc_read(g, s, qx, qy - 1, qz, a1, o);
          const float ny = a0 - a1;
          mc_read(g, s, qx, qy, qz + 1, a0, o); mc_read(g, s, qx, qy, qz - 1, a1, o);
          const float nz = a0 - a1;
          const float nn = sqrtf((nx * nx + ny * ny) + nz * nz);
          no[0] = nx / nn; no[1] = ny / nn; no[2] = nz / nn;
        }
      }
    }
  }
}

extern "C" int tslam_mc_generate(tslam_tsdf_t* m, int32_t step, float thres, int64_t cap_tri, float* verts, float* normals,
                                 int64_t* n_tri_out, void* stream) {
  return tslam_mc_generate2(m, step, thres, cap_tri, verts, normals, nullptr, n_tri_out, stream);
}
extern "C" int tslam_mc_generate2(tslam_tsdf_t* m, int32_t step, float thres, int64_t cap_tri, float* verts, float* normals,
                                  float* colors, int64_t* n_tri_out, void* stream) {
  if (!m || !verts || !normals || !n_tri_out || step < 1 || cap_tri < 0) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = mc_upload_tables();
  if (rc) return rc;
  rc = ts_flush_pending(m, st);
  if (rc) return rc;
  unsigned long long total = 0;
  unsigned long long* d_total = (unsigned long long*)(m->scratch_i + 10);
  if (step == 1) {
    if (!m->mc_scratch) TS_CUDA(cudaMalloc(&m->mc_scratch, (size_t)m->g.max_blocks * 12));  // persistent: per-block counts + offsets
    unsigned long long* blk_off = (unsigned long long*)m->mc_scratch;
    unsigned int* blk_tris = (unsigned int*)(blk_off + m->g.max_blocks);
    k_mc_count<false><<<m->sm_count * 4, 256, 0, st>>>(m->g, thres, blk_tris, nullptr, nullptr, nullptr);
    TS_LAUNCH_CHECK(m);
    k_mc_scan<<<1, 1024, 0, st>>>(m->g.n_blocks, m->g.max_blocks, blk_tris, blk_off, d_total);
    TS_LAUNCH_CHECK(m);
    k_mc_emit<false><<<m->sm_count * 4, 256, 0, st>>>(m->g, thres, m->in.vs, blk_tris, blk_off, cap_tri, verts, normals, colors, nullptr,
                                                      nullptr);
    TS_LAUNCH_CHECK(m);
    TS_CUDA(cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
  } else {
    TS_CUDA(cudaMemsetAsync(d_total, 0, 8, st));
    k_mc_generic<<<m->sm_count * 8, 256, 0, st>>>(m->g, step, thres, m->in.vs, cap_tri, verts, normals, colors, d_total);
    TS_LAUNCH_CHECK(m);
    TS_CUDA(cudaMemcpyAsync(&total, d_total, 8, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
  }
  *n_tri_out = (int64_t)total;
  rc = ts_check_deferred(m);  // a map that silently stopped growing (pool exhausted) must not be meshed as if complete
  if (rc) return rc;
  if ((int64_t)total > cap_tri) {
    ts_set_error("marching cubes: %lld triangles > capacity %lld (output saturated)", (long long)total, (long long)cap_tri);
    return TSLAM_E_CAPACITY;
  }
  return TSLAM_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Incremental mesh (tslam_mesh_*): the step-1 mesh of one map kept on the device, remeshing only the blocks a commit
// could have changed.  Output bit-identical to tslam_mc_generate2(step = 1); the dependency argument is in DESIGN.md
// section 4.  Blocks keep the pool order of the two-pass mesh: block b's triangles sit at off[b] .. off[b] + cnt[b].
// ---------------------------------------------------------------------------------------------------------------------
struct McCtl {
  unsigned long long total;  // triangles of the new mesh (k_mc_scan)
  int n_stamp, n_touch, n_dirty, nb;
};

struct tslam_mesh {
  tslam_tsdf* m;
  unsigned int* cnt;            // [max_blocks] triangles per block of the kept mesh
  unsigned long long* off[2];   // [max_blocks] first triangle per block, one array per mesh buffer
  uint8_t* neg;                 // [max_blocks] mc_block_neg at the last update
  uint8_t* neg_now;             // [max_blocks] mc_block_neg now (stamped blocks only, written by k_mesh_touch)
  int* touch_flag;              // [max_blocks] block is on touch_list (cleared again by k_mesh_dirty)
  int* stamp_list;              // [max_blocks]
  int* touch_list;              // [max_blocks]
  int* dirty_list;              // [max_blocks] blocks remeshed by this update
  unsigned int* mark;           // [max_blocks] number of the last update that remeshed the block
  McCtl* ctl;
  float* buf[2];                // mesh buffers: verts | normals [| colours], planes of cap[i] * 9 floats
  long long cap[2];
  int cur;                      // buffer (and offsets) of the kept mesh
  int valid;                    // an update completed and the kept state describes the map
  int colored, full, nb;
  long long total;              // triangles of the kept mesh
  float thres;
  unsigned long long seq, epoch;
  unsigned int upd;             // updates so far
};

static inline float* mc_plane(tslam_mesh* c, int i, int p) { return c->buf[i] + (size_t)p * (size_t)c->cap[i] * 9; }

// step 0 (incremental): list the blocks stamped since the last update.  Blocks allocated since then (b >= nb_last)
// had no triangles and no negative voxel.
__global__ void __launch_bounds__(256) k_mesh_stamped(TsGrid g, const unsigned long long* stamp, unsigned long long seq, int nb_last,
                                                       unsigned int* cnt, uint8_t* neg, int* stamp_list, McCtl* ctl) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  if (blockIdx.x == 0 && threadIdx.x == 0) ctl->nb = nb;
  const int stride = gridDim.x * blockDim.x;
  const int iters = (nb + stride - 1) / stride;
  for (int it = 0; it < iters; ++it) {  // uniform trip count: the append below is warp-collective
    const int b = it * stride + blockIdx.x * blockDim.x + threadIdx.x;
    bool want = false;
    if (b < nb) {
      if (b >= nb_last) { cnt[b] = 0; neg[b] = 0; }
      want = stamp[b] > seq;
    }
    const int row = warp_append_i32(want, &ctl->n_stamp);
    if (want) stamp_list[row] = b;
  }
}

// full rebuild: every block is listed
__global__ void __launch_bounds__(256) k_mesh_all(TsGrid g, int* dirty_list, McCtl* ctl) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  if (blockIdx.x == 0 && threadIdx.x == 0) { ctl->nb = nb; ctl->n_dirty = nb; }
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) dirty_list[b] = b;
}

// mark, kernel A: one CTA per stamped block S.  neg_now[S], then every existing block of S's 27-neighbourhood is
// touched (its mesh reads S), each listed once.
__global__ void __launch_bounds__(256) k_mesh_touch(TsGrid g, const int* stamp_list, uint8_t* neg_now, int* touch_flag, int* touch_list,
                                                     McCtl* ctl) {
  const int n = ctl->n_stamp;
  for (int q = blockIdx.x; q < n; q += gridDim.x) {
    const int b = stamp_list[q];
    const bool ng = mc_block_neg(g, b);
    if (threadIdx.x < 32) {
      if (threadIdx.x == 0) neg_now[b] = ng;
      int s, bx, by, bz;
      ts_unpack_key(g.block_key[b], s, bx, by, bz);
      int nbk = -1;
      if (threadIdx.x < 27)  // the keys mc_stage looks up, wrapped the same way
        nbk = ts_find(g, ts_pack_key(s, bx + (int)threadIdx.x / 9 - 1, by + ((int)threadIdx.x / 3) % 3 - 1, bz + (int)threadIdx.x % 3 - 1));
      const bool want = nbk >= 0 && atomicExch(&touch_flag[nbk], 1) == 0;
      const int row = warp_append_i32(want, &ctl->n_touch);
      if (want) touch_list[row] = nbk;
    }
  }
}

// mark, kernel B: one lane per touched block B.  Dirty iff some block M of B + {0,1}^3 had or has a negative observed
// voxel (neg_then(M) || neg_now(M); neg_now = neg_then unless M is stamped).
__global__ void __launch_bounds__(256) k_mesh_dirty(TsGrid g, const unsigned long long* stamp, unsigned long long seq, const uint8_t* neg,
                                                     const uint8_t* neg_now, int* touch_flag, const int* touch_list, int* dirty_list,
                                                     unsigned int* mark, unsigned int upd, McCtl* ctl) {
  const int n = ctl->n_touch;
  const int stride = gridDim.x * blockDim.x;
  const int iters = (n + stride - 1) / stride;
  for (int it = 0; it < iters; ++it) {
    const int i = it * stride + blockIdx.x * blockDim.x + threadIdx.x;
    bool want = false;
    int b = -1;
    if (i < n) {
      b = touch_list[i];
      touch_flag[b] = 0;
      int s, bx, by, bz;
      ts_unpack_key(g.block_key[b], s, bx, by, bz);
      for (int d = 0; d < 8 && !want; d++) {
        const int mb = ts_find(g, ts_pack_key(s, bx + (d >> 2), by + ((d >> 1) & 1), bz + (d & 1)));
        if (mb >= 0) want = neg[mb] || (stamp[mb] > seq && neg_now[mb]);
      }
      if (want) mark[b] = upd;
    }
    const int row = warp_append_i32(want, &ctl->n_dirty);
    if (want) dirty_list[row] = b;
  }
}

// n floats src -> dst by one CTA: 16-byte loads from the source's first aligned word on, 16-byte stores when the
// destination shares that alignment, else four 4-byte stores
__device__ __forceinline__ void mc_copy_range(const float* __restrict__ src, float* __restrict__ dst, size_t n) {
  const size_t head = min((size_t)((4 - (((uintptr_t)src >> 2) & 3)) & 3), n);
  if (threadIdx.x < head) dst[threadIdx.x] = src[threadIdx.x];
  const size_t nv = (n - head) >> 2;
  const float4* s4 = reinterpret_cast<const float4*>(src + head);
  float* d = dst + head;
  if ((((uintptr_t)d) & 15) == 0) {
    float4* d4 = reinterpret_cast<float4*>(d);
    for (size_t i = threadIdx.x; i < nv; i += blockDim.x) d4[i] = s4[i];
  } else {
    for (size_t i = threadIdx.x; i < nv; i += blockDim.x) {
      const float4 v = s4[i];
      d[4 * i] = v.x; d[4 * i + 1] = v.y; d[4 * i + 2] = v.z; d[4 * i + 3] = v.w;
    }
  }
  for (size_t i = head + 4 * nv + threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

// clean blocks with triangles: their range moves from the kept mesh to the new offsets, one CTA per block
struct McPlanes { const float* src[3]; float* dst[3]; int n; };
__global__ void __launch_bounds__(256) k_mesh_copy(int nb_last, const unsigned int* cnt, const unsigned int* mark, unsigned int upd,
                                                    const unsigned long long* off_old, const unsigned long long* off_new, McPlanes p) {
  for (int b = blockIdx.x; b < nb_last; b += gridDim.x) {
    const unsigned int n = cnt[b];
    if (n == 0 || mark[b] == upd) continue;
    const size_t so = (size_t)off_old[b] * 9, dn = (size_t)off_new[b] * 9;
#pragma unroll
    for (int k = 0; k < 3; k++)  // (constant indices: the planes stay in the parameter space, no local copy)
      if (k < p.n) mc_copy_range(p.src[k] + so, p.dst[k] + dn, (size_t)n * 9);
  }
}

// the remeshed blocks in pool order (single CTA, ordered compaction): keys, first triangle, triangle count
__global__ void __launch_bounds__(1024) k_mesh_updated(TsGrid g, int nb, int full, const unsigned int* mark, unsigned int upd, const unsigned int* cnt,
                                                        const unsigned long long* off, long long cap, int* blk4, long long* first, int* ntri,
                                                        long long* n_out) {
  __shared__ int wsum[32];
  __shared__ long long carry;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += 1024) {
    const int b = base + threadIdx.x;
    const bool want = b < nb && (full || mark[b] == upd);
    const unsigned m = __ballot_sync(0xffffffffu, want);
    if (lane == 0) wsum[wid] = __popc(m);
    __syncthreads();
    int woff = 0, tot = 0;
    for (int w = 0; w < 32; w++) {
      const int x = wsum[w];
      if (w < wid) woff += x;
      tot += x;
    }
    const long long row = carry + woff + __popc(m & ((1u << lane) - 1));
    if (want && row < cap) {
      int s, bx, by, bz;
      ts_unpack_key(g.block_key[b], s, bx, by, bz);
      blk4[4 * row] = s; blk4[4 * row + 1] = bx; blk4[4 * row + 2] = by; blk4[4 * row + 3] = bz;
      first[row] = (long long)off[b];
      ntri[row] = (int)cnt[b];
    }
    __syncthreads();
    if (threadIdx.x == 0) carry += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) *n_out = carry;
}

static void mc_mesh_free_bufs(tslam_mesh* c) {
  for (int i = 0; i < 2; i++) {
    if (c->buf[i]) cudaFree(c->buf[i]);
    c->buf[i] = nullptr;
    c->cap[i] = 0;
  }
}

extern "C" int tslam_mesh_create(tslam_tsdf_t* m, tslam_mesh_t** out) {
  if (!m || !out) return TSLAM_E_INVALID;
  *out = nullptr;
  tslam_mesh* c = new tslam_mesh();
  memset(c, 0, sizeof(*c));
  c->m = m;
  const size_t mb = (size_t)m->g.max_blocks;
  int rc = TSLAM_OK;
  auto alloc = [&](void** p, size_t bytes) {
    if (rc) return;
    if (cudaMalloc(p, bytes) != cudaSuccess || cudaMemset(*p, 0, bytes) != cudaSuccess) rc = ts_cuda_fail(cudaGetLastError(), "tslam_mesh_create");
  };
  alloc((void**)&c->cnt, mb * 4);
  alloc((void**)&c->off[0], mb * 8);
  alloc((void**)&c->off[1], mb * 8);
  alloc((void**)&c->neg, mb);
  alloc((void**)&c->neg_now, mb);
  alloc((void**)&c->touch_flag, mb * 4);
  alloc((void**)&c->stamp_list, mb * 4);
  alloc((void**)&c->touch_list, mb * 4);
  alloc((void**)&c->dirty_list, mb * 4);
  alloc((void**)&c->mark, mb * 4);
  alloc((void**)&c->ctl, sizeof(McCtl));
  if (rc) { tslam_mesh_destroy(c); return rc; }
  *out = c;
  return TSLAM_OK;
}

extern "C" int tslam_mesh_destroy(tslam_mesh_t* c) {
  if (!c) return TSLAM_OK;
  cudaDeviceSynchronize();
  void* p[] = {c->cnt, c->off[0], c->off[1], c->neg, c->neg_now, c->touch_flag, c->stamp_list, c->touch_list, c->dirty_list, c->mark, c->ctl};
  for (void* q : p)
    if (q) cudaFree(q);
  mc_mesh_free_bufs(c);
  delete c;
  return TSLAM_OK;
}

extern "C" int tslam_mesh_update(tslam_mesh_t* c, float thres, int64_t cap_tri, float* verts, float* normals, float* colors,
                                 int64_t* n_tri_out, int32_t* stats4, void* stream) {
  if (!c || !verts || !normals || !n_tri_out || cap_tri < 0) return TSLAM_E_INVALID;
  tslam_tsdf* m = c->m;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = mc_upload_tables();
  if (rc) return rc;
  rc = ts_flush_pending(m, st);
  if (rc) return rc;
  const int colored = colors != nullptr;
  const bool full = !c->valid || c->epoch != m->mesh_epoch || memcmp(&c->thres, &thres, sizeof(float)) != 0 || c->colored != colored;
  c->valid = 0;  // until this update completes
  if (c->colored != colored) {
    TS_CUDA(cudaStreamSynchronize(st));
    mc_mesh_free_bufs(c);  // a different number of planes
    c->colored = colored;
  }
  const unsigned long long seq = m->commit_seq;  // stamps above this are seen by the next update
  const unsigned int upd = ++c->upd;
  McCtl h;
  memset(&h, 0, sizeof(h));
  int out = c->cur;
  int nb_now = 0;
  // Nothing committed or imported since the last update: no block is stamped, none is remeshed, and the kept mesh is the
  // answer.  Blocks allocated since hold no triangles; c->nb stays, so the next pass initialises them.
  const bool unchanged = !full && seq == c->seq;
  if (unchanged) {
    h.total = (unsigned long long)c->total;
    TS_CUDA(cudaMemcpyAsync(&nb_now, m->g.n_blocks, 4, cudaMemcpyDeviceToHost, st));  // (statistics only; read after the sync below)
  } else {
    const int grid = m->sm_count * 4;
    TS_CUDA(cudaMemsetAsync(c->ctl, 0, sizeof(McCtl), st));
    if (full) {
      TS_CUDA(cudaMemsetAsync(c->touch_flag, 0, (size_t)m->g.max_blocks * 4, st));
      k_mesh_all<<<grid, 256, 0, st>>>(m->g, c->dirty_list, c->ctl);
      TS_LAUNCH_CHECK(m);
    } else {
      k_mesh_stamped<<<grid, 256, 0, st>>>(m->g, m->blk_stamp, c->seq, c->nb, c->cnt, c->neg, c->stamp_list, c->ctl);
      TS_LAUNCH_CHECK(m);
      k_mesh_touch<<<grid, 256, 0, st>>>(m->g, c->stamp_list, c->neg_now, c->touch_flag, c->touch_list, c->ctl);
      TS_LAUNCH_CHECK(m);
      k_mesh_dirty<<<grid, 256, 0, st>>>(m->g, m->blk_stamp, c->seq, c->neg, c->neg_now, c->touch_flag, c->touch_list, c->dirty_list,
                                         c->mark, upd, c->ctl);
      TS_LAUNCH_CHECK(m);
    }
    const int nxt = c->cur ^ 1;
    k_mc_count<true><<<grid, 256, 0, st>>>(m->g, thres, c->cnt, c->dirty_list, &c->ctl->n_dirty, c->neg);
    TS_LAUNCH_CHECK(m);
    k_mc_scan<<<1, 1024, 0, st>>>(m->g.n_blocks, m->g.max_blocks, c->cnt, c->off[nxt], &c->ctl->total);
    TS_LAUNCH_CHECK(m);
    TS_CUDA(cudaMemcpyAsync(&h, c->ctl, sizeof(McCtl), cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
    nb_now = h.nb;
    if (h.n_dirty > 0) {
      // (no block remeshed: nothing moved, the kept mesh and its offsets stay as they are - blocks allocated since hold
      // no triangles)
      const long long total = (long long)h.total;
      const int planes = colored ? 3 : 2;
      if (total > c->cap[nxt]) {
        if (c->buf[nxt]) TS_CUDA(cudaFree(c->buf[nxt]));
        c->buf[nxt] = nullptr;
        c->cap[nxt] = 0;
        const long long want = total + total / 4 + 1024;
        TS_CUDA(cudaMalloc(&c->buf[nxt], (size_t)want * 9 * sizeof(float) * planes));
        c->cap[nxt] = want;
      }
      k_mc_emit<true><<<grid, 256, 0, st>>>(m->g, thres, m->in.vs, c->cnt, c->off[nxt], c->cap[nxt], mc_plane(c, nxt, 0), mc_plane(c, nxt, 1),
                                            colored ? mc_plane(c, nxt, 2) : nullptr, c->dirty_list, &c->ctl->n_dirty);
      TS_LAUNCH_CHECK(m);
      if (!full && c->nb > 0) {
        McPlanes p;
        p.n = planes;
        for (int k = 0; k < 3; k++) {
          p.src[k] = k < planes ? mc_plane(c, c->cur, k) : nullptr;
          p.dst[k] = k < planes ? mc_plane(c, nxt, k) : nullptr;
        }
        k_mesh_copy<<<grid, 256, 0, st>>>(c->nb, c->cnt, c->mark, upd, c->off[c->cur], c->off[nxt], p);
        TS_LAUNCH_CHECK(m);
      }
      out = nxt;
    }
  }
  // one tail for both: the output contract of tslam_mc_generate2(step = 1)
  const long long total = (long long)h.total;
  const long long n_out = total < cap_tri ? total : (long long)cap_tri;
  if (n_out > 0) {
    const size_t bytes = (size_t)n_out * 9 * sizeof(float);
    TS_CUDA(cudaMemcpyAsync(verts, mc_plane(c, out, 0), bytes, cudaMemcpyDeviceToDevice, st));
    TS_CUDA(cudaMemcpyAsync(normals, mc_plane(c, out, 1), bytes, cudaMemcpyDeviceToDevice, st));
    if (colored) TS_CUDA(cudaMemcpyAsync(colors, mc_plane(c, out, 2), bytes, cudaMemcpyDeviceToDevice, st));
  }
  TS_CUDA(cudaStreamSynchronize(st));
  c->cur = out;
  c->seq = seq;
  c->epoch = m->mesh_epoch;
  c->thres = thres;
  if (!unchanged) c->nb = h.nb;
  c->total = total;
  c->full = full;
  c->valid = 1;
  if (stats4) {
    stats4[0] = nb_now < m->g.max_blocks ? nb_now : m->g.max_blocks;
    stats4[1] = h.n_stamp; stats4[2] = h.n_touch; stats4[3] = h.n_dirty;
  }
  *n_tri_out = (int64_t)total;
  rc = ts_check_deferred(m);  // as tslam_mc_generate2
  if (rc) return rc;
  if (total > cap_tri) {
    ts_set_error("marching cubes: %lld triangles > capacity %lld (output saturated)", total, (long long)cap_tri);
    return TSLAM_E_CAPACITY;
  }
  return TSLAM_OK;
}

extern "C" int tslam_mesh_updated_blocks(tslam_mesh_t* c, int64_t cap, int32_t* blk4, int64_t* first_tri, int32_t* n_tri, int64_t* n_out,
                                         int32_t* full_out, void* stream) {
  if (!c || !n_out || cap < 0 || (cap > 0 && (!blk4 || !first_tri || !n_tri))) return TSLAM_E_INVALID;
  if (!c->valid) { ts_set_error("tslam_mesh_updated_blocks: no completed update"); return TSLAM_E_INVALID; }
  tslam_tsdf* m = c->m;
  cudaStream_t st = (cudaStream_t)stream;
  long long* d_n = (long long*)&c->ctl->total;  // (the update's scratch word, free between updates)
  k_mesh_updated<<<1, 1024, 0, st>>>(m->g, c->nb, c->full, c->mark, c->upd, c->cnt, c->off[c->cur], cap, blk4, (long long*)first_tri, n_tri, d_n);
  TS_LAUNCH_CHECK(m);
  long long n = 0;
  TS_CUDA(cudaMemcpyAsync(&n, d_n, 8, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  *n_out = (int64_t)n;
  if (full_out) *full_out = c->full;
  if (n > cap) {
    ts_set_error("tslam_mesh_updated_blocks: %lld blocks > capacity %lld (output saturated)", n, (long long)cap);
    return TSLAM_E_CAPACITY;
  }
  return TSLAM_OK;
}
