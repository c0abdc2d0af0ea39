// libtslam.so - TSDF map: hash grid of 16^3 voxel blocks; the handle, I/O, export and fusion kernels.  sm_90a.
// (Integration lives in tslam_integrate.cu, tslam_march.cu and tslam_queue.cu.)
//
// Reference semantics: taichi_slam/mapping/dense_tsdf.py (cited per kernel).
// Compiled with -fmad=false: the index-forming arithmetic must round exactly like
// the strict-IEEE statement of the reference source (voxel indices are compared
// bit-for-bit by the parity tests).
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <cmath>
#include <mutex>
#include <unordered_map>
#include <vector>
#include <cuda_fp16.h>
#include "tslam_internal.cuh"
#include "tslam_bucket.cuh"

// ---------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------
static thread_local char g_err[512] = "";
void ts_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int ts_cuda_fail(cudaError_t e, const char* what) {
  ts_set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) ? TSLAM_E_NOGPU : TSLAM_E_CUDA;
}
extern "C" const char* tslam_last_error(void) { return g_err; }
extern "C" int tslam_abi_version(void) { return TSLAM_ABI_VERSION; }
extern "C" int tslam_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

// ---------------------------------------------------------------------------
// host: create / destroy / reset
// ---------------------------------------------------------------------------
static size_t next_pow2(size_t v) {
  size_t p = 1;
  while (p < v) p <<= 1;
  return p;
}

static void fill_jet_host(float* cm) {
  // colormap[i] = matplotlib.cm.jet(i/1024) (mapping_common.py:158-163) = 256-entry LUT of
  // the piecewise-linear jet segment data, sampled at i//4.
  static const float r[][2] = {{0, 0}, {0.35f, 0}, {0.66f, 1}, {0.89f, 1}, {1, 0.5f}};
  static const float gg[][2] = {{0, 0}, {0.125f, 0}, {0.375f, 1}, {0.64f, 1}, {0.91f, 0}, {1, 0}};
  static const float b[][2] = {{0, 0.5f}, {0.11f, 1}, {0.34f, 1}, {0.65f, 0}, {1, 0}};
  auto seg = [](const float (*d)[2], int n, float x) {
    for (int i = 1; i < n; i++)
      if (x <= d[i][0]) {
        float t = (x - d[i - 1][0]) / (d[i][0] - d[i - 1][0]);
        return d[i - 1][1] + t * (d[i][1] - d[i - 1][1]);
      }
    return d[n - 1][1];
  };
  for (int i = 0; i < 1024; i++) {
    float x = (float)(i / 4) / 255.0f;
    cm[3 * i] = seg(r, 5, x);
    cm[3 * i + 1] = seg(gg, 6, x);
    cm[3 * i + 2] = seg(b, 5, x);
  }
}

// Whether div_vs(a, b, RN(1/b)) equals the IEEE quotient a / b for every f32 a whose quotient and residual stay normal
// (|a| within about 2^+-100 of b).  Scaling a by a power of two scales q0, the residual and the result alike, so the
// 2^23 significands of [1, 2) decide it.  About 70 ms per divisor; the answers are kept, since handles are created
// and re-calibrated with a handful of focal lengths.
static bool ts_fdiv_exact(float b) {
  static std::mutex mu;
  static std::unordered_map<uint32_t, bool> known;
  uint32_t bb;
  std::memcpy(&bb, &b, 4);
  std::lock_guard<std::mutex> lock(mu);
  const auto it = known.find(bb);
  if (it != known.end()) return it->second;
  bool ok = std::isnormal(b) && std::isnormal(1.0f / b);
  const volatile float vb = b;  // a / vb: the IEEE division, not a multiplication by a folded reciprocal
  const float r = 1.0f / b;
  for (uint32_t s = 0; ok && s < (1u << 23); ++s) {
    const uint32_t ab = 0x3f800000u | s;
    float a;
    std::memcpy(&a, &ab, 4);
    const float q0 = a * r;
    const float q1 = std::fmaf(std::fmaf(-q0, b, a), r, q0);
    ok = q1 == a / vb;
  }
  known.emplace(bb, ok);
  return ok;
}

static void ts_fill_intrin(tslam_tsdf* m) {
  const tslam_tsdf_config_t& c = m->cfg;
  m->in.fx = (float)c.fx; m->in.fy = (float)c.fy; m->in.cx = (float)c.cx; m->in.cy = (float)c.cy;
  m->in.rfx = 1.0f / m->in.fx; m->in.rfy = 1.0f / m->in.fy;
  m->in.fdiv = ts_fdiv_exact(m->in.fx) && ts_fdiv_exact(m->in.fy);
  m->in.dmin_mm = (float)(c.min_ray_length * 1000.0);
  m->in.dmax_mm = (float)(c.max_ray_length * 1000.0);
  m->in.vs = (float)c.voxel_scale;
  m->in.rvs = 1.0f / m->in.vs;
  m->in.max_steps = (float)(c.max_ray_length / c.voxel_scale);
  m->in.max_ray = (float)c.max_ray_length;
  m->in.internal_voxels = c.internal_voxels;
  m->in.step = c.recast_step;
  m->in.tex = c.texture_enabled;
}


extern "C" int tslam_tsdf_create(const tslam_tsdf_config_t* cfg, tslam_tsdf_t** out) {
  if (!cfg || !out) { ts_set_error("null argument"); return TSLAM_E_INVALID; }
  *out = nullptr;
  if (cfg->voxel_scale <= 0 || cfg->N <= 0 || cfg->Nz <= 0 || cfg->recast_step <= 0 || cfg->N > 16384 || cfg->Nz > 16384) {
    ts_set_error("invalid config (voxel_scale/N/Nz/recast_step)");
    return TSLAM_E_INVALID;
  }
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    ts_set_error("no CUDA device visible: libtslam has no CPU fallback");
    return TSLAM_E_NOGPU;
  }
  tslam_tsdf* m = new tslam_tsdf();
  memset(m, 0, sizeof(*m));
  m->cfg = *cfg;
  TS_CUDA(cudaGetDevice(&m->device));
  cudaDeviceProp prop;
  TS_CUDA(cudaGetDeviceProperties(&prop, m->device));
  m->sm_count = prop.multiProcessorCount;
  if (m->cfg.max_submaps <= 0) m->cfg.max_submaps = 1024;
  if (m->cfg.max_submaps > 1024) m->cfg.max_submaps = 1024;
  if (m->cfg.max_image_pixels <= 0) m->cfg.max_image_pixels = 640 * 480;
  if (m->cfg.max_points <= 0) m->cfg.max_points = 1 << 20;
  // block pool capacity: the dense block count when that is small, else 32768 blocks
  const long long nb = (long long)((cfg->N + TS_B - 1) / TS_B + 1);
  const long long nbz = (long long)((cfg->Nz + TS_B - 1) / TS_B + 1);
  long long dense_blocks = nb * nb * nbz * (cfg->is_global_map ? 1 : 4);
  // default pool: the dense block count, at least 32768 blocks (2.4 GB: a submap collection keeps growing with every
  // keyframe - the reference's pointer SNodes grow on demand), at most 131072 (9.4 GB); callers that know better pass
  // max_blocks.  Exhaustion drops samples and raises a sticky TSLAM_E_POOL_FULL on the next flush / reader.
  if (m->cfg.max_blocks <= 0) m->cfg.max_blocks = (int)(dense_blocks < 32768 ? 32768 : (dense_blocks > 131072 ? 131072 : dense_blocks));
  if (m->cfg.max_blocks > TS_MAX_BLOCKS) m->cfg.max_blocks = TS_MAX_BLOCKS;
  ts_fill_intrin(m);
  m->clamp_on_commit = true;

  TsGrid& g = m->g;
  g.max_blocks = m->cfg.max_blocks;
  g.N = cfg->N; g.Nz = cfg->Nz; g.hN = cfg->N / 2; g.hNz = cfg->Nz / 2;
  m->table_cap = next_pow2((size_t)g.max_blocks * 2 + 64);
  g.table_mask = (uint32_t)(m->table_cap - 1);
  const size_t nv = (size_t)g.max_blocks * TS_B3;
  TS_CUDA(cudaMalloc(&g.table, m->table_cap * 8));
  TS_CUDA(cudaMemset(g.table, 0xFF, m->table_cap * 8));
  TS_CUDA(cudaMalloc(&g.block_key, (size_t)g.max_blocks * 8));
  TS_CUDA(cudaMalloc(&g.acc, nv * sizeof(float2)));
  TS_CUDA(cudaMalloc(&g.tw, nv * sizeof(float2)));
  TS_CUDA(cudaMalloc(&g.obs, nv));
  TS_CUDA(cudaMalloc(&g.occ, nv));
  TS_CUDA(cudaMemset(g.acc, 0, nv * sizeof(float2)));
  TS_CUDA(cudaMemset(g.tw, 0, nv * sizeof(float2)));
  TS_CUDA(cudaMemset(g.obs, 0, nv));
  TS_CUDA(cudaMemset(g.occ, 0, nv));
  g.esdf = nullptr;
  g.cword = nullptr;
  g.col = nullptr;
  if (m->cfg.texture_enabled) {
    TS_CUDA(cudaMalloc(&g.cword, nv * 8));
    TS_CUDA(cudaMalloc(&g.col, nv * 16));
    TS_CUDA(cudaMemset(g.cword, 0, nv * 8));
    TS_CUDA(cudaMemset(g.col, 0, nv * 16));
  }
  TS_CUDA(cudaMalloc(&g.ghost, (size_t)g.max_blocks));
  TS_CUDA(cudaMemset(g.ghost, 0, (size_t)g.max_blocks));
  TS_CUDA(cudaMalloc(&g.dirty_flag, (size_t)g.max_blocks * 4));
  TS_CUDA(cudaMalloc(&g.dirty_list, (size_t)g.max_blocks * 4));
  TS_CUDA(cudaMemset(g.dirty_flag, 0, (size_t)g.max_blocks * 4));
  TS_CUDA(cudaMalloc(&g.esdf_dirty, (size_t)g.max_blocks * 4));
  TS_CUDA(cudaMemset(g.esdf_dirty, 0, (size_t)g.max_blocks * 4));
  TS_CUDA(cudaMalloc(&m->blk_stamp, (size_t)g.max_blocks * 8));
  TS_CUDA(cudaMemset(m->blk_stamp, 0, (size_t)g.max_blocks * 8));
  TS_CUDA(cudaMalloc(&m->scratch_i, 64 * sizeof(int)));
  TS_CUDA(cudaMemset(m->scratch_i, 0, 64 * sizeof(int)));
  g.n_blocks = m->scratch_i + 0;
  g.n_dirty = m->scratch_i + 1;
  g.err = m->scratch_i + 2;
  m->n_rays = m->scratch_i + 3;

  // integrate workspace
  const int step = m->cfg.recast_step;
  size_t sampled = (size_t)m->cfg.max_image_pixels / ((size_t)step * step) + 1024;
  m->bucket_cap = (uint32_t)next_pow2(sampled + sampled / 2);
  if (const char* bc = getenv("TSLAM_BUCKET_CAP")) { if (atoi(bc) >= 1024) m->bucket_cap = (uint32_t)next_pow2((size_t)atoi(bc)); }  // experiment
  // the point-cloud path treats the TSLAM_MAX_BATCH per-frame tables as ONE table
  if ((size_t)m->cfg.max_points * 3 / 2 > (size_t)TSLAM_MAX_BATCH * m->bucket_cap || (size_t)m->cfg.max_points > BK_MAX_SLOTS || m->bucket_cap > BK_MAX_SLOTS) {
    ts_set_error("max_points=%d too large for the bucket workspace", m->cfg.max_points);
    return TSLAM_E_INVALID;
  }
  TS_CUDA(cudaMalloc(&m->buckets, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * sizeof(TsBucket)));
  if (m->cfg.texture_enabled) TS_CUDA(cudaMalloc(&m->bcol, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * sizeof(uint4)));
  TS_CUDA(cudaMalloc(&m->bidx, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * 8));
  TS_CUDA(cudaMemset(m->bidx, 0, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * 8));
  m->bk_slot_bits = ts_bucket_slot_bits(m->bucket_cap, (uint32_t)m->cfg.max_points);
  if (m->bk_slot_bits >= TS_BK_SLOT_FIELD) TS_CUDA(cudaMalloc(&m->bpos, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * 4));
  m->bk_epoch_max = m->bk_slot_bits >= TS_BK_SLOT_FIELD ? 0u : (1u << (TS_BK_SLOT_FIELD - m->bk_slot_bits)) - 1u;
  m->bk_epoch = 0;
  {  // a launch in which one bucket can collect more points than the packed count word holds keeps its counts in a plane
    const uint64_t n_max = std::max((uint64_t)m->cfg.max_image_pixels / ((uint64_t)step * step), (uint64_t)m->cfg.max_points);
    if (ts_bucket_cnt_shift(n_max, ts_bucket_dmax(m)) < 0) TS_CUDA(cudaMalloc(&m->bcnt, (size_t)TSLAM_MAX_BATCH * m->bucket_cap * 4));
  }
  m->ray_list_cap = (uint32_t)((size_t)TSLAM_MAX_BATCH * sampled);
  if (m->ray_list_cap < (uint32_t)m->cfg.max_points) m->ray_list_cap = (uint32_t)m->cfg.max_points;
  TS_CUDA(cudaMalloc(&m->ray_list, (size_t)m->ray_list_cap * 4));
  TS_CUDA(cudaMalloc(&m->depth_stage, (size_t)2 * TSLAM_MAX_BATCH * m->cfg.max_image_pixels * 2));  // double buffered
  { int rcq = ts_queue_init(m); if (rcq) return rcq; }
  TS_CUDA(cudaMalloc(&m->points_stage, (size_t)m->cfg.max_points * 12));
  if (m->cfg.texture_enabled) {
    TS_CUDA(cudaMalloc(&m->tex_stage, (size_t)2 * TSLAM_MAX_BATCH * m->cfg.max_image_pixels * 3));
    TS_CUDA(cudaMalloc(&m->rgb_stage, (size_t)m->cfg.max_points * 3));
  }
  TS_CUDA(cudaMalloc(&m->counters, sizeof(TsCounters)));
  TS_CUDA(cudaMemset(m->counters, 0, sizeof(TsCounters)));
  TS_CUDA(cudaMalloc(&m->pose_R, (size_t)m->cfg.max_submaps * 9 * 4));
  TS_CUDA(cudaMalloc(&m->pose_T, (size_t)m->cfg.max_submaps * 3 * 4));
  TS_CUDA(cudaMemset(m->pose_R, 0, (size_t)m->cfg.max_submaps * 9 * 4));  // ti fields start at zero
  TS_CUDA(cudaMemset(m->pose_T, 0, (size_t)m->cfg.max_submaps * 3 * 4));
  std::vector<float> cm(1024 * 3);
  fill_jet_host(cm.data());
  TS_CUDA(cudaMalloc(&m->colormap, cm.size() * 4));
  TS_CUDA(cudaMemcpy(m->colormap, cm.data(), cm.size() * 4, cudaMemcpyHostToDevice));
  m->march_verify = getenv("TSLAM_MARCH_VERIFY") != nullptr;
  // tests: start the frame counter close to the 22-bit limit of the colour word, to run its renormalisation (ts_seq_renorm)
  if (const char* fs = getenv("TSLAM_FRAME_SEQ0")) m->frame_seq = (unsigned)std::min(strtoul(fs, nullptr, 10), (1ul << 22) - 2ul);
  // (the workspace of the block-binned march - ~2 GB for 640x480 frames - is allocated by the first integrate launch:
  // global maps that are only ever fused into never pay for it)
  { int rci = ts_integrate_init(); if (rci) return rci; }
  fz_ver_init(m->ver, m->cfg.max_submaps);
  TS_CUDA(cudaDeviceSynchronize());
  *out = m;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_destroy(tslam_tsdf_t* m) {
  if (!m) return TSLAM_OK;
  cudaDeviceSynchronize();
  TsGrid& g = m->g;
  cudaFree(g.table); cudaFree(g.block_key); cudaFree(g.acc); cudaFree(g.tw); cudaFree(g.obs); cudaFree(g.occ);
  if (g.esdf) cudaFree(g.esdf);
  if (m->esdf_aux) cudaFree(m->esdf_aux);
  if (m->mc_scratch) cudaFree(m->mc_scratch);
  if (m->tile_hist) cudaFree(m->tile_hist);
  if (m->reg_blk) cudaFree(m->reg_blk);
  if (m->reg_pts) cudaFree(m->reg_pts);
  if (m->render_jobs) cudaFree(m->render_jobs);
  if (m->traj_mem) cudaFree(m->traj_mem);
  if (m->rc_mem) cudaFree(m->rc_mem);
  if (g.cword) cudaFree(g.cword);
  if (g.col) cudaFree(g.col);
  if (m->tex_stage) cudaFree(m->tex_stage);
  if (m->rgb_stage) cudaFree(m->rgb_stage);
  cudaFree(g.ghost); cudaFree(g.dirty_flag); cudaFree(g.esdf_dirty); cudaFree(m->blk_stamp); cudaFree(g.dirty_list); cudaFree(m->scratch_i);
  cudaFree(m->buckets); cudaFree(m->bidx); cudaFree(m->ray_list);
  if (m->bcol) cudaFree(m->bcol);
  if (m->bpos) cudaFree(m->bpos);
  if (m->bcnt) cudaFree(m->bcnt);
  cudaFree(m->depth_stage); cudaFree(m->points_stage);
  ts_queue_free(m);
  fz_ver_free(m->ver);
  ts_fuse_free(m);
  if (m->mw.rays) ts_march_free(m);
  cudaFree(m->counters); cudaFree(m->pose_R); cudaFree(m->pose_T); cudaFree(m->colormap);
  if (m->prof) cudaFree(m->prof);
  delete m;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_reset(tslam_tsdf_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  TsGrid& g = m->g;
  int nb = 0;
  m->n_integrate_calls = 0;  // pending sums are discarded with the blocks
  m->esdf_full_needed = 1;   // ... and the ESDF state
  m->mesh_epoch++;           // ... and the incremental mesh (planes cleared and pool slots recycled without stamps)
  m->q_n = 0;                // ... and so are queued frames
  m->q_gathered = 0;
  fz_written(m->ver, -1);    // ... and every submap's content
  TS_CUDA(cudaMemcpyAsync(&nb, g.n_blocks, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (nb > g.max_blocks) nb = g.max_blocks;
  const size_t nv = (size_t)nb * TS_B3;
  TS_CUDA(cudaMemsetAsync(g.table, 0xFF, m->table_cap * 8, st));
  if (nv) {
    TS_CUDA(cudaMemsetAsync(g.acc, 0, nv * sizeof(float2), st));
    TS_CUDA(cudaMemsetAsync(g.tw, 0, nv * sizeof(float2), st));
    TS_CUDA(cudaMemsetAsync(g.obs, 0, nv, st));
    TS_CUDA(cudaMemsetAsync(g.occ, 0, nv, st));
    if (g.esdf) TS_CUDA(cudaMemsetAsync(g.esdf, 0, nv * 4, st));
    TS_CUDA(cudaMemsetAsync(g.dirty_flag, 0, (size_t)nb * 4, st));
    TS_CUDA(cudaMemsetAsync(g.ghost, 0, (size_t)nb, st));
    if (g.cword) TS_CUDA(cudaMemsetAsync(g.cword, 0, nv * 8, st));
    if (g.col) TS_CUDA(cudaMemsetAsync(g.col, 0, nv * 16, st));
  }
  TS_CUDA(cudaMemsetAsync(m->scratch_i, 0, 4 * sizeof(int), st));  // n_blocks, n_dirty, err, n_rays
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_set_intrinsics(tslam_tsdf_t* m, double fx, double fy, double cx, double cy) {
  if (!m) return TSLAM_E_INVALID;
  m->cfg.fx = fx; m->cfg.fy = fy; m->cfg.cx = cx; m->cfg.cy = cy;
  ts_fill_intrin(m);
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_set_color_intrinsics(tslam_tsdf_t* m, double fx, double fy, double cx, double cy, int color_same_proj) {
  if (!m) return TSLAM_E_INVALID;
  m->in.fxc = (float)fx; m->in.fyc = (float)fy; m->in.cxc = (float)cx; m->in.cyc = (float)cy;
  m->in.same_proj = color_same_proj ? 1 : 0;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_set_submap_pose(tslam_tsdf_t* m, int32_t s, const float* R9, const float* T3) {
  if (!m || !R9 || !T3 || s < 0 || s >= m->cfg.max_submaps) { ts_set_error("bad submap id %d", s); return TSLAM_E_INVALID; }
  TS_CUDA(cudaMemcpy(m->pose_R + 9 * (size_t)s, R9, 36, cudaMemcpyHostToDevice));
  TS_CUDA(cudaMemcpy(m->pose_T + 3 * (size_t)s, T3, 12, cudaMemcpyHostToDevice));
  return TSLAM_OK;
}

// ---------------------------------------------------------------------------
// count / gather / scatter  (dense_tsdf.py:412-454)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_count_active(TsGrid g, int submap, unsigned long long* out) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  unsigned int c = 0;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap || g.ghost[b]) continue;
    const uint8_t* obs = g.obs + (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) c += obs[v] > 0;
  }
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

__global__ void __launch_bounds__(256) k_gather(TsGrid g, int submap, long long cap, int32_t* idx, float* tsdf, float* wts,
                                                 int8_t* occ, float* color, unsigned long long* counter) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap || g.ghost[b]) continue;
    const size_t base = (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const bool want = g.obs[base + v] > 0;
      const long long row = warp_append_u64(want, counter);
      if (want && row < cap) {
        idx[3 * row] = bx * TS_B + (v >> 8);
        idx[3 * row + 1] = by * TS_B + ((v >> 4) & 15);
        idx[3 * row + 2] = bz * TS_B + (v & 15);
        const float2 t = g.tw[base + v];
        tsdf[row] = t.x;
        wts[row] = t.y;
        occ[row] = g.occ[base + v];
        if (color) {  // :437-440
          const float4 c = g.col ? g.col[base + v] : make_float4(0.f, 0.f, 0.f, 0.f);
          color[3 * row] = c.x; color[3 * row + 1] = c.y; color[3 * row + 2] = c.z;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_scatter(TsGrid g, int submap, long long n, const int32_t* idx, const float* tsdf,
                                                  const float* wts, const int8_t* occ, const float* color) {
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    const int i = idx[3 * r], j = idx[3 * r + 1], k = idx[3 * r + 2];
    if (!ts_in_bounds(g, i, j, k)) continue;
    const int blk = ts_get_or_alloc(g, ts_pack_key(submap, i >> TS_BSHIFT, j >> TS_BSHIFT, k >> TS_BSHIFT));
    if (blk < 0) continue;
    const size_t o = (size_t)blk * TS_B3 + ts_voxel_off(i, j, k);
    g.tw[o] = make_float2(tsdf[r], wts[r]);  // :447-448
    g.occ[o] = occ[r];                        // :449
    g.obs[o] = 1;                             // :454
    if (color && g.col) g.col[o] = make_float4(color[3 * r], color[3 * r + 1], color[3 * r + 2], 0.0f);  // :450-453
  }
}

extern "C" int tslam_tsdf_count_active(tslam_tsdf_t* m, int32_t submap, int64_t* n_out) {
  if (!m || !n_out) return TSLAM_E_INVALID;
  cudaStream_t st = 0;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  unsigned long long* ctr = (unsigned long long*)(m->scratch_i + 8);
  TS_CUDA(cudaMemsetAsync(ctr, 0, 8, st));
  k_count_active<<<m->sm_count * 4, 256, 0, st>>>(m->g, submap, ctr);
  TS_LAUNCH_CHECK(m);
  unsigned long long v = 0;
  TS_CUDA(cudaMemcpy(&v, ctr, 8, cudaMemcpyDeviceToHost));
  *n_out = (int64_t)v;
  return ts_check_deferred(m);
}

extern "C" int tslam_tsdf_gather(tslam_tsdf_t* m, int32_t submap, int64_t cap, int32_t* idx, float* tsdf, float* w, int8_t* occ,
                                 int64_t* n_out, void* stream) {
  return tslam_tsdf_gather2(m, submap, cap, idx, tsdf, w, occ, nullptr, n_out, stream);
}
extern "C" int tslam_tsdf_gather2(tslam_tsdf_t* m, int32_t submap, int64_t cap, int32_t* idx, float* tsdf, float* w, int8_t* occ,
                                  float* color, int64_t* n_out, void* stream) {
  if (!m || !n_out) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  unsigned long long* ctr = (unsigned long long*)(m->scratch_i + 8);
  TS_CUDA(cudaMemsetAsync(ctr, 0, 8, st));
  k_gather<<<m->sm_count * 4, 256, 0, st>>>(m->g, submap, cap, idx, tsdf, w, occ, color, ctr);
  TS_LAUNCH_CHECK(m);
  unsigned long long v = 0;
  TS_CUDA(cudaMemcpyAsync(&v, ctr, 8, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  *n_out = (int64_t)v;
  rc = ts_check_deferred(m);
  if (rc) return rc;
  if ((int64_t)v > cap) { ts_set_error("gather: %lld observed voxels > capacity %lld", (long long)v, (long long)cap); return TSLAM_E_CAPACITY; }
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_scatter(tslam_tsdf_t* m, int32_t submap, int64_t n, const int32_t* idx, const float* tsdf, const float* w,
                                  const int8_t* occ, void* stream) {
  return tslam_tsdf_scatter2(m, submap, n, idx, tsdf, w, occ, nullptr, stream);
}
extern "C" int tslam_tsdf_scatter2(tslam_tsdf_t* m, int32_t submap, int64_t n, const int32_t* idx, const float* tsdf, const float* w,
                                   const int8_t* occ, const float* color, void* stream) {
  if (!m || n < 0 || submap < 0 || submap >= m->cfg.max_submaps) return TSLAM_E_INVALID;
  if (n == 0) return TSLAM_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  int grid = (int)((n + 255) / 256);
  if (grid > m->sm_count * 32) grid = m->sm_count * 32;
  m->esdf_full_needed = 1;  // bulk load: values change without a commit
  m->mesh_epoch++;          // (same for the incremental mesh)
  fz_written(m->ver, submap);
  k_scatter<<<grid, 256, 0, st>>>(m->g, submap, n, idx, tsdf, w, occ, color);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

// ---------------------------------------------------------------------------
// exporters  (dense_tsdf.py:339-385)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_extract_surface(TsGrid g, int submap, int global_map, const float* pR, const float* pT,
                                                          float vs, float thres, float fl, float ce, const float* cmap,
                                                          long long cap, float* xyz, float* rgb, int* counter) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap || g.ghost[b]) continue;  // :348
    const size_t base = (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      bool want = false;
      float x = 0, y = 0, z = 0;
      if (g.obs[base + v] == 1) {                      // :349
        const float t = g.tw[base + v].x;
        if (fabsf(t) < thres) {                        // :350
          voxel_xyz(g, global_map, pR, pT, s, bx * TS_B + (v >> 8), by * TS_B + ((v >> 4) & 15), bz * TS_B + (v & 15), vs, x, y, z);
          want = !(z > ce || z < fl);                  // :356
        }
      }
      const int row = warp_append_i32(want, counter);  // :358
      if (want && row < cap) {                         // :359 (saturating, see DESIGN.md)
        xyz[3 * (size_t)row] = x; xyz[3 * (size_t)row + 1] = y; xyz[3 * (size_t)row + 2] = z;
        if (rgb && g.col) {  // enable_texture: the voxel's own colour (:360-362)
          const float4 c = g.col[base + v];
          rgb[3 * (size_t)row] = c.x; rgb[3 * (size_t)row + 1] = c.y; rgb[3 * (size_t)row + 2] = c.z;
        } else if (rgb) {
          const int ci = (int)fmaxf(fminf(((z - fl) / (ce - fl)) * 1023.0f, 1023.0f), 0.0f);  // mapping_common.py:216-219
          rgb[3 * (size_t)row] = cmap[3 * ci]; rgb[3 * (size_t)row + 1] = cmap[3 * ci + 1]; rgb[3 * (size_t)row + 2] = cmap[3 * ci + 2];
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_extract_slice(TsGrid g, int submap, int global_map, const float* pR, const float* pT,
                                                        float vs, int index, float dz, const float* cmap, long long cap,
                                                        float* xyz, float* val, float* rgb, int* counter) {
  const int nb = min(*g.n_blocks, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap || g.ghost[b]) continue;  // :375
    const size_t base = (size_t)b * TS_B3;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      const int k = bz * TS_B + (v & 15);
      const bool want = g.obs[base + v] > 0 && ((float)index - dz < (float)k) && ((float)k < (float)index + dz);  // :376-377
      const int row = warp_append_i32(want, counter);
      if (want && row < cap) {
        float x, y, z;
        voxel_xyz(g, global_map, pR, pT, s, bx * TS_B + (v >> 8), by * TS_B + ((v >> 4) & 15), k, vs, x, y, z);
        const float t = g.tw[base + v].x;
        xyz[3 * (size_t)row] = x; xyz[3 * (size_t)row + 1] = y; xyz[3 * (size_t)row + 2] = z;
        if (val) val[row] = t;  // :380
        if (rgb) {
          const int ci = (int)fmaxf(fminf(((t - (-0.5f)) / (0.5f - (-0.5f))) * 1023.0f, 1023.0f), 0.0f);  // :385
          rgb[3 * (size_t)row] = cmap[3 * ci]; rgb[3 * (size_t)row + 1] = cmap[3 * ci + 1]; rgb[3 * (size_t)row + 2] = cmap[3 * ci + 2];
        }
      }
    }
  }
}

extern "C" int tslam_tsdf_extract_surface(tslam_tsdf_t* m, int32_t submap, int64_t cap, float* xyz, float* rgb, int32_t* count_dev,
                                          void* stream) {
  if (!m || !xyz || !count_dev) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  const float thres = (float)(m->cfg.voxel_scale * 1.8);  // dense_tsdf.py:39
  k_extract_surface<<<m->sm_count * 4, 256, 0, st>>>(m->g, submap, m->cfg.is_global_map, m->pose_R, m->pose_T, m->in.vs, thres,
                                                     (float)m->cfg.disp_floor, (float)m->cfg.disp_ceiling, m->colormap, cap, xyz,
                                                     rgb, count_dev);
  TS_LAUNCH_CHECK(m);
  return ts_check_deferred_async(m, st);
}

static float h16_round(float x) {  // slice_z is an f16 field (dense_tsdf.py:72)
  __half hv = __float2half_rn(x);
  return __half2float(hv);
}

extern "C" int tslam_tsdf_extract_slice(tslam_tsdf_t* m, int32_t submap, float z, float dz, int64_t cap, float* xyz, float* val,
                                        float* rgb, int32_t* count_dev, void* stream) {
  if (!m || !xyz || !count_dev) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  const int index = (int)(h16_round(z) / m->in.vs);  // :369-370
  k_extract_slice<<<m->sm_count * 4, 256, 0, st>>>(m->g, submap, m->cfg.is_global_map, m->pose_R, m->pose_T, m->in.vs, index, dz,
                                                   m->colormap, cap, xyz, val, rgb, count_dev);
  TS_LAUNCH_CHECK(m);
  return ts_check_deferred_async(m, st);
}

// ---------------------------------------------------------------------------
// submap -> global fusion  (dense_tsdf.py:272-318)
// One CTA per SOURCE block; each observed source voxel splats into the 7 upper
// trilinear corners (:297-300) with one 8-byte reduction per corner; commit
// (no Wmax clamp, :274-278) turns the sums into (TSDF, W).
// ---------------------------------------------------------------------------
__device__ __forceinline__ void sat_add_i8(int8_t* p, int add) {
  if (add == 0) return;
  unsigned int* wp = (unsigned int*)((uintptr_t)p & ~(uintptr_t)3);
  const int sh = (int)((uintptr_t)p & 3) * 8;
  unsigned int old = *wp, assumed;
  do {
    assumed = old;
    int cur = (int)(int8_t)((assumed >> sh) & 0xFF);
    int nv = cur + add;
    nv = nv > 127 ? 127 : (nv < -128 ? -128 : nv);  // reference wraps (i8); we saturate (DESIGN.md)
    unsigned int repl = (assumed & ~(0xFFu << sh)) | (((unsigned int)(nv & 0xFF)) << sh);
    old = atomicCAS(wp, assumed, repl);
  } while (old != assumed);
}

__global__ void __launch_bounds__(256) k_fuse(TsGrid dst, TsGrid src, const float* pR, const float* pT, float vs) {
  const int nb = min(*src.n_blocks, src.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(src.block_key[b], s, bx, by, bz);
    if (src.ghost[b]) continue;
    const size_t base = (size_t)b * TS_B3;
    unsigned long long cur_key = TS_EMPTY;
    int cur_blk = -1;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) {
      if (!(src.obs[base + v] > 0)) continue;  // :292
      const float2 t = src.tw[base + v];
      const int occ = src.occ[base + v];
      const bool tex = dst.col != nullptr && src.col != nullptr;
      float4 sc = make_float4(0.f, 0.f, 0.f, 0.f);
      if (tex) sc = src.col[base + v];
      const TsSplatPos p = ts_splat_pos(pR + 9 * s, pT + 3 * s, (float)(bx * TS_B + (v >> 8)) * vs, (float)(by * TS_B + ((v >> 4) & 15)) * vs,
                                        (float)(bz * TS_B + (v & 15)) * vs, vs);
#pragma unroll
      for (int c = 1; c < 8; c++) {  // c=0 (di=dj=dk=0) skipped: reference quirk :300
        int ci, cj, ck;
        float wt;
        if (!ts_splat_corner(dst, p, c, ci, cj, ck, wt)) continue;
        const unsigned long long key = ts_pack_key(0, ci >> TS_BSHIFT, cj >> TS_BSHIFT, ck >> TS_BSHIFT);
        if (key != cur_key) {
          cur_key = key;
          cur_blk = ts_get_or_alloc_cached(dst, key);
          if (cur_blk >= 0) ts_mark_dirty(dst, cur_blk);
        }
        if (cur_blk < 0) continue;
        const size_t o = (size_t)cur_blk * TS_B3 + ts_voxel_off(ci, cj, ck);
        const float w = t.y * wt;                    // :307
        red_add_f32x2(&dst.acc[o], w * t.x, w);      // :274-275
        if (tex) {                                   // :276-277: sum w*c here, / sum w at commit
          float* dc = (float*)&dst.col[o];
          atomicAdd(dc, w * sc.x); atomicAdd(dc + 1, w * sc.y); atomicAdd(dc + 2, w * sc.z);
        }
        if (dst.obs[o] == 0) dst.obs[o] = 2;         // :279 observed, value pending (2 -> 1 at commit)
        sat_add_i8(&dst.occ[o], occ);                // :280
      }
    }
  }
}

extern "C" int tslam_tsdf_fuse(tslam_tsdf_t* dst, tslam_tsdf_t* src, void* stream) {
  int rc = tslam_tsdf_fuse_pending(dst, src, stream);
  if (rc) return rc;
  return ts_launch_commit(dst, (cudaStream_t)stream, 0, 1);
}

// multi-GPU building block (see tslam_dist.cu): fusion that leaves its sums pending, for tslam_tsdf_commit_fused
extern "C" int tslam_tsdf_fuse_pending(tslam_tsdf_t* dst, tslam_tsdf_t* src, void* stream) {
  if (!dst || !src || dst == src) return TSLAM_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(src, st);
  if (rc) return rc;
  dst->n_integrate_calls = 0;  // pending updates of dst are discarded by reset() (:312-313)
  rc = tslam_tsdf_reset(dst, stream);
  if (rc) return rc;
  k_fuse<<<dst->sm_count * 8, 256, 0, st>>>(dst->g, src->g, dst->pose_R, dst->pose_T, dst->in.vs);
  TS_LAUNCH_CHECK(dst);
  return TSLAM_OK;
}

// ---------------------------------------------------------------------------
// stats / sync / profiling
// ---------------------------------------------------------------------------
extern "C" int tslam_tsdf_get_stats(tslam_tsdf_t* m, int64_t* out8, int clear) {
  if (!m || !out8) return TSLAM_E_INVALID;
  TS_CUDA(cudaDeviceSynchronize());
  TsCounters c;
  TS_CUDA(cudaMemcpy(&c, m->counters, sizeof(c), cudaMemcpyDeviceToHost));
  int sc[4];
  TS_CUDA(cudaMemcpy(sc, m->scratch_i, sizeof(sc), cudaMemcpyDeviceToHost));
  out8[0] = (int64_t)c.n_px; out8[1] = (int64_t)c.n_valid; out8[2] = (int64_t)c.n_rays; out8[3] = (int64_t)c.n_updates;
  out8[4] = (int64_t)c.n_oob; out8[5] = sc[0]; out8[6] = sc[2]; out8[7] = m->launches;
  if (clear) TS_CUDA(cudaMemset(m->counters, 0, sizeof(TsCounters)));
  return TSLAM_OK;
}

// the first n <= 7 counters of the binned march
static int ts_march_stats(tslam_tsdf* m, int64_t* out, int n) {
  if (!m || !out) return TSLAM_E_INVALID;
  TS_CUDA(cudaDeviceSynchronize());
  TsCounters c;
  TS_CUDA(cudaMemcpy(&c, m->counters, sizeof(c), cudaMemcpyDeviceToHost));
  const unsigned long long v[7] = {c.n_segs, c.n_items, c.n_slow, c.n_fallback, c.n_generic, c.n_verify_bad, c.n_seg_guard};
  for (int i = 0; i < n; i++) out[i] = (int64_t)v[i];
  return TSLAM_OK;
}
extern "C" int tslam_tsdf_get_march_stats(tslam_tsdf_t* m, int64_t* out6) { return ts_march_stats(m, out6, 6); }
extern "C" int tslam_tsdf_get_march_stats2(tslam_tsdf_t* m, int64_t* out7) { return ts_march_stats(m, out7, 7); }

extern "C" int tslam_tsdf_sync(tslam_tsdf_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  TS_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return ts_check_deferred(m);
}

extern "C" int64_t tslam_tsdf_launch_count(tslam_tsdf_t* m) { return m ? m->launches : 0; }

extern "C" int tslam_tsdf_set_profiling(tslam_tsdf_t* m, int on) {
  if (!m) return TSLAM_E_INVALID;
  if (on && !m->prof) {
    TS_CUDA(cudaMalloc(&m->prof, (size_t)TS_PROF_RING * TS_PROF_WORDS * 8));
    TS_CUDA(cudaMemset(m->prof, 0, (size_t)TS_PROF_RING * TS_PROF_WORDS * 8));
  }
  m->profiling = on;
  m->prof_launches = 0;
  return TSLAM_OK;
}
// ms3[3*i + {0,1,2}] = bucket / ray-march / commit kernel time of the i-th most recent recorded integrate launch,
// i < n (n <= TS_PROF_RING).  Returns the number of rows written in *n_out.
// ms7[7*i + ...] = bucket, ray march (all of its kernels), commit (k_collect_dirty + k_commit_tma; 0 without one), then
// the parts of the ray march: 0 (kept for the ABI: nothing is charged between the bucket kernel and the march),
// set-up + segment count + class + scan, scattering walk, march (with the generic path and the resets).  The last
// three are 0 for textured maps (k_raymarch).
// Times come from the kernels' %globaltimer stamps (TS_PROF_WORDS).  Under programmatic dependent launch a kernel can
// start before its predecessor ends, so one rule charges every column: a stage runs from the LATER of its first kernel's
// start and the end of the stage before it, to its last kernel's end.  The stages of a launch are disjoint intervals:
// the columns never sum to more than the launch's span, and the gaps between stages are charged to none.
// Both write `cols` columns per row (3 or 7), walking the profiling ring backwards from the last recorded launch.
static int ts_kernel_ms(tslam_tsdf* m, int32_t n, int cols, float* ms, int32_t* n_out) {
  if (!m || !ms || !n_out || !m->prof) return TSLAM_E_INVALID;
  TS_CUDA(cudaDeviceSynchronize());
  static_assert(2 * TS_K_N <= TS_PROF_WORDS, "stamp row");
  unsigned long long* ring = new unsigned long long[(size_t)TS_PROF_RING * TS_PROF_WORDS];
  const cudaError_t e = cudaMemcpy(ring, m->prof, (size_t)TS_PROF_RING * TS_PROF_WORDS * 8, cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) { delete[] ring; return ts_cuda_fail(e, "cudaMemcpy(profiling ring)"); }
  long long have = m->prof_launches < TS_PROF_RING ? m->prof_launches : TS_PROF_RING;
  if (n > have) n = (int32_t)have;
  for (int i = 0; i < n; i++) {
    const long long r = (m->prof_launches - 1 - i) % TS_PROF_RING;
    const unsigned long long* s = ring + TS_PROF_WORDS * r;
    const unsigned ran = m->prof_ran[r];
    // stage [first, last] kernel, charged after `prev_end`; returns the stage's end (prev_end when it did not run)
    auto stage = [&](int first, int last, unsigned long long prev_end, float& out) {
      out = 0.0f;
      if (!(ran & (1u << last))) return prev_end;
      const unsigned long long b = std::max(s[2 * first], prev_end), en = s[2 * last + 1];
      out = en > b ? (float)((double)(en - b) * 1e-6) : 0.0f;
      return en;
    };
    float c[7] = {0, 0, 0, 0, 0, 0, 0};
    const unsigned long long e0 = stage(TS_K_BUCKET, TS_K_BUCKET, 0ull, c[0]);
    const bool binned = (ran & (1u << TS_K_COUNT)) != 0;
    const unsigned long long e1 = stage(binned ? TS_K_COUNT : TS_K_MARCH, TS_K_MARCH, e0, c[1]);
    stage(TS_K_COLLECT, TS_K_COMMIT, e1, c[2]);
    if (binned) {
      const unsigned long long e2 = stage(TS_K_COUNT, TS_K_CLASS_SCAN, e0, c[4]);
      const unsigned long long e3 = stage(TS_K_SCATTER, TS_K_SCATTER, e2, c[5]);
      stage(TS_K_MARCH, TS_K_MARCH, e3, c[6]);
    }
    for (int q = 0; q < cols; q++) ms[cols * i + q] = c[q];
  }
  delete[] ring;
  *n_out = n;
  return TSLAM_OK;
}
extern "C" int tslam_tsdf_kernel_ms2(tslam_tsdf_t* m, int32_t n, float* ms7, int32_t* n_out) { return ts_kernel_ms(m, n, 7, ms7, n_out); }
extern "C" int tslam_tsdf_kernel_ms(tslam_tsdf_t* m, int32_t n, float* ms3, int32_t* n_out) { return ts_kernel_ms(m, n, 3, ms3, n_out); }
