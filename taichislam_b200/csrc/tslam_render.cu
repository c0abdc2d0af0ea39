// libtslam.so - rendering of the TSDF's zero level (tslam_tsdf_render, DESIGN.md section 7, "Rendering"): depth, normal
// and colour images of n pinhole cameras, each ray marched at fixed steps of camera-frame depth through the committed
// TSDF of its camera's submap until the interpolated value crosses from positive to non-positive between two valid
// samples.  The value of a sample is the zero level that registration and frame tracking align to (ts_sdf_corners,
// tslam_esdf_common.cuh), so a rendered frame is the surface the tracker sees.
//   k_render  one thread per pixel, CTA = a 16 x 16 tile of one camera (grid: tiles x cameras), each warp an 8 x 4
//             sub-tile, so that the rays of a warp walk the same blocks.  Every sample is the per-sample definition of
//             the header, bit for bit; what is skipped is only what cannot change the result: the hash probe of a block
//             the thread looked up last (memoised), the samples before the ray enters the volume (arithmetic only), and
//             the samples after the first hit or after the ray has left the volume (the volume is a box and the sample
//             points move monotonically along each axis, so a ray that left it does not come back).
// The call reads the committed tw / obs / col planes and writes nothing to the map.
#include <cmath>
#include <vector>
#include "tslam_esdf_common.cuh"

#define RD_TILE 16  // pixels per CTA edge

struct RdJob {        // one camera
  float R[9], T[3];   // its pose, rounded to f32 once
  int submap;
};

struct RdParams {
  const RdJob* jobs;
  float* depth;
  float* normal;      // may be null
  float* color;       // may be null
  uint8_t* status;
  int h, w, tiles_x, K;
  float fx, fy, cx, cy, z_min, step, vs;
};

__global__ void __launch_bounds__(256) k_render(TsGrid g, RdParams p) {
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const int tx = (int)blockIdx.x % p.tiles_x, ty = (int)blockIdx.x / p.tiles_x;
  const int i = tx * RD_TILE + (wp & 1) * 8 + (lane & 7), j = ty * RD_TILE + (wp >> 1) * 4 + (lane >> 3);
  if (i >= p.w || j >= p.h) return;
  const RdJob& jb = p.jobs[blockIdx.y];
  float R[9], T[3];
#pragma unroll
  for (int q = 0; q < 9; q++) R[q] = jb.R[q];
#pragma unroll
  for (int q = 0; q < 3; q++) T[q] = jb.T[q];
  const int sb = jb.submap;
  // ray direction in the submap's local frame: the camera-frame direction (x, y, 1) through pose_apply with T = 0
  const float rx = __fdiv_rn(__fsub_rn((float)i, p.cx), p.fx), ry = __fdiv_rn(__fsub_rn((float)j, p.cy), p.fy);
  const float zero[3] = {0.0f, 0.0f, 0.0f};
  float dir[3];
  pose_apply(R, zero, rx, ry, 1.0f, dir[0], dir[1], dir[2]);
  // the last block looked up: consecutive samples are about a voxel apart, so most need no hash probe
  unsigned long long mkey = ~0ull;
  int mblk = -1;
  const auto find = [&](int bx, int by, int bz) {
    const unsigned long long key = ts_pack_key(sb, bx, by, bz);
    if (key != mkey) { mkey = key; mblk = ts_sdf_block(g, sb, bx, by, bz); }
    return mblk;
  };
  bool entered = false, pv = false, hit = false;
  float pD = 0.0f, pz = 0.0f, D = 0.0f;
  for (int k = 0; k < p.K; k++) {
    const float z = __fadd_rn(p.z_min, __fmul_rn((float)k, p.step));
    const float x[3] = {__fadd_rn(T[0], __fmul_rn(z, dir[0])), __fadd_rn(T[1], __fmul_rn(z, dir[1])), __fadd_rn(T[2], __fmul_rn(z, dir[2]))};
    float u[3];
    int c0[3];
    if (!(esq_low_corner(g, p.vs, x, u, c0) && c0[0] < g.N - g.hN - 1 && c0[1] < g.N - g.hN - 1 && c0[2] < g.Nz - g.hNz - 1)) {
      if (entered) break;  // left the volume: every later sample is outside too
      continue;
    }
    entered = true;
    float e[8];
    const bool v = ts_sdf_corners(g, c0, find, e);
    if (v) D = esq_value(e, __fsub_rn(u[0], (float)c0[0]), __fsub_rn(u[1], (float)c0[1]), __fsub_rn(u[2], (float)c0[2]));
    if (v && pv && pD > 0.0f && D <= 0.0f) { hit = true; break; }
    pv = v;
    pD = D;
    pz = z;
  }
  const size_t o = ((size_t)blockIdx.y * p.h + j) * p.w + i;
  const float qnan = __int_as_float(0x7fc00000);
  // the pixel's outputs; normal and colour are NaN unless status is 1
  const auto put = [&](float zs, uint8_t st, const float* nrm, const float* col) {
    p.depth[o] = zs;
    p.status[o] = st;
    if (p.normal) {
      p.normal[3 * o] = nrm ? nrm[0] : qnan; p.normal[3 * o + 1] = nrm ? nrm[1] : qnan; p.normal[3 * o + 2] = nrm ? nrm[2] : qnan;
    }
    if (p.color) {
      p.color[3 * o] = col ? col[0] : qnan; p.color[3 * o + 1] = col ? col[1] : qnan; p.color[3 * o + 2] = col ? col[2] : qnan;
    }
  };
  if (!hit) { put(0.0f, 0, nullptr, nullptr); return; }
  // samples k (pz, pD) and k + 1 (D)
  const float a = __fsub_rn(pD, D), f = __fdiv_rn(pD, a);
  const float zs = __fadd_rn(pz, __fmul_rn(p.step, f));
  const float x[3] = {__fadd_rn(T[0], __fmul_rn(zs, dir[0])), __fadd_rn(T[1], __fmul_rn(zs, dir[1])), __fadd_rn(T[2], __fmul_rn(zs, dir[2]))};
  float u[3], e[8];
  int c0[3];
  size_t off[8];
  if (!(esq_low_corner(g, p.vs, x, u, c0) && c0[0] < g.N - g.hN - 1 && c0[1] < g.N - g.hN - 1 && c0[2] < g.Nz - g.hNz - 1) ||
      !ts_sdf_corners(g, c0, find, e, [&](int c, size_t q) { off[c] = q; })) {
    put(zs, 2, nullptr, nullptr);
    return;
  }
  const float fx = __fsub_rn(u[0], (float)c0[0]), fy = __fsub_rn(u[1], (float)c0[1]), fz = __fsub_rn(u[2], (float)c0[2]);
  float d, gx, gy, gz;
  esq_interp(e, fx, fy, fz, p.vs, d, gx, gy, gz);
  const float gn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz)));
  if (!(gn > 0.0f)) { put(zs, 2, nullptr, nullptr); return; }
  const float nrm[3] = {__fdiv_rn(gx, gn), __fdiv_rn(gy, gn), __fdiv_rn(gz, gn)};
  float col[3];
  if (p.color) {
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
      float ec[8];
#pragma unroll
      for (int c = 0; c < 8; c++) ec[c] = ((const float*)&g.col[off[c]])[ch];
      col[ch] = esq_value(ec, fx, fy, fz);
    }
  }
  put(zs, 1, nrm, col);
}

extern "C" int tslam_tsdf_render(tslam_tsdf_t* m, int32_t n, int32_t height, int32_t width, const double* K4, const int32_t* submaps,
                                 const double* R, const double* T, float z_min, float z_max, float step, float* depth, float* normal,
                                 float* color, uint8_t* status, void* stream) {
  static const char* fn = "tslam_tsdf_render";
  if (n < 1 || n > TSLAM_RENDER_MAX_CAMERAS) {
    ts_set_error("%s: n %d outside [1, %d]", fn, n, TSLAM_RENDER_MAX_CAMERAS);
    return TSLAM_E_INVALID;
  }
  if (height < 1 || width < 1 || (long long)n * height * width >= (1ll << 31)) {
    ts_set_error("%s: height and width must be >= 1 and n h w < 2^31", fn);
    return TSLAM_E_INVALID;
  }
  if (!K4 || !depth || !status) {
    ts_set_error("%s: NULL K4, depth or status", fn);
    return TSLAM_E_INVALID;
  }
  const float fx = (float)K4[0], fy = (float)K4[1], cx = (float)K4[2], cy = (float)K4[3];
  if (!std::isfinite(fx) || !(fx > 0.0f) || !std::isfinite(fy) || !(fy > 0.0f) || !std::isfinite(cx) || !std::isfinite(cy)) {
    ts_set_error("%s: fx, fy must be finite and > 0, cx, cy finite", fn);
    return TSLAM_E_INVALID;
  }
  if (!std::isfinite(z_min) || !(z_min > 0.0f) || !std::isfinite(z_max) || !(z_max > z_min) || !std::isfinite(step) || !(step > 0.0f)) {
    ts_set_error("%s: z_min finite and > 0, z_max finite and > z_min, step finite and > 0", fn);
    return TSLAM_E_INVALID;
  }
  const double Kd = std::floor(((double)z_max - (double)z_min) / (double)step) + 1.0;
  if (Kd > (double)TSLAM_RENDER_MAX_SAMPLES) {
    ts_set_error("%s: %.0f samples per ray > %d", fn, Kd, TSLAM_RENDER_MAX_SAMPLES);
    return TSLAM_E_INVALID;
  }
  if (!m || !R || !T) {
    ts_set_error("%s: NULL handle or pose array", fn);
    return TSLAM_E_INVALID;
  }
  std::vector<RdJob> jobs(n);
  for (int c = 0; c < n; c++) {
    const int s = submaps ? submaps[c] : 0;
    if (s < 0 || s >= m->cfg.max_submaps) {
      ts_set_error("%s: camera %d: submap %d out of range", fn, c, s);
      return TSLAM_E_INVALID;
    }
    RdJob& jb = jobs[c];
    jb.submap = s;
    bool fin = true;
    for (int q = 0; q < 9; q++) { jb.R[q] = (float)R[9 * c + q]; fin &= std::isfinite(R[9 * c + q]) && std::isfinite(jb.R[q]); }
    for (int q = 0; q < 3; q++) { jb.T[q] = (float)T[3 * c + q]; fin &= std::isfinite(T[3 * c + q]) && std::isfinite(jb.T[q]); }
    if (!fin) {
      ts_set_error("%s: camera %d: pose not finite", fn, c);
      return TSLAM_E_INVALID;
    }
  }
  if (color && !m->cfg.texture_enabled) {
    ts_set_error("%s: colour requested on a map without texture", fn);
    return TSLAM_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(m, st);
  if (rc) return rc;
  rc = rg_reserve(&m->render_jobs, &m->render_jobs_bytes, (size_t)n * sizeof(RdJob));
  if (rc) return rc;
  TS_CUDA(cudaMemcpyAsync(m->render_jobs, jobs.data(), (size_t)n * sizeof(RdJob), cudaMemcpyHostToDevice, st));
  RdParams p;
  p.jobs = (const RdJob*)m->render_jobs;
  p.depth = depth;
  p.normal = normal;
  p.color = color;
  p.status = status;
  p.h = height;
  p.w = width;
  p.tiles_x = (width + RD_TILE - 1) / RD_TILE;
  p.K = (int)Kd;
  p.fx = fx; p.fy = fy; p.cx = cx; p.cy = cy;
  p.z_min = z_min;
  p.step = step;
  p.vs = m->in.vs;
  const dim3 grid((unsigned)(p.tiles_x * ((height + RD_TILE - 1) / RD_TILE)), (unsigned)n);
  k_render<<<grid, 256, 0, st>>>(m->g, p);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}
