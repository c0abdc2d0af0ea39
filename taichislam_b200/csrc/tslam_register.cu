// libtslam.so - SDF-to-SDF registration of TSDF submap pairs (tslam_tsdf_register, DESIGN.md section 7, "Submap
// registration"), the pair term of Voxgraph (Reijgwart et al., 2019): the near-surface voxels of a submap of the reference
// map A are looked up in a submap of the reading map B, and Levenberg-Marquardt on the host (f64) solves for the relative
// pose that makes the two signed distances agree.  The normal equations at the final pose are the information a pose-graph
// optimiser consumes.
//   selection   once per call.  Per pool block of A, the registration points of every requested reference submap are
//               counted (k_rg_count); CUB sorts the blocks stably by the submap's slot and scans their counts; k_rg_fill
//               writes (p_v, d_v) records.  A submap's points are therefore contiguous, in pool order, and in voxel order
//               inside a block, whatever else the call asks for: pairs that share a reference submap share its range.
//   evaluation  one k_rg_eval launch per LM iteration over every active pair: one CTA per chunk of RG_CHUNK points of one
//               pair, RG_PPT passes of one point per thread (transform, corner lookup, trilinear interpolant and its
//               gradient, residual, Huber weight, 29 f64 terms), a warp-shuffle and shared-memory reduction to one partial
//               per chunk; then k_rg_final sums the chunk partials of each pair in chunk order.  The host reads P x 29
//               doubles, the iteration's one synchronisation.  Every sum is over a fixed order that depends on the pair
//               alone, so a pair's result is the same bits alone or in a batch, and two identical calls agree bit for bit.
// The call reads the committed tw / obs planes and writes nothing to either map.
// Frame tracking (tslam_tsdf_track_depth / _points, DESIGN.md section 7, "Frame tracking") is the same solver (rg_lm)
// over other records: the kept points of depth frames or a point cloud in the sensor frame, with d = 0, selected by
// k_tr_select (count, scan, fill).
#include <cub/cub.cuh>
#include <cmath>
#include <cstring>
#include <vector>
#include "tslam_esdf_common.cuh"

#define RG_THREADS 256
#define RG_PPT 4                           // points per thread and chunk
#define RG_CHUNK (RG_THREADS * RG_PPT)     // points per CTA
#define RG_NS 29                           // sums per pair: H (21, upper triangle row by row), b (6), cost, n_valid

struct RgJob {        // one pair of an evaluation launch
  float R[9], t[3];   // its pose, rounded to f32
  long long p0;       // first point record of its reference submap
  int n;              // points of that submap
  int submap;         // reading submap of B
  int pair;           // row of the sums
  int cta0;           // first CTA of the pair in the launch
};

// registration point: observed, W > 0, W >= min_weight, |TSDF| <= band (a NaN TSDF fails the band test)
__device__ __forceinline__ bool rg_point(const TsGrid& g, size_t off, float band, float min_w) {
  if (!g.obs[off]) return false;
  const float2 t = g.tw[off];
  return t.y > 0.0f && t.y >= min_w && fabsf(t.x) <= band;
}

// per pool block of A: cnt = registration points when the block is a non-ghost block of a requested submap (key = its
// slot), else 0 (key = n_slots, sorted last); slot_cnt[slot] += cnt
__global__ void __launch_bounds__(256) k_rg_count(TsGrid g, int nb, const int* __restrict__ slot_of, int n_slots, float band,
                                                  float min_w, int* cnt, int* key, int* val, int* slot_cnt) {
  __shared__ int s_n;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    const int sl = g.ghost[b] ? -1 : slot_of[s];
    if (sl < 0) {  // (uniform per CTA)
      if (threadIdx.x == 0) { cnt[b] = 0; key[b] = n_slots; val[b] = b; }
      continue;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const size_t base = (size_t)b * TS_B3;
    int mine = 0;
    for (int v = threadIdx.x; v < TS_B3; v += blockDim.x) mine += rg_point(g, base + v, band, min_w) ? 1 : 0;
    es_cta_add(mine, &s_n);
    __syncthreads();
    if (threadIdx.x == 0) {
      cnt[b] = s_n; key[b] = sl; val[b] = b;
      if (s_n) atomicAdd(&slot_cnt[sl], s_n);
    }
  }
}

// counts in sorted block order (the scan's input); cs[nb] = 0 so that the exclusive scan's last entry is the total
__global__ void __launch_bounds__(256) k_rg_permute(int nb, const int* __restrict__ cnt, const int* __restrict__ order, int* cs) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= nb; i += gridDim.x * blockDim.x) cs[i] = i < nb ? cnt[order[i]] : 0;
}

// One CTA per sorted block with points: thread t takes voxels 16t .. 16t + 15, a block scan places them, so the records of
// a block lie in voxel order.  Record = (f32(i) vs, f32(j) vs, f32(k) vs, TSDF) (ijk_to_xyz, mapping_common.py:221-223).
__global__ void __launch_bounds__(256) k_rg_fill(TsGrid g, int nb, const int* __restrict__ order, const int* __restrict__ cs,
                                                 const int* __restrict__ off, float band, float min_w, float vs, float4* pts) {
  typedef cub::BlockScan<int, 256> Scan;
  __shared__ typename Scan::TempStorage tmp;
  for (int i = blockIdx.x; i < nb; i += gridDim.x) {
    if (cs[i] == 0) continue;  // (uniform per CTA)
    const int b = order[i];
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    const size_t base = (size_t)b * TS_B3;
    unsigned keep = 0;
    for (int q = 0; q < 16; q++) keep |= rg_point(g, base + threadIdx.x * 16 + q, band, min_w) ? 1u << q : 0u;
    int pos;
    __syncthreads();
    Scan(tmp).ExclusiveSum(__popc(keep), pos);
    long long row = (long long)off[i] + pos;
    for (int q = 0; q < 16; q++) {
      if (!(keep >> q & 1u)) continue;
      const int v = threadIdx.x * 16 + q;
      const float x = (float)(bx * TS_B + (v >> 8)) * vs, y = (float)(by * TS_B + ((v >> 4) & 15)) * vs, z = (float)(bz * TS_B + (v & 15)) * vs;
      pts[row++] = make_float4(x, y, z, g.tw[base + v].x);
    }
  }
}

// The 29 terms of one point p = (p_v, d_v) at pose (R, t) against submap sb of the reading grid g, added to s; nothing
// when a corner is invalid (outside the volume; absent or ghost block; unobserved or W = 0)
__device__ __forceinline__ void rg_term(const TsGrid& g, int sb, float4 p, const float* R, const float* t, float vs, double delta,
                                        double s[RG_NS]) {
  float x[3];
  pose_apply(R, t, p.x, p.y, p.z, x[0], x[1], x[2]);
  float u[3];
  int c0[3];
  if (!(esq_low_corner(g, vs, x, u, c0) && c0[0] < g.N - g.hN - 1 && c0[1] < g.N - g.hN - 1 && c0[2] < g.Nz - g.hNz - 1)) return;
  float e[8];
  if (!ts_sdf_corners(g, c0, [&](int bx, int by, int bz) { return ts_sdf_block(g, sb, bx, by, bz); }, e)) return;
  const float fx = __fsub_rn(u[0], (float)c0[0]), fy = __fsub_rn(u[1], (float)c0[1]), fz = __fsub_rn(u[2], (float)c0[2]);
  float d, gx, gy, gz;
  esq_interp(e, fx, fy, fz, vs, d, gx, gy, gz);
  const double r = (double)__fsub_rn(d, p.w), ar = fabs(r);
  const double w = ar <= delta ? 1.0 : delta / ar;
  const double rho = ar <= delta ? 0.5 * r * r : delta * (ar - 0.5 * delta);
  const double X = x[0], Y = x[1], Z = x[2], Gx = gx, Gy = gy, Gz = gz;
  const double J[6] = {Gx, Gy, Gz, Y * Gz - Z * Gy, Z * Gx - X * Gz, X * Gy - Y * Gx};  // [g, x cross g]
  int q = 0;
#pragma unroll
  for (int i = 0; i < 6; i++) {
    const double wj = w * J[i];
#pragma unroll
    for (int j = i; j < 6; j++) s[q++] += wj * J[j];
  }
#pragma unroll
  for (int i = 0; i < 6; i++) s[21 + i] += (w * J[i]) * r;
  s[27] += rho;
  s[28] += 1.0;
}

__global__ void __launch_bounds__(RG_THREADS) k_rg_eval(TsGrid g, const float4* __restrict__ pts, const RgJob* __restrict__ jobs,
                                                        int n_jobs, float vs, double delta, double* __restrict__ part) {
  __shared__ double sh[RG_THREADS / 32][RG_NS];
  int lo = 0, hi = n_jobs - 1;  // the job of this CTA: the last with cta0 <= blockIdx.x
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].cta0 <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const RgJob& jb = jobs[lo];
  float R[9], t[3];
#pragma unroll
  for (int i = 0; i < 9; i++) R[i] = jb.R[i];
#pragma unroll
  for (int i = 0; i < 3; i++) t[i] = jb.t[i];
  const int c = (int)blockIdx.x - jb.cta0, n = jb.n, sb = jb.submap;
  const float4* p = pts + jb.p0;
  double s[RG_NS];
#pragma unroll
  for (int q = 0; q < RG_NS; q++) s[q] = 0.0;
  for (int k = 0; k < RG_PPT; k++) {
    const int i = c * RG_CHUNK + k * RG_THREADS + threadIdx.x;
    if (i >= n) break;
    rg_term(g, sb, p[i], R, t, vs, delta, s);
  }
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < RG_NS; q++) {
    double v = s[q];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sh[wp][q] = v;
  }
  __syncthreads();
  if (threadIdx.x < RG_NS) {
    double v = 0.0;
    for (int w = 0; w < RG_THREADS / 32; w++) v += sh[w][threadIdx.x];
    part[(size_t)blockIdx.x * RG_NS + threadIdx.x] = v;
  }
}

// one warp per job: its chunk partials summed lane-strided in chunk order, then a shuffle tree
__global__ void __launch_bounds__(256) k_rg_final(const RgJob* __restrict__ jobs, int n_jobs, int n_ctas, const double* __restrict__ part,
                                                  double* __restrict__ sums) {
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (j >= n_jobs) return;  // (uniform per warp)
  const int c0 = jobs[j].cta0, c1 = j + 1 < n_jobs ? jobs[j + 1].cta0 : n_ctas, row = jobs[j].pair;
  for (int q = 0; q < RG_NS; q++) {
    double v = 0.0;
    for (int c = c0 + lane; c < c1; c += 32) v += part[(size_t)c * RG_NS + q];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sums[(size_t)row * RG_NS + q] = v;
  }
}

// ---- host --------------------------------------------------------------------------------------------------------
// *p holds at least `need` bytes: reallocated (contents dropped) to max(need, 2 x the old size) when smaller
int rg_reserve(void** p, size_t* bytes, size_t need) {
  if (need <= *bytes) return TSLAM_OK;
  const size_t nb = need > 2 * *bytes ? need : 2 * *bytes;
  if (*p) cudaFree(*p);
  *p = nullptr;
  *bytes = 0;
  TS_CUDA(cudaMalloc(p, nb));
  *bytes = nb;
  return TSLAM_OK;
}
static size_t rg_align(size_t x) { return (x + 255) & ~(size_t)255; }

// f64 pose of a pair: R row-major, t
struct RgPose { double R[9], t[3]; };

// exp(xi) * T for xi = (rho, phi): R' = Exp(phi) R, t' = Exp(phi) t + V(phi) rho (SE(3) exponential, left perturbation)
static RgPose rg_update(const RgPose& T, const double xi[6]) {
  const double* rho = xi;
  const double* phi = xi + 3;
  const double th2 = phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2], th = std::sqrt(th2);
  double A, Bc, Cc;  // sin(th)/th, (1 - cos th)/th^2, (th - sin th)/th^3
  if (th < 1e-4) {
    A = 1.0 - th2 / 6.0; Bc = 0.5 - th2 / 24.0; Cc = 1.0 / 6.0 - th2 / 120.0;
  } else {
    A = std::sin(th) / th; Bc = (1.0 - std::cos(th)) / th2; Cc = (th - std::sin(th)) / (th2 * th);
  }
  const double K[9] = {0.0, -phi[2], phi[1], phi[2], 0.0, -phi[0], -phi[1], phi[0], 0.0};
  double K2[9], E[9], V[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) K2[3 * i + j] = K[3 * i] * K[j] + K[3 * i + 1] * K[3 + j] + K[3 * i + 2] * K[6 + j];
  for (int i = 0; i < 9; i++) {
    const double I = (i % 4 == 0) ? 1.0 : 0.0;
    E[i] = I + A * K[i] + Bc * K2[i];
    V[i] = I + Bc * K[i] + Cc * K2[i];
  }
  RgPose o;
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 3; j++) o.R[3 * i + j] = E[3 * i] * T.R[j] + E[3 * i + 1] * T.R[3 + j] + E[3 * i + 2] * T.R[6 + j];
    o.t[i] = (E[3 * i] * T.t[0] + E[3 * i + 1] * T.t[1] + E[3 * i + 2] * T.t[2]) + (V[3 * i] * rho[0] + V[3 * i + 1] * rho[1] + V[3 * i + 2] * rho[2]);
  }
  return o;
}

// Solve (H + lam diag(max(H_ii, 1e-9 max_j H_jj))) xi = -b by Cholesky; false when the matrix is not positive definite
static bool rg_solve(const double* S, double lam, double xi[6]) {
  double H[36], L[36] = {0};
  int q = 0;
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++) H[6 * i + j] = H[6 * j + i] = S[q++];
  double hmax = 0.0;
  for (int i = 0; i < 6; i++) hmax = std::fmax(hmax, H[7 * i]);
  for (int i = 0; i < 6; i++) H[7 * i] += lam * std::fmax(H[7 * i], 1e-9 * hmax);
  for (int j = 0; j < 6; j++) {
    double d = H[7 * j];
    for (int k = 0; k < j; k++) d -= L[6 * j + k] * L[6 * j + k];
    if (!(d > 0.0)) return false;
    L[7 * j] = std::sqrt(d);
    for (int i = j + 1; i < 6; i++) {
      double v = H[6 * i + j];
      for (int k = 0; k < j; k++) v -= L[6 * i + k] * L[6 * j + k];
      L[6 * i + j] = v / L[7 * j];
    }
  }
  double y[6];
  for (int i = 0; i < 6; i++) {
    double v = -S[21 + i];
    for (int k = 0; k < i; k++) v -= L[6 * i + k] * y[k];
    y[i] = v / L[7 * i];
  }
  for (int i = 5; i >= 0; i--) {
    double v = y[i];
    for (int k = i + 1; k < 6; k++) v -= L[6 * k + i] * xi[k];
    xi[i] = v / L[7 * i];
  }
  return true;
}

static double rg_mean_cost(const double* S) { return S[28] > 0.0 ? S[27] / S[28] : INFINITY; }

// Chunks (CTAs of one evaluation) of P problems of n[p] points
static long long rg_lm_ctas(int P, const int* n) {
  long long c = 0;
  for (int p = 0; p < P; p++) c += (n[p] + RG_CHUNK - 1) / RG_CHUNK;
  return c;
}
// Device scratch of rg_lm: chunk partials, jobs, sums
static size_t rg_lm_bytes(int P, long long ctas) {
  return rg_align((size_t)(ctas + 1) * RG_NS * 8) + rg_align((size_t)P * sizeof(RgJob)) + rg_align((size_t)P * RG_NS * 8);
}

// Levenberg-Marquardt of P problems, all active problems evaluated by one launch per iteration: problem p solves for the
// pose of the records pts[p0[p] .. p0[p] + n[p]) against submap sub[p] of the grid g, from (R0, T0) row p.  The launches
// count on A.  scratch: rg_lm_bytes(P, rg_lm_ctas(P, n)) bytes of device memory.  Writes the outputs of
// tslam_tsdf_register (include/tslam.h), info5[5p] = n[p].
static int rg_lm(tslam_tsdf_t* A, const TsGrid& g, const float4* pts, void* scratch, int P, const long long* p0, const int* n,
                 const int* sub, const double* R0, const double* T0, float vs, float huber, int max_iters, int min_points,
                 double* R_out, double* T_out, double* H_out, double* b_out, double* cost2, int64_t* info5, cudaStream_t st) {
  char* w = (char*)scratch;
  double* part = (double*)w; w += rg_align((size_t)(rg_lm_ctas(P, n) + 1) * RG_NS * 8);
  RgJob* d_jobs = (RgJob*)w; w += rg_align((size_t)P * sizeof(RgJob));
  double* d_sums = (double*)w;
  std::vector<RgPose> T(P), trial(P);
  std::vector<double> S((size_t)P * RG_NS), Sn((size_t)P * RG_NS), lam(P, 1e-4);
  std::vector<int> iters(P, 0), conv(P, 0), status(P, 0);
  std::vector<char> active(P, 0);
  std::vector<RgJob> jobs;
  jobs.reserve(P);
  const double delta = (double)huber;
  // evaluate the poses Q[p] of the listed problems into out
  auto evaluate = [&](const std::vector<int>& list, const std::vector<RgPose>& Q, std::vector<double>& out) -> int {
    jobs.clear();
    int ctas = 0;
    for (int p : list) {
      RgJob j;
      for (int i = 0; i < 9; i++) j.R[i] = (float)Q[p].R[i];
      for (int i = 0; i < 3; i++) j.t[i] = (float)Q[p].t[i];
      j.p0 = p0[p];
      j.n = n[p];
      j.submap = sub[p];
      j.pair = p;
      j.cta0 = ctas;
      ctas += (j.n + RG_CHUNK - 1) / RG_CHUNK;
      jobs.push_back(j);
    }
    TS_CUDA(cudaMemsetAsync(d_sums, 0, (size_t)P * RG_NS * 8, st));
    TS_CUDA(cudaMemcpyAsync(d_jobs, jobs.data(), jobs.size() * sizeof(RgJob), cudaMemcpyHostToDevice, st));
    if (ctas > 0) {
      k_rg_eval<<<ctas, RG_THREADS, 0, st>>>(g, pts, d_jobs, (int)jobs.size(), vs, delta, part);
      TS_LAUNCH_CHECK(A);
      k_rg_final<<<((int)jobs.size() * 32 + 255) / 256, 256, 0, st>>>(d_jobs, (int)jobs.size(), ctas, part, d_sums);
      TS_LAUNCH_CHECK(A);
    }
    TS_CUDA(cudaMemcpyAsync(out.data(), d_sums, (size_t)P * RG_NS * 8, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
    return TSLAM_OK;
  };
  std::vector<int> list;
  for (int p = 0; p < P; p++) {
    for (int i = 0; i < 9; i++) T[p].R[i] = R0[9 * p + i];
    for (int i = 0; i < 3; i++) T[p].t[i] = T0[3 * p + i];
    list.push_back(p);
  }
  int rc = evaluate(list, T, S);
  if (rc) return rc;
  std::vector<double> cost0(P);
  for (int p = 0; p < P; p++) {
    const double* s = &S[(size_t)p * RG_NS];
    cost0[p] = s[27];
    if (s[28] < (double)min_points) status[p] = 1;
    active[p] = status[p] == 0 && max_iters > 0;
  }
  const double rho_tol = 1e-4 * (double)vs, phi_tol = 1e-6;
  for (;;) {
    list.clear();
    for (int p = 0; p < P; p++) {
      if (!active[p]) continue;
      double xi[6];
      if (!rg_solve(&S[(size_t)p * RG_NS], lam[p], xi)) { active[p] = 0; continue; }  // H + lam D singular: stop here
      const double nr = std::sqrt(xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2]);
      const double nf = std::sqrt(xi[3] * xi[3] + xi[4] * xi[4] + xi[5] * xi[5]);
      if (nr < rho_tol && nf < phi_tol) { conv[p] = 1; active[p] = 0; continue; }
      trial[p] = rg_update(T[p], xi);
      list.push_back(p);
    }
    if (list.empty()) break;
    rc = evaluate(list, trial, Sn);
    if (rc) return rc;
    for (int p : list) {
      const double* sn = &Sn[(size_t)p * RG_NS];
      double* s = &S[(size_t)p * RG_NS];
      iters[p]++;
      if (sn[28] >= (double)min_points && rg_mean_cost(sn) < rg_mean_cost(s)) {
        T[p] = trial[p];
        std::memcpy(s, sn, RG_NS * 8);
        lam[p] /= 10.0;
      } else {
        lam[p] *= 10.0;
      }
      if (iters[p] >= max_iters) active[p] = 0;
    }
  }
  for (int p = 0; p < P; p++) {
    const double* s = &S[(size_t)p * RG_NS];
    std::memcpy(R_out + 9 * p, T[p].R, 9 * 8);
    std::memcpy(T_out + 3 * p, T[p].t, 3 * 8);
    int q = 0;
    for (int i = 0; i < 6; i++)
      for (int j = i; j < 6; j++) H_out[36 * p + 6 * i + j] = H_out[36 * p + 6 * j + i] = s[q++];
    for (int i = 0; i < 6; i++) b_out[6 * p + i] = s[21 + i];
    cost2[2 * p] = cost0[p];
    cost2[2 * p + 1] = s[27];
    info5[5 * p] = n[p];
    info5[5 * p + 1] = (int64_t)s[28];
    info5[5 * p + 2] = iters[p];
    info5[5 * p + 3] = conv[p];
    info5[5 * p + 4] = status[p];
  }
  return TSLAM_OK;
}

// Point selection (shared by tslam_tsdf_register and tslam_tsdf_place_describe): the registration points of the submaps
// s with slot_of[s] >= 0 (slots 0 .. U-1), in slot order, then pool order, then voxel order.  rg_select_count counts them
// per block and per slot (k_rg_count), sorts the blocks by slot and scans their counts, and returns the per-slot counts
// (synchronises); the block arrays live in A->reg_blk.  rg_select_fill writes the records (k_rg_fill) to pts, which
// holds at least the total.
int rg_select_count(tslam_tsdf_t* A, const std::vector<int>& slot_of, int U, float band, float min_weight, RgSel& sel,
                    std::vector<int>& slot_cnt, cudaStream_t st) {
  const int ms = (int)slot_of.size();
  int nb = 0;
  TS_CUDA(cudaMemcpyAsync(&nb, A->g.n_blocks, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (nb > A->g.max_blocks) nb = A->g.max_blocks;
  int end_bit = 1;
  while ((1 << end_bit) <= U) end_bit++;
  size_t sort_tmp = 0, scan_tmp = 0;
  TS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (int*)nullptr, (int*)nullptr, (int*)nullptr, (int*)nullptr, nb, 0, end_bit, st));
  TS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (int*)nullptr, (int*)nullptr, nb + 1, st));
  const size_t nbs = rg_align((size_t)(nb + 1) * 4), mss = rg_align((size_t)ms * 4);
  const size_t tmp_bytes = rg_align(sort_tmp > scan_tmp ? sort_tmp : scan_tmp);
  int rc = rg_reserve(&A->reg_blk, &A->reg_blk_bytes, 7 * nbs + 2 * mss + tmp_bytes);
  if (rc) return rc;
  char* w = (char*)A->reg_blk;
  int* cnt = (int*)w; w += nbs;
  int* key = (int*)w; w += nbs;
  int* val = (int*)w; w += nbs;
  int* key_s = (int*)w; w += nbs;
  int* val_s = (int*)w; w += nbs;
  int* cs = (int*)w; w += nbs;
  int* off = (int*)w; w += nbs;
  int* d_slot_of = (int*)w; w += mss;
  int* d_slot_cnt = (int*)w; w += mss;
  void* tmp = w;
  TS_CUDA(cudaMemcpyAsync(d_slot_of, slot_of.data(), (size_t)ms * 4, cudaMemcpyHostToDevice, st));
  TS_CUDA(cudaMemsetAsync(d_slot_cnt, 0, (size_t)U * 4, st));
  slot_cnt.assign(U, 0);
  if (nb > 0) {
    const float bw = band, mw = min_weight;
    k_rg_count<<<A->sm_count * 4, 256, 0, st>>>(A->g, nb, d_slot_of, U, bw, mw, cnt, key, val, d_slot_cnt);
    TS_LAUNCH_CHECK(A);
    TS_CUDA(cub::DeviceRadixSort::SortPairs(tmp, sort_tmp, key, key_s, val, val_s, nb, 0, end_bit, st));
    k_rg_permute<<<oc_grid(nb + 1, 256, A->sm_count * 8), 256, 0, st>>>(nb, cnt, val_s, cs);
    TS_LAUNCH_CHECK(A);
    TS_CUDA(cub::DeviceScan::ExclusiveSum(tmp, scan_tmp, cs, off, nb + 1, st));
    TS_CUDA(cudaMemcpyAsync(slot_cnt.data(), d_slot_cnt, (size_t)U * 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
  }
  sel.nb = nb;
  sel.order = val_s;
  sel.cs = cs;
  sel.off = off;
  return TSLAM_OK;
}

int rg_select_fill(tslam_tsdf_t* A, const RgSel& sel, float band, float min_weight, float4* pts, cudaStream_t st) {
  k_rg_fill<<<A->sm_count * 4, 256, 0, st>>>(A->g, sel.nb, sel.order, sel.cs, sel.off, band, min_weight, A->in.vs, pts);
  TS_LAUNCH_CHECK(A);
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_register(tslam_tsdf_t* A, tslam_tsdf_t* B, int32_t n_pairs, const int32_t* ref_submaps,
                                   const int32_t* read_submaps, const double* R0, const double* T0, float band, float min_weight,
                                   float huber, int32_t max_iters, int32_t min_points, double* R_out, double* T_out, double* H_out,
                                   double* b_out, double* cost2, int64_t* info5, void* stream) {
  if (n_pairs < 1 || n_pairs > TSLAM_REG_MAX_PAIRS) {
    ts_set_error("tslam_tsdf_register: n_pairs %d outside [1, %d]", n_pairs, TSLAM_REG_MAX_PAIRS);
    return TSLAM_E_INVALID;
  }
  if (!std::isfinite(band) || !(band > 0.0f) || !std::isfinite(huber) || !(huber > 0.0f) || !std::isfinite(min_weight) ||
      max_iters < 0 || min_points < 0) {
    ts_set_error("tslam_tsdf_register: band and huber must be finite and > 0, min_weight finite, max_iters and min_points >= 0");
    return TSLAM_E_INVALID;
  }
  if (!A || !B || !ref_submaps || !read_submaps || !R0 || !T0 || !R_out || !T_out || !H_out || !b_out || !cost2 || !info5) {
    ts_set_error("tslam_tsdf_register: NULL handle or array");
    return TSLAM_E_INVALID;
  }
  if (std::memcmp(&A->in.vs, &B->in.vs, sizeof(float)) != 0) {
    ts_set_error("tslam_tsdf_register: the maps' voxel scales differ (%.9g vs %.9g)", (double)A->in.vs, (double)B->in.vs);
    return TSLAM_E_INVALID;
  }
  for (int p = 0; p < n_pairs; p++) {
    if (ref_submaps[p] < 0 || ref_submaps[p] >= A->cfg.max_submaps || read_submaps[p] < 0 || read_submaps[p] >= B->cfg.max_submaps) {
      ts_set_error("tslam_tsdf_register: pair %d: submap (%d, %d) out of range", p, ref_submaps[p], read_submaps[p]);
      return TSLAM_E_INVALID;
    }
    for (int i = 0; i < 12; i++) {
      if (!std::isfinite(i < 9 ? R0[9 * p + i] : T0[3 * p + i - 9])) {
        ts_set_error("tslam_tsdf_register: pair %d: initial pose not finite", p);
        return TSLAM_E_INVALID;
      }
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ts_flush_pending(A, st);
  if (!rc && B != A) rc = ts_flush_pending(B, st);
  if (!rc) rc = ts_check_deferred_async(A, st);
  if (!rc && B != A) rc = ts_check_deferred_async(B, st);
  if (rc) return rc;
  const float vs = A->in.vs;

  // ---- point selection: one slot per distinct reference submap, in order of first appearance
  const int ms = 1024;  // every submap a block key can name
  std::vector<int> slot_of(ms, -1), pair_slot(n_pairs), slot_sub;
  for (int p = 0; p < n_pairs; p++) {
    int& sl = slot_of[ref_submaps[p]];
    if (sl < 0) { sl = (int)slot_sub.size(); slot_sub.push_back(ref_submaps[p]); }
    pair_slot[p] = sl;
  }
  const int U = (int)slot_sub.size();
  RgSel sel;
  std::vector<int> slot_cnt;
  rc = rg_select_count(A, slot_of, U, band, min_weight, sel, slot_cnt, st);
  if (rc) return rc;
  std::vector<long long> slot_p0(U + 1, 0);
  for (int u = 0; u < U; u++) slot_p0[u + 1] = slot_p0[u] + slot_cnt[u];
  const long long n_pts = slot_p0[U];
  std::vector<long long> p0(n_pairs);
  std::vector<int> np(n_pairs);
  for (int p = 0; p < n_pairs; p++) { p0[p] = slot_p0[pair_slot[p]]; np[p] = slot_cnt[pair_slot[p]]; }
  const long long max_ctas = rg_lm_ctas(n_pairs, np.data());  // a launch covers at most every pair
  if (max_ctas > INT32_MAX / 2) { ts_set_error("tslam_tsdf_register: too many points (%lld)", n_pts); return TSLAM_E_CAPACITY; }
  const size_t pts_b = rg_align((size_t)n_pts * 16);
  rc = rg_reserve(&A->reg_pts, &A->reg_pts_bytes, pts_b + rg_lm_bytes(n_pairs, max_ctas));
  if (rc) return rc;
  float4* pts = (float4*)A->reg_pts;
  if (n_pts > 0) {
    rc = rg_select_fill(A, sel, band, min_weight, pts, st);
    if (rc) return rc;
  }
  return rg_lm(A, B->g, pts, (char*)A->reg_pts + pts_b, n_pairs, p0.data(), np.data(), read_submaps, R0, T0, vs, huber, max_iters,
               min_points, R_out, T_out, H_out, b_out, cost2, info5, st);
}

// ---- frame tracking (tslam_tsdf_track_depth / tslam_tsdf_track_points, DESIGN.md section 7, "Frame tracking") --------
// The records of a frame are its kept points (x, y, z, 0) in the sensor frame, aligned with rg_lm against d = 0: the
// pose that puts them on the zero level of the map's TSDF.  Selection is a count, a scan and a fill over chunks of
// TR_CHUNK consecutive candidates of one frame (CTA (chunk, frame)), so that a frame's records are contiguous and in
// candidate order whatever else the call holds.
#define TR_PPT 4                           // candidates per thread and chunk
#define TR_CHUNK (256 * TR_PPT)            // candidates per CTA

// candidates of a depth call: the sampled pixels (step ii, step jj), ii < ww, jj < hh, of n frames of h x w, row-major
struct TrDepth {
  const uint16_t* data;
  int w, step, ww;
  long long frame_px, n;  // h w, hh ww
  TsIntrin in;
  __device__ __forceinline__ bool point(int f, long long q, float4& r) const {
    const int qi = (int)q, jj = qi / ww, ii = qi - jj * ww, i = ii * step, j = jj * step;  // q < INT32_MAX
    const uint16_t d = data[(size_t)f * frame_px + (size_t)j * w + i];
    if (!ts_depth_kept(in, d)) return false;
    const float3 c = ts_unproject(in, i, j, d);
    r = make_float4(c.x, c.y, c.z, 0.0f);
    return true;
  }
};
// candidates of a point-cloud call: the n points of one cloud f32[n, 3]
struct TrCloud {
  const float* data;
  float rmin, rmax;       // f32(min_ray_length), f32(max_ray_length)
  long long n;
  __device__ __forceinline__ bool point(int, long long q, float4& r) const {
    const float x = data[3 * q], y = data[3 * q + 1], z = data[3 * q + 2];
    if (!(isfinite(x) && isfinite(y) && isfinite(z))) return false;
    const float len = sqrtf((x * x + y * y) + z * z);
    if (!(len >= rmin && len < rmax)) return false;
    r = make_float4(x, y, z, 0.0f);
    return true;
  }
};

// CTA (c, f): candidates c TR_CHUNK .. of frame f, TR_PPT consecutive ones per thread.  COUNT: cnt[f C + c] = kept;
// else the kept records go to pts[off[f C + c] ..] in candidate order (a block scan places each thread's run).
template <class Src, bool COUNT>
__global__ void __launch_bounds__(256) k_tr_select(Src src, int C, long long* __restrict__ cnt, const long long* __restrict__ off,
                                                   float4* __restrict__ pts) {
  typedef cub::BlockScan<int, 256> Scan;
  __shared__ typename Scan::TempStorage tmp;
  const int f = blockIdx.y;
  const long long q0 = (long long)blockIdx.x * TR_CHUNK + threadIdx.x * TR_PPT;
  float4 r[TR_PPT];
  unsigned keep = 0;
#pragma unroll
  for (int k = 0; k < TR_PPT; k++) keep |= (q0 + k < src.n && src.point(f, q0 + k, r[k])) ? 1u << k : 0u;
  int pos, total;
  Scan(tmp).ExclusiveSum(__popc(keep), pos, total);
  const size_t chunk = (size_t)f * C + blockIdx.x;
  if (COUNT) {
    if (threadIdx.x == 0) cnt[chunk] = total;
    return;
  }
  long long row = off[chunk] + pos;
#pragma unroll
  for (int k = 0; k < TR_PPT; k++)
    if (keep >> k & 1u) pts[row++] = r[k];
}

// Tracking of n frames against submaps sub of m: selection of src (whose data is `input`, in `mem`, in_bytes long), then
// rg_lm.  The arguments have been checked.
template <class Src>
static int tr_track(tslam_tsdf_t* m, Src src, const void* input, int mem, size_t in_bytes, int n, const int* sub, const double* R0,
                    const double* T0, float huber, int max_iters, int min_points, double* R_out, double* T_out, double* H_out,
                    double* b_out, double* cost2, int64_t* info5, cudaStream_t st) {
  int rc = ts_flush_pending(m, st);
  if (!rc) rc = ts_check_deferred_async(m, st);
  if (rc) return rc;
  const long long C = src.n > 0 ? (src.n + TR_CHUNK - 1) / TR_CHUNK : 1;  // chunks per frame
  const long long nc = (long long)n * C;
  if (C > INT32_MAX) { ts_set_error("tslam_tsdf_track: %lld candidates per frame", src.n); return TSLAM_E_INVALID; }
  size_t scan_tmp = 0;
  TS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (long long*)nullptr, (long long*)nullptr, nc + 1, st));
  const size_t cb = rg_align((size_t)(nc + 1) * 8), stage_b = mem == TSLAM_MEM_HOST ? rg_align(in_bytes) : 0;
  rc = rg_reserve(&m->reg_blk, &m->reg_blk_bytes, 2 * cb + rg_align(scan_tmp) + stage_b);
  if (rc) return rc;
  char* w = (char*)m->reg_blk;
  long long* cnt = (long long*)w; w += cb;
  long long* off = (long long*)w; w += cb;
  void* tmp = w; w += rg_align(scan_tmp);
  src.data = (decltype(src.data))input;
  if (mem == TSLAM_MEM_HOST) {
    TS_CUDA(cudaMemcpyAsync(w, input, in_bytes, cudaMemcpyHostToDevice, st));
    src.data = (decltype(src.data))w;
  }
  const dim3 grid((unsigned)C, (unsigned)n);
  TS_CUDA(cudaMemsetAsync(cnt + nc, 0, 8, st));
  k_tr_select<Src, true><<<grid, 256, 0, st>>>(src, (int)C, cnt, nullptr, nullptr);
  TS_LAUNCH_CHECK(m);
  TS_CUDA(cub::DeviceScan::ExclusiveSum(tmp, scan_tmp, cnt, off, nc + 1, st));
  std::vector<long long> p0(n + 1);  // off[f C]: the first record of frame f, p0[n] = every record
  TS_CUDA(cudaMemcpy2DAsync(p0.data(), 8, off, (size_t)C * 8, 8, (size_t)n + 1, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  std::vector<int> np(n);
  for (int f = 0; f < n; f++) np[f] = (int)(p0[f + 1] - p0[f]);  // at most src.n <= INT32_MAX
  const long long ctas = rg_lm_ctas(n, np.data());
  if (ctas > INT32_MAX / 2) { ts_set_error("tslam_tsdf_track: too many points (%lld)", p0[n]); return TSLAM_E_CAPACITY; }
  const size_t pts_b = rg_align((size_t)p0[n] * 16);
  rc = rg_reserve(&m->reg_pts, &m->reg_pts_bytes, pts_b + rg_lm_bytes(n, ctas));
  if (rc) return rc;
  float4* pts = (float4*)m->reg_pts;
  if (p0[n] > 0) {
    k_tr_select<Src, false><<<grid, 256, 0, st>>>(src, (int)C, nullptr, off, pts);
    TS_LAUNCH_CHECK(m);
  }
  return rg_lm(m, m->g, pts, (char*)m->reg_pts + pts_b, n, p0.data(), np.data(), sub, R0, T0, m->in.vs, huber, max_iters, min_points,
               R_out, T_out, H_out, b_out, cost2, info5, st);
}

// Argument checks shared by both entries: the submaps and the initial poses of n frames
static int tr_check_frames(const tslam_tsdf_t* m, const char* fn, int n, const int32_t* submaps, const double* R0, const double* T0) {
  for (int f = 0; f < n; f++) {
    const int s = submaps ? submaps[f] : 0;
    if (s < 0 || s >= m->cfg.max_submaps) {
      ts_set_error("%s: frame %d: submap %d out of range", fn, f, s);
      return TSLAM_E_INVALID;
    }
    for (int i = 0; i < 12; i++) {
      if (!std::isfinite(i < 9 ? R0[9 * f + i] : T0[3 * f + i - 9])) {
        ts_set_error("%s: frame %d: initial pose not finite", fn, f);
        return TSLAM_E_INVALID;
      }
    }
  }
  return TSLAM_OK;
}

static bool tr_bad_params(float huber, int32_t max_iters, int32_t min_points) {
  return !std::isfinite(huber) || !(huber > 0.0f) || max_iters < 0 || min_points < 0;
}

extern "C" int tslam_tsdf_track_depth(tslam_tsdf_t* m, const uint16_t* depth, int mem, int32_t n, int32_t height, int32_t width,
                                      const int32_t* submaps, const double* R0, const double* T0, int32_t step, float huber,
                                      int32_t max_iters, int32_t min_points, double* R_out, double* T_out, double* H_out, double* b_out,
                                      double* cost2, int64_t* info5, void* stream) {
  static const char* fn = "tslam_tsdf_track_depth";
  if (n < 1 || n > TSLAM_REG_MAX_PAIRS) {
    ts_set_error("%s: n %d outside [1, %d]", fn, n, TSLAM_REG_MAX_PAIRS);
    return TSLAM_E_INVALID;
  }
  if (step < 1 || height <= 0 || width <= 0 || tr_bad_params(huber, max_iters, min_points) ||
      (mem != TSLAM_MEM_DEVICE && mem != TSLAM_MEM_HOST)) {
    ts_set_error("%s: step >= 1, height and width > 0, huber finite and > 0, max_iters and min_points >= 0, mem a TSLAM_MEM_*", fn);
    return TSLAM_E_INVALID;
  }
  if (!m || !depth || !R0 || !T0 || !R_out || !T_out || !H_out || !b_out || !cost2 || !info5) {
    ts_set_error("%s: NULL handle or array", fn);
    return TSLAM_E_INVALID;
  }
  int rc = tr_check_frames(m, fn, n, submaps, R0, T0);
  if (rc) return rc;
  TrDepth src;
  src.data = nullptr;
  src.w = width;
  src.step = step;
  src.ww = width / step;
  src.frame_px = (long long)height * width;
  src.n = (long long)(height / step) * src.ww;  // range(0, h / step) x range(0, w / step), as integrate samples
  src.in = m->in;
  if (src.n > INT32_MAX) { ts_set_error("%s: %lld sampled pixels per frame", fn, src.n); return TSLAM_E_INVALID; }
  std::vector<int> sub(n);
  for (int f = 0; f < n; f++) sub[f] = submaps ? submaps[f] : 0;
  return tr_track(m, src, depth, mem, (size_t)n * src.frame_px * 2, n, sub.data(), R0, T0, huber, max_iters, min_points, R_out, T_out,
                  H_out, b_out, cost2, info5, (cudaStream_t)stream);
}

extern "C" int tslam_tsdf_track_points(tslam_tsdf_t* m, const float* xyz, int mem, int32_t n_points, int32_t submap, const double* R0,
                                       const double* T0, float huber, int32_t max_iters, int32_t min_points, double* R_out, double* T_out,
                                       double* H_out, double* b_out, double* cost2, int64_t* info5, void* stream) {
  static const char* fn = "tslam_tsdf_track_points";
  if (n_points < 0 || tr_bad_params(huber, max_iters, min_points) || (mem != TSLAM_MEM_DEVICE && mem != TSLAM_MEM_HOST)) {
    ts_set_error("%s: n_points >= 0, huber finite and > 0, max_iters and min_points >= 0, mem a TSLAM_MEM_*", fn);
    return TSLAM_E_INVALID;
  }
  if (!m || (!xyz && n_points > 0) || !R0 || !T0 || !R_out || !T_out || !H_out || !b_out || !cost2 || !info5) {
    ts_set_error("%s: NULL handle or array", fn);
    return TSLAM_E_INVALID;
  }
  int rc = tr_check_frames(m, fn, 1, &submap, R0, T0);
  if (rc) return rc;
  TrCloud src;
  src.data = nullptr;
  src.rmin = (float)m->cfg.min_ray_length;
  src.rmax = m->in.max_ray;
  src.n = n_points;
  return tr_track(m, src, xyz, mem, (size_t)n_points * 12, 1, &submap, R0, T0, huber, max_iters, min_points, R_out, T_out, H_out, b_out,
                  cost2, info5, (cudaStream_t)stream);
}
