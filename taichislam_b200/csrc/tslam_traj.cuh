// Trajectories against an ESDF (DESIGN.md section 7, "Trajectories"; include/tslam.h, tslam_esdf_trajectory): uniform
// cubic B-splines whose free control points an L-BFGS solve pushes out of the clearance while keeping them smooth and
// within velocity and acceleration limits.  One CTA per trajectory runs the whole solve, evaluations included; the
// field is read through es_point, the body of the ESDF queries, so a sample sees exactly what tslam_esdf_query /
// tslam_octo_esdf_query return at the same f32 point.  Instantiated next to each ESDF (tslam_esdf.cu, EsTsdf;
// tslam_octo_esdf.cu, EsOcto).  tests/trajectory_reference.py restates every operation below in numpy.
//
// Trajectory t: control points Q_0 .. Q_{N-1} (f64, the submap-local map frame), knot span dt; spans j = 0 .. N-4 use
// Q_j .. Q_{j+3}.  Q_0..2 and Q_{N-3..N-1} are fixed; the free variables are the 3 (N - 6) coordinates of Q_3 .. Q_{N-4},
// in index order e = 3 i + axis.  A sample at u of span j has position x = ((b0 Q_j + b1 Q_{j+1}) + b2 Q_{j+2}) + b3 Q_{j+3}
// (f64, rounded to f32 once), with the basis rows the host tabulates (tj_basis); collision samples sit at u = k/K on every
// span plus u = 1 on the last one, check samples likewise at k/C.
//
// Cost, all f64 (every operation correctly rounded and never contracted: the library is built with -fmad=false):
//   J_s = sum_i |jerk_i|^2,  jerk_i = ((Q_{i+3} - 3 Q_{i+2}) + 3 Q_{i+1}) - Q_i,  |v|^2 = (vx vx + vy vy) + vz vz
//   J_c = sum over valid samples with d < c of r^2,  r = c - d;  its gradient -2 r b_o g reaches Q_{j+o}
//   J_u = the number of invalid samples (no gradient)
//   J_f = sum_i max(0, |V_i|^2 - v^2)^2 + sum_i max(0, |A_i|^2 - a^2)^2,  V_i = (Q_{i+1} - Q_i) / dt,
//         A_i = ((Q_{i+2} - 2 Q_{i+1}) + Q_i) / dt2,  dt2 = dt dt
//   J   = ((w_s J_s + w_c J_c) + w_f J_f) + w_u J_u
// Sums over a trajectory: thread t of the CTA (TJ_THREADS threads) adds its items t, t + TJ_THREADS, ... in order to a
// partial starting at 0 (the collision items of a span are its samples in order; J_f's items are the velocity terms,
// then the acceleration terms, into the same partial); the partials p[0..TJ_THREADS-1] are then added by the halving
// tree p[i] += p[i + s], s = TJ_THREADS/2 .. 1 (tj_sum).  Dot products over the free variables are sums of this kind
// with items e.  A span's collision gradient goes to global scratch, 12 values per span, each its samples' terms in
// order; the gradient of free coordinate (i, axis) is then, each sum in the order written,
//   G_s = sum_{m=i-3..i} (2 jerk_m) cj[i-m],  cj = (-1, 3, -3, 1)
//   G_c = sum_{j=i-3..i} (span j's term for its control point i - j)
//   G_f = sum_{m=i-1..i} (+-(4 h_m) V_m) / dt  +  sum_{m=i-2..i} (ca[i-m] (4 k_m) A_m) / dt2 over the active hinges,
//         h_m = |V_m|^2 - v^2 > 0, k_m = |A_m|^2 - a^2 > 0, ca = (1, -2, 1), the sign - for m = i
//   G   = (w_s G_s + w_c G_c) + w_f G_f.
// Solver: L-BFGS over the free variables with memory M.  Direction: -(g * (vs / |g|inf)) when there is no pair (vs the
// voxel size in f64), else the two-loop recursion with gamma = s'y / y'y of the newest pair; a direction with g'd >= 0
// drops the history and takes the scaled -g.  Armijo backtracking from alpha = 1 (J_t <= J + (c1 alpha) g'd, c1 = 1e-4,
// halving, at most 30 trials).  A step keeps s = X - Q, y = G_t - G when s'y > 1e-10 y'y.  Stop: |g|inf <= g_tol
// (status 1), no acceptable trial (2), max_iters steps (0); N < 7: one evaluation, status 3.
#pragma once
#include <cmath>
#include <vector>
#include "tslam_esdf_common.cuh"

#define TJ_THREADS 256
#define TJ_MAX_N 1024
#define TJ_MAX_T 1024
#define TJ_MAX_SUM_N (1 << 20)
#define TJ_MAX_K 16
#define TJ_MAX_C 64
#define TJ_MAX_M 16
#define TJ_TRIALS 30
#define TJ_COST 6  // cost row: J_s, J_c, J_f, J_u at the result, J at the input, least valid check distance
#define TJ_INFO 7  // info row: iterations, evaluations, status, invalid check samples, valid with d < c, its span, its k

struct TjArgs {
  const double* bk;      // [(K+1)*4] basis rows of the collision samples (row k: u = k/K)
  const double* bc;      // [(C+1)*4] basis rows of the check samples
  const long long* off;  // [T+1] first control point of each trajectory
  const double* q_in;    // [sum N * 3]
  double* q_out;
  double* ws;            // per trajectory (18 + 6 M) N doubles from off[t] (18 + 6 M): D, G_t, span terms, M s, M y
  double* cost;          // [T * TJ_COST]
  int* info;             // [T * TJ_INFO]
  double dt, dt2, v2, a2, w_s, w_c, w_f, w_u, c, g_tol, vs;
  int K, C, M, max_iters;
};

// The sum over the CTA of each v[q] (tj sum order, header): partials in red[q * TJ_THREADS + t], the halving tree in
// shared memory down to one warp, then shuffles; every thread gets the sums.
template <int NV>
__device__ __forceinline__ void tj_sum(double (&v)[NV], double* red) {
  const int t = threadIdx.x;
  __syncthreads();
#pragma unroll
  for (int q = 0; q < NV; q++) red[q * TJ_THREADS + t] = v[q];
  __syncthreads();
  for (int s = TJ_THREADS / 2; s >= 32; s >>= 1) {
    if (t < s) {
#pragma unroll
      for (int q = 0; q < NV; q++) red[q * TJ_THREADS + t] += red[q * TJ_THREADS + t + s];
    }
    __syncthreads();
  }
  if (t < 32) {
#pragma unroll
    for (int q = 0; q < NV; q++) {
      double x = red[q * TJ_THREADS + t];
      for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
      if (t == 0) red[q * TJ_THREADS] = x;
    }
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < NV; q++) v[q] = red[q * TJ_THREADS];
}

// a'b over the free coordinates e = 9 .. 3N - 10
__device__ __forceinline__ double tj_dot(const double* x, const double* y, int n3, double* red) {
  double v[1] = {0.0};
  for (int e = 9 + threadIdx.x; e < n3 - 9; e += TJ_THREADS) v[0] += x[e] * y[e];
  tj_sum(v, red);
  return v[0];
}

// f32 position of the sample with basis row b on span j
__device__ __forceinline__ void tj_pos(const double* Q, int j, const double* b, float x[3]) {
#pragma unroll
  for (int a = 0; a < 3; a++) {
    const double* q = Q + 3 * j + a;
    x[a] = __double2float_rn(((b[0] * q[0] + b[1] * q[3]) + b[2] * q[6]) + b[3] * q[9]);
  }
}
__device__ __forceinline__ double tj_jerk(const double* Q, int i, int a) {
  const double* q = Q + 3 * i + a;
  return ((q[9] - 3.0 * q[6]) + 3.0 * q[3]) - q[0];
}
__device__ __forceinline__ double tj_vel(const double* Q, int i, int a, double dt) { return (Q[3 * i + 3 + a] - Q[3 * i + a]) / dt; }
__device__ __forceinline__ double tj_acc(const double* Q, int i, int a, double dt2) {
  const double* q = Q + 3 * i + a;
  return ((q[6] - 2.0 * q[3]) + q[0]) / dt2;
}
__device__ __forceinline__ double tj_sq3(double x, double y, double z) { return (x * x + y * y) + z * z; }

// J at Q (returned) with its terms J4 = (J_s, J_c, J_f, J_u) and its gradient at the free coordinates into G; span terms
// go through cs (global scratch, 12 per span)
template <class P>
__device__ __forceinline__ double tj_eval(const P& p, int nb, const TjArgs& a, int N, const double* Q, double* G, double* cs, double* red, double J4[4]) {
  const int tid = threadIdx.x, nsp = N - 3;
  __syncthreads();  // Q complete
  double v[4] = {0.0, 0.0, 0.0, 0.0};  // J_s, J_c, J_f, J_u partials
  for (int j = tid; j < nsp; j += TJ_THREADS) {
    double cg[12];
#pragma unroll
    for (int q = 0; q < 12; q++) cg[q] = 0.0;
    const int kn = a.K + (j == nsp - 1 ? 1 : 0);
    for (int k = 0; k < kn; k++) {
      const double* b = a.bk + 4 * k;
      float x[3], d, g[3];
      tj_pos(Q, j, b, x);
      if (!es_point(p, nb, x, d, g[0], g[1], g[2])) { v[3] += 1.0; continue; }
      if (!((double)d < a.c)) continue;
      const double r = a.c - (double)d;
      v[1] += r * r;
      const double m = -2.0 * r;
#pragma unroll
      for (int o = 0; o < 4; o++) {
        const double mo = m * b[o];
#pragma unroll
        for (int ax = 0; ax < 3; ax++) cg[3 * o + ax] += mo * (double)g[ax];
      }
    }
#pragma unroll
    for (int q = 0; q < 12; q++) cs[12 * j + q] = cg[q];
  }
  for (int i = tid; i < nsp; i += TJ_THREADS) v[0] += tj_sq3(tj_jerk(Q, i, 0), tj_jerk(Q, i, 1), tj_jerk(Q, i, 2));
  for (int i = tid; i < N - 1; i += TJ_THREADS) {
    const double h = tj_sq3(tj_vel(Q, i, 0, a.dt), tj_vel(Q, i, 1, a.dt), tj_vel(Q, i, 2, a.dt)) - a.v2;
    if (h > 0.0) v[2] += h * h;
  }
  for (int i = tid; i < N - 2; i += TJ_THREADS) {
    const double h = tj_sq3(tj_acc(Q, i, 0, a.dt2), tj_acc(Q, i, 1, a.dt2), tj_acc(Q, i, 2, a.dt2)) - a.a2;
    if (h > 0.0) v[2] += h * h;
  }
  tj_sum(v, red);  // (also makes the span terms visible to the CTA)
  for (int e = 9 + tid; e < 3 * N - 9; e += TJ_THREADS) {
    const int i = e / 3, ax = e - 3 * i;
    double gs = 0.0, gc = 0.0, gf = 0.0;
    for (int m = i - 3; m <= i; m++) {
      const int o = i - m;
      gs += (2.0 * tj_jerk(Q, m, ax)) * (o == 0 ? -1.0 : (o == 1 ? 3.0 : (o == 2 ? -3.0 : 1.0)));
    }
    for (int j = i - 3; j <= i; j++) gc += cs[12 * j + 3 * (i - j) + ax];
    for (int m = i - 1; m <= i; m++) {
      const double vx = tj_vel(Q, m, 0, a.dt), vy = tj_vel(Q, m, 1, a.dt), vz = tj_vel(Q, m, 2, a.dt);
      const double h = tj_sq3(vx, vy, vz) - a.v2;
      if (h > 0.0) {
        const double t = (4.0 * h) * (ax == 0 ? vx : (ax == 1 ? vy : vz));
        gf += (m == i ? -t : t) / a.dt;
      }
    }
    for (int m = i - 2; m <= i; m++) {
      const double ux = tj_acc(Q, m, 0, a.dt2), uy = tj_acc(Q, m, 1, a.dt2), uz = tj_acc(Q, m, 2, a.dt2);
      const double h = tj_sq3(ux, uy, uz) - a.a2;
      if (h > 0.0) {
        const double t = (4.0 * h) * (ax == 0 ? ux : (ax == 1 ? uy : uz));
        gf += (i - m == 1 ? -2.0 * t : t) / a.dt2;
      }
    }
    G[e] = (a.w_s * gs + a.w_c * gc) + a.w_f * gf;
  }
  J4[0] = v[0]; J4[1] = v[1]; J4[2] = v[2]; J4[3] = v[3];
  return ((a.w_s * v[0] + a.w_c * v[1]) + a.w_f * v[2]) + a.w_u * v[3];
}

// |G|inf over the free coordinates (a max: exact in any order)
__device__ __forceinline__ double tj_max_abs(const double* G, int n3, double* red) {
  double m = 0.0;
  for (int e = 9 + threadIdx.x; e < n3 - 9; e += TJ_THREADS) m = fmax(m, fabs(G[e]));
  __syncthreads();
  red[threadIdx.x] = m;
  __syncthreads();
  for (int s = TJ_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  return red[0];
}

// The dense check of Q: C samples per span (+ u = 1 on the last); the least valid d and its sample (ties: the lower
// index j (C + 1) + k), invalid samples, valid samples with d < c
template <class P>
__device__ __forceinline__ void tj_check(const P& p, int nb, const TjArgs& a, int N, const double* Q, double* red, float& dmin, int& imin, int& n_inv,
                         int& n_close) {
  const int tid = threadIdx.x, nsp = N - 3;
  float best = __int_as_float(0x7f800000);
  int bi = 0x7fffffff;
  double v[2] = {0.0, 0.0};
  for (int j = tid; j < nsp; j += TJ_THREADS) {
    const int kn = a.C + (j == nsp - 1 ? 1 : 0);
    for (int k = 0; k < kn; k++) {
      float x[3], d, g[3];
      tj_pos(Q, j, a.bc + 4 * k, x);
      if (!es_point(p, nb, x, d, g[0], g[1], g[2])) { v[0] += 1.0; continue; }
      if ((double)d < a.c) v[1] += 1.0;
      if (d < best) { best = d; bi = j * (a.C + 1) + k; }
    }
  }
  tj_sum(v, red);
  n_inv = (int)v[0];
  n_close = (int)v[1];
  float* rd = (float*)red;
  int* ri = (int*)(red + TJ_THREADS);
  __syncthreads();
  rd[tid] = best;
  ri[tid] = bi;
  __syncthreads();
  for (int s = TJ_THREADS / 2; s > 0; s >>= 1) {
    if (tid < s) {
      const float d2 = rd[tid + s];
      const int i2 = ri[tid + s];
      if (d2 < rd[tid] || (d2 == rd[tid] && i2 < ri[tid])) { rd[tid] = d2; ri[tid] = i2; }
    }
    __syncthreads();
  }
  dmin = rd[0];
  imin = ri[0];
}

// One CTA per trajectory.  Dynamic shared memory: Q, G, X (3N doubles each), the reduction buffer (4 TJ_THREADS doubles),
// alpha and rho of the two-loop recursion (2 TJ_MAX_M doubles).
template <class P>
__global__ void __launch_bounds__(TJ_THREADS, 1) k_traj_solve(P p, TjArgs a) {
  extern __shared__ double tj_sm[];
  const int tid = threadIdx.x;
  const long long o = a.off[blockIdx.x];
  const int N = (int)(a.off[blockIdx.x + 1] - o), n3 = 3 * N, M = a.M;
  double* Q = tj_sm;
  double* G = Q + n3;
  double* X = G + n3;
  double* red = X + n3;
  double* al = red + 4 * TJ_THREADS;
  double* rho = al + TJ_MAX_M;
  double* D = a.ws + o * (18 + 6 * M);
  double* GT = D + n3;
  double* cs = GT + n3;
  double* S = cs + 12 * N;
  double* Y = S + (size_t)M * n3;
  const int nb = *p.a.nb_seen;
  for (int e = tid; e < n3; e += TJ_THREADS) {
    const double q = a.q_in[3 * o + e];
    Q[e] = q; X[e] = q; G[e] = 0.0; GT[e] = 0.0;
  }
  double J4[4], J4t[4];
  double J = tj_eval(p, nb, a, N, Q, G, cs, red, J4);
  const double J_in = J;
  int iters = 0, evals = 1, status = 3, hn = 0, hh = 0;  // pairs kept, next slot (the oldest when hn == M)
  double gamma = 1.0;
  while (N >= 7) {
    const double gi = tj_max_abs(G, n3, red);
    if (gi <= a.g_tol) { status = 1; break; }
    if (iters >= a.max_iters) { status = 0; break; }
    double gd = 0.0;
    bool steep = hn == 0;
    if (!steep) {  // two-loop recursion, newest pair first
      for (int e = 9 + tid; e < n3 - 9; e += TJ_THREADS) D[e] = G[e];
      for (int q = 0; q < hn; q++) {
        const int sl = (hh - 1 - q + M) % M;
        const double* s = S + (size_t)sl * n3;
        const double* y = Y + (size_t)sl * n3;
        const double aq = rho[sl] * tj_dot(s, D, n3, red);
        if (tid == 0) al[q] = aq;
        for (int e = 9 + tid; e < n3 - 9; e += TJ_THREADS) D[e] = D[e] - aq * y[e];
      }
      for (int e = 9 + tid; e < n3 - 9; e += TJ_THREADS) D[e] = gamma * D[e];
      for (int q = hn - 1; q >= 0; q--) {
        const int sl = (hh - 1 - q + M) % M;
        const double* s = S + (size_t)sl * n3;
        const double* y = Y + (size_t)sl * n3;
        const double b = rho[sl] * tj_dot(y, D, n3, red);  // (its barriers publish al[q])
        const double aq = al[q];
        for (int e = 9 + tid; e < n3 - 9; e += TJ_THREADS) D[e] = D[e] + (aq - b) * s[e];
      }
      for (int e = 9 + tid; e < n3 - 9; e += TJ_THREADS) D[e] = -D[e];
      gd = tj_dot(G, D, n3, red);
      if (!(gd < 0.0)) { steep = true; hn = 0; hh = 0; }
    }
    if (steep) {
      const double sc = a.vs / gi;
      for (int e = 9 + tid; e < n3 - 9; e += TJ_THREADS) D[e] = -(G[e] * sc);
      gd = tj_dot(G, D, n3, red);
    }
    double alpha = 1.0, Jt = 0.0;
    bool ok = false;
    for (int k = 0; k < TJ_TRIALS; k++) {
      for (int e = 9 + tid; e < n3 - 9; e += TJ_THREADS) X[e] = Q[e] + alpha * D[e];
      Jt = tj_eval(p, nb, a, N, X, GT, cs, red, J4t);
      evals++;
      if (Jt <= J + (1e-4 * alpha) * gd) { ok = true; break; }
      alpha *= 0.5;
    }
    if (!ok) { status = 2; break; }
    // the pair (s, y) = (X - Q, G_t - G), kept when s'y > 1e-10 y'y
    double sy[2] = {0.0, 0.0};
    for (int e = 9 + tid; e < n3 - 9; e += TJ_THREADS) {
      const double s = X[e] - Q[e], y = GT[e] - G[e];
      sy[0] += s * y;
      sy[1] += y * y;
    }
    tj_sum(sy, red);
    if (sy[0] > 1e-10 * sy[1]) {
      double* s = S + (size_t)hh * n3;
      double* y = Y + (size_t)hh * n3;
      for (int e = 9 + tid; e < n3 - 9; e += TJ_THREADS) { s[e] = X[e] - Q[e]; y[e] = GT[e] - G[e]; }
      if (tid == 0) rho[hh] = 1.0 / sy[0];
      gamma = sy[0] / sy[1];
      hh = (hh + 1) % M;
      hn = hn < M ? hn + 1 : M;
    }
    for (int e = 9 + tid; e < n3 - 9; e += TJ_THREADS) { Q[e] = X[e]; G[e] = GT[e]; }
    J = Jt;
#pragma unroll
    for (int q = 0; q < 4; q++) J4[q] = J4t[q];
    iters++;
  }
  __syncthreads();
  float dmin;
  int imin, n_inv, n_close;
  tj_check(p, nb, a, N, Q, red, dmin, imin, n_inv, n_close);
  for (int e = tid; e < n3; e += TJ_THREADS) a.q_out[3 * o + e] = Q[e];
  if (tid == 0) {
    double* c = a.cost + (size_t)blockIdx.x * TJ_COST;
    c[0] = J4[0]; c[1] = J4[1]; c[2] = J4[2]; c[3] = J4[3]; c[4] = J_in; c[5] = (double)dmin;
    int* f = a.info + (size_t)blockIdx.x * TJ_INFO;
    const bool any = imin != 0x7fffffff;
    f[0] = iters; f[1] = evals; f[2] = status; f[3] = n_inv; f[4] = n_close;
    f[5] = any ? imin / (a.C + 1) : -1;
    f[6] = any ? imin % (a.C + 1) : -1;
  }
}

// ---- host ------------------------------------------------------------------------------------------------------------
// The basis rows of n samples per span, u = k / n for k = 0 .. n (row n: u = 1), in f64:
//   w = 1 - u, u2 = u u, u3 = u2 u;  b0 = ((w w) w) / 6,  b1 = ((3 u3 - 6 u2) + 4) / 6,
//   b2 = (((-3 u3 + 3 u2) + 3 u) + 1) / 6,  b3 = u3 / 6
static void tj_basis(int n, double* b) {
  for (int k = 0; k <= n; k++) {
    const double u = (double)k / (double)n, w = 1.0 - u, u2 = u * u, u3 = u2 * u;
    b[4 * k] = ((w * w) * w) / 6.0;
    b[4 * k + 1] = ((3.0 * u3 - 6.0 * u2) + 4.0) / 6.0;
    b[4 * k + 2] = (((-3.0 * u3 + 3.0 * u2) + 3.0 * u) + 1.0) / 6.0;
    b[4 * k + 3] = u3 / 6.0;
  }
}

static bool tj_fin_pos(double x) { return std::isfinite(x) && x > 0.0; }
static bool tj_fin_nneg(double x) { return std::isfinite(x) && x >= 0.0; }

// The argument checks of both entries, before the handle is looked at; *sum_n = sum of N
static int tj_check_args(const char* what, int32_t T, const int32_t* n_ctrl, const double* q_in, const tslam_traj_params_t* prm,
                         const double* q_out, const double* cost, const int32_t* info, long long* sum_n) {
  if (!n_ctrl || !q_in || !prm || !q_out || !cost || !info) {
    ts_set_error("%s: n_ctrl, ctrl_in, params, ctrl_out, cost and info must not be NULL", what);
    return TSLAM_E_INVALID;
  }
  if (T < 1 || T > TJ_MAX_T) { ts_set_error("%s: %d trajectories outside [1, %d]", what, T, TJ_MAX_T); return TSLAM_E_INVALID; }
  long long s = 0;
  for (int t = 0; t < T; t++) {
    if (n_ctrl[t] < 4 || n_ctrl[t] > TJ_MAX_N) {
      ts_set_error("%s: trajectory %d has %d control points, outside [4, %d]", what, t, n_ctrl[t], TJ_MAX_N);
      return TSLAM_E_INVALID;
    }
    s += n_ctrl[t];
  }
  if (s > TJ_MAX_SUM_N) { ts_set_error("%s: %lld control points in all, above 2^20", what, s); return TSLAM_E_INVALID; }
  const tslam_traj_params_t& p = *prm;
  if (p.samples < 1 || p.samples > TJ_MAX_K || p.check_samples < 1 || p.check_samples > TJ_MAX_C || p.memory < 1 ||
      p.memory > TJ_MAX_M) {
    ts_set_error("%s: samples %d, check_samples %d or memory %d outside [1, %d], [1, %d], [1, %d]", what, p.samples, p.check_samples,
                 p.memory, TJ_MAX_K, TJ_MAX_C, TJ_MAX_M);
    return TSLAM_E_INVALID;
  }
  if (!tj_fin_pos(p.dt) || !tj_fin_pos(p.v_max) || !tj_fin_pos(p.a_max)) {
    ts_set_error("%s: dt, v_max and a_max must be finite and > 0", what);
    return TSLAM_E_INVALID;
  }
  if (!tj_fin_nneg(p.w_smooth) || !tj_fin_nneg(p.w_collision) || !tj_fin_nneg(p.w_feasibility) || !tj_fin_nneg(p.w_unknown) ||
      !tj_fin_nneg(p.clearance) || !tj_fin_nneg(p.g_tol)) {
    ts_set_error("%s: the weights, clearance and g_tol must be finite and >= 0", what);
    return TSLAM_E_INVALID;
  }
  if (p.max_iters < 0) { ts_set_error("%s: max_iters %d < 0", what, p.max_iters); return TSLAM_E_INVALID; }
  for (long long e = 0; e < 3 * s; e++)
    if (!std::isfinite(q_in[e])) { ts_set_error("%s: control point coordinate %lld is not finite", what, e); return TSLAM_E_INVALID; }
  *sum_n = s;
  return TSLAM_OK;
}

// *mem holds at least `need` bytes: reallocated (contents dropped) to max(need, 2 x the old size) when smaller
static int tj_reserve(const char* what, void** mem, size_t* bytes, size_t need) {
  if (need <= *bytes) return TSLAM_OK;
  const size_t nb = need > 2 * *bytes ? need : 2 * *bytes;
  if (*mem) cudaFree(*mem);
  *mem = nullptr;
  *bytes = 0;
  const cudaError_t e = cudaMalloc(mem, nb);
  if (e != cudaSuccess) {
    cudaGetLastError();
    *mem = nullptr;
    ts_set_error("%s: cannot allocate %zu bytes of trajectory scratch (%s)", what, nb, cudaGetErrorString(e));
    return TSLAM_E_CUDA;
  }
  *bytes = nb;
  return TSLAM_OK;
}

// Upload, one launch, download, synchronise.  vs: the field's voxel size.
template <class P, class M>
static int tj_run(M* m, const P& p, float vs, const char* what, void** mem, size_t* mem_bytes, int32_t T, const int32_t* n_ctrl,
                  long long sum_n, const double* q_in, const tslam_traj_params_t* prm, double* q_out, double* cost, int32_t* info,
                  cudaStream_t st) {
  const int K = prm->samples, C = prm->check_samples, Mm = prm->memory;
  std::vector<double> hb(4 * (K + 1 + C + 1));
  tj_basis(K, hb.data());
  tj_basis(C, hb.data() + 4 * (K + 1));
  std::vector<long long> off(T + 1, 0);
  int n_max = 0;
  for (int t = 0; t < T; t++) { off[t + 1] = off[t] + n_ctrl[t]; n_max = n_ctrl[t] > n_max ? n_ctrl[t] : n_max; }
  // layout (8-byte words): basis, offsets, q_in, q_out, cost, work, then the int info rows
  const size_t w_b = hb.size(), w_off = T + 1, w_q = 3 * (size_t)sum_n, w_cost = (size_t)T * TJ_COST, w_ws = (size_t)(18 + 6 * Mm) * sum_n;
  const size_t words = w_b + w_off + 2 * w_q + w_cost + w_ws;
  const int rc = tj_reserve(what, mem, mem_bytes, words * 8 + (size_t)T * TJ_INFO * 4);
  if (rc) return rc;
  double* base = (double*)*mem;
  TjArgs a;
  a.bk = base;
  a.bc = base + 4 * (K + 1);
  a.off = (const long long*)(base + w_b);
  double* dq_in = base + w_b + w_off;
  a.q_in = dq_in;
  a.q_out = dq_in + w_q;
  a.cost = a.q_out + w_q;
  a.ws = a.cost + w_cost;
  a.info = (int*)(a.ws + w_ws);
  a.dt = prm->dt; a.dt2 = prm->dt * prm->dt; a.v2 = prm->v_max * prm->v_max; a.a2 = prm->a_max * prm->a_max;
  a.w_s = prm->w_smooth; a.w_c = prm->w_collision; a.w_f = prm->w_feasibility; a.w_u = prm->w_unknown;
  a.c = prm->clearance; a.g_tol = prm->g_tol; a.vs = (double)vs;
  a.K = K; a.C = C; a.M = Mm; a.max_iters = prm->max_iters;
  TS_CUDA(cudaMemcpyAsync(base, hb.data(), w_b * 8, cudaMemcpyHostToDevice, st));
  TS_CUDA(cudaMemcpyAsync(base + w_b, off.data(), w_off * 8, cudaMemcpyHostToDevice, st));
  TS_CUDA(cudaMemcpyAsync(dq_in, q_in, w_q * 8, cudaMemcpyHostToDevice, st));
  const size_t smem = (size_t)(9 * n_max + 4 * TJ_THREADS + 2 * TJ_MAX_M) * 8;
  TS_CUDA(cudaFuncSetAttribute(k_traj_solve<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_traj_solve<P><<<T, TJ_THREADS, smem, st>>>(p, a);
  TS_LAUNCH_CHECK(m);
  TS_CUDA(cudaMemcpyAsync(q_out, a.q_out, w_q * 8, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(cost, a.cost, w_cost * 8, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(info, a.info, (size_t)T * TJ_INFO * 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  return TSLAM_OK;
}
