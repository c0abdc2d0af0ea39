// libtslam.so - submap pose-graph optimisation (tslam_pose_graph_solve; DESIGN.md section 7, "Pose-graph optimisation").
//
// Levenberg-Marquardt over SE(3) node poses with odometry and loop edges, Cauchy-robust per edge (IRLS), all in f64.
// The damped normal equations are solved by block-Jacobi preconditioned conjugate gradients in one cooperative launch.
//
// Per LM evaluation, on `stream`:
//   k_pg_nodes<1>   damping and the 6x6 Cholesky preconditioner of every free node
//   k_pg_pcg        every CG iteration of the step (grid.sync() between phases; no host round trip)
//   k_pg_step       trial poses exp(delta) X
//   k_pg_edges<0>   per-edge cost terms at the trial poses, then k_pg_reduce (F, max |rho|, max |phi|): the host reads
//                   these 8 doubles, the only synchronisation of the iteration
// and after an accepted step k_pg_edges<1> (blocks and gradient pieces) and k_pg_nodes<0> (per-node sums in CSR order).
//
// J_j = -J_i exactly (negation is exact), so an edge's three blocks are B, B and -B with B = w J_i^T Omega J_i, and its
// gradient pieces are +-w J_i^T Omega e: k_pg_edges stores B and the piece once.
//
// Determinism: every per-node and per-edge quantity is computed by one thread from fixed inputs in a fixed order; F sums
// chunks of 256 edges in edge order and then the chunk sums in order (k_pg_reduce); CG dot products are per-warp butterfly
// sums over fixed chunks of 32 free nodes, summed by every thread in chunk order.  Nothing depends on the grid size or
// the SM count.
#include <cooperative_groups.h>
#include <cmath>
#include <vector>
#include "tslam_internal.cuh"

namespace cg = cooperative_groups;

#define PG_MAX_N 4096
#define PG_MAX_E 65536
#define PG_SMALL 1e-2  // rotation angle below which every coefficient is its series (terms through theta^4)
#define PG_CHUNK 256   // k_pg_reduce: elements per thread, summed in order
#define PG_CG_BLOCK 128

namespace {

// packed upper triangle of a symmetric 6x6, row-major: (0,0) (0,1) .. (0,5) (1,1) ..
__host__ __device__ constexpr int pu(int r, int c) { return r <= c ? r * 6 - r * (r - 1) / 2 + (c - r) : c * 6 - c * (c - 1) / 2 + (r - c); }
// packed lower triangle (Cholesky factor), row-major: (0,0) (1,0) (1,1) (2,0) ..
__host__ __device__ constexpr int pl(int r, int c) { return r * (r + 1) / 2 + c; }

struct PgEdgeArgs {
  int E;
  const int2* ij;
  const double* X;      // [N,12] R row-major, t
  const double* Z;      // [E,12]
  const double* om;     // [E,21] packed upper
  const double* c;      // [E]
  double *s, *w, *term; // [E]
  double *B, *gv;       // [E,21], [E,6] (linearise mode)
};

__device__ __forceinline__ void pg_coeffs(double th, double& A, double& B, double& C, double& D, double& c2, double& c3) {
  const double t2 = th * th, t4 = t2 * t2;
  if (th < PG_SMALL) {
    A = 1.0 - t2 / 6.0 + t4 / 120.0;
    B = 0.5 - t2 / 24.0 + t4 / 720.0;
    C = 1.0 / 6.0 - t2 / 120.0 + t4 / 5040.0;
    D = 1.0 / 12.0 + t2 / 720.0 + t4 / 30240.0;
    c2 = 1.0 / 24.0 - t2 / 720.0 + t4 / 40320.0;
    c3 = 1.0 / 120.0 - t2 / 2520.0 + t4 / 120960.0;
  } else {
    double sn, cs, h, hc;
    sincos(th, &sn, &cs);
    sincos(0.5 * th, &h, &hc);
    A = sn / th;
    B = 2.0 * h * h / t2;
    C = (th - sn) / (t2 * th);
    D = (1.0 - 0.5 * th * hc / h) / t2;
    c2 = (t2 - 4.0 * h * h) / (2.0 * t4);
    c3 = (2.0 * th - 3.0 * sn + th * cs) / (2.0 * t4 * th);
  }
}

__device__ __forceinline__ void hat3(const double* v, double* K) {
  K[0] = 0.0;   K[1] = -v[2]; K[2] = v[1];
  K[3] = v[2];  K[4] = 0.0;   K[5] = -v[0];
  K[6] = -v[1]; K[7] = v[0];  K[8] = 0.0;
}

__device__ __forceinline__ void mul3(const double* a, const double* b, double* o) {
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) o[r * 3 + c] = a[r * 3] * b[c] + a[r * 3 + 1] * b[3 + c] + a[r * 3 + 2] * b[6 + c];
}

// Log(R, t) -> (rho, phi): the exact inverse of exp (tests/pose_graph_reference.log states the same operations).
__device__ void pg_log(const double* R, const double* t, double* xi) {
  const double w0 = R[7] - R[5], w1 = R[2] - R[6], w2 = R[3] - R[1];
  const double c = 0.5 * (R[0] + R[4] + R[8] - 1.0);
  const double sn = 0.5 * sqrt(w0 * w0 + w1 * w1 + w2 * w2);
  const double th = atan2(sn, c);
  double phi[3];
  if (c < 0.0) {  // near pi: the axis from the symmetric part, signed by w
    const double oc = 1.0 - c;
    double S[9];
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
      for (int q = 0; q < 3; q++) S[r * 3 + q] = 0.5 * (R[r * 3 + q] + R[q * 3 + r]) - (r == q ? c : 0.0);
    int k = 0;
    if (S[4] > S[0]) k = 1;
    if (S[8] > S[k * 4]) k = 2;
    const double uk = sqrt(S[k * 4] / oc);
    double u[3];
#pragma unroll
    for (int q = 0; q < 3; q++) u[q] = S[k * 3 + q] / (oc * uk);
    u[k] = uk;
    const double sg = (u[0] * w0 + u[1] * w1 + u[2] * w2) < 0.0 ? -th : th;
#pragma unroll
    for (int q = 0; q < 3; q++) phi[q] = sg * u[q];
  } else {
    const double t2 = th * th;
    const double f = th < PG_SMALL ? 0.5 * (1.0 + t2 / 6.0 + 7.0 * t2 * t2 / 360.0) : 0.5 * th / sn;
    phi[0] = f * w0;
    phi[1] = f * w1;
    phi[2] = f * w2;
  }
  double A, B, C, D, c2, c3;
  pg_coeffs(th, A, B, C, D, c2, c3);
  double K[9], K2[9];
  hat3(phi, K);
  mul3(K, K, K2);
#pragma unroll
  for (int r = 0; r < 3; r++) {
    double v = t[r];
#pragma unroll
    for (int q = 0; q < 3; q++) v += (-0.5 * K[r * 3 + q] + D * K2[r * 3 + q]) * t[q];
    xi[r] = v;
    xi[3 + r] = phi[r];
  }
}

// X' = exp(xi) X: R' = E R, t' = E t + V rho.
__device__ void pg_update(const double* xi, const double* X, double* Xo) {
  const double* phi = xi + 3;
  double A, B, C, D, c2, c3;
  pg_coeffs(sqrt(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2]), A, B, C, D, c2, c3);
  double K[9], K2[9], E[9], V[9];
  hat3(phi, K);
  mul3(K, K, K2);
#pragma unroll
  for (int q = 0; q < 9; q++) {
    const double I = (q % 4 == 0) ? 1.0 : 0.0;
    E[q] = I + A * K[q] + B * K2[q];
    V[q] = I + B * K[q] + C * K2[q];
  }
  mul3(E, X, Xo);
#pragma unroll
  for (int r = 0; r < 3; r++)
    Xo[9 + r] = (E[r * 3] * X[9] + E[r * 3 + 1] * X[10] + E[r * 3 + 2] * X[11]) +
                (V[r * 3] * xi[0] + V[r * 3 + 1] * xi[1] + V[r * 3 + 2] * xi[2]);
}

// One thread per edge.  MODE 0: s, w, cost term.  MODE 1: also B = w J_i^T Omega J_i (packed upper) and gv = w J_i^T Omega e.
template <int MODE>
__global__ void __launch_bounds__(128) k_pg_edges(PgEdgeArgs a) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.E) return;
  const int2 ij = a.ij[k];
  const double* Xi = a.X + (size_t)ij.x * 12;
  const double* Xj = a.X + (size_t)ij.y * 12;
  const double* Z = a.Z + (size_t)k * 12;
  double Rjt[9], RM[9], RE[9], tE[3], e[6];
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int q = 0; q < 3; q++) Rjt[r * 3 + q] = Xj[q * 3 + r];
  mul3(Rjt, Xi, RM);
  double dt[3] = {Xi[9] - Xj[9], Xi[10] - Xj[10], Xi[11] - Xj[11]};
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int q = 0; q < 3; q++) RE[r * 3 + q] = RM[r * 3] * Z[q * 3] + RM[r * 3 + 1] * Z[q * 3 + 1] + RM[r * 3 + 2] * Z[q * 3 + 2];
#pragma unroll
  for (int r = 0; r < 3; r++)
    tE[r] = (Rjt[r * 3] * dt[0] + Rjt[r * 3 + 1] * dt[1] + Rjt[r * 3 + 2] * dt[2]) -
            (RE[r * 3] * Z[9] + RE[r * 3 + 1] * Z[10] + RE[r * 3 + 2] * Z[11]);
  pg_log(RE, tE, e);
  const double* O = a.om + (size_t)k * 21;
  double y[6];
#pragma unroll
  for (int r = 0; r < 6; r++) {
    double v = 0.0;
#pragma unroll
    for (int q = 0; q < 6; q++) v += O[pu(r, q)] * e[q];
    y[r] = v;
  }
  double s = 0.0;
#pragma unroll
  for (int r = 0; r < 6; r++) s += e[r] * y[r];
  const double c = a.c[k];
  double w = 1.0, term = s;
  if (c > 0.0) {
    const double c2 = c * c;
    w = 1.0 / (1.0 + s / c2);
    term = c2 * log1p(s / c2);
  }
  a.s[k] = s;
  a.w[k] = w;
  a.term[k] = term;
  if (MODE == 0) return;
  // J_i = [[P, Qb], [0, P]]: P = Ji Rj^T, Qb = Ji ([u]x - Q Ji) Rj^T, u = -Rj^T t_j, Ji / Q at e.
  const double *rho = e, *phi = e + 3;
  double A, Bc, C, D, c2, c3;
  pg_coeffs(sqrt(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2]), A, Bc, C, D, c2, c3);
  double P[9], Rh[9], T1[9], T2[9], Q[9], Ji[9];
  hat3(phi, P);
  hat3(rho, Rh);
  mul3(P, P, T1);
#pragma unroll
  for (int q = 0; q < 9; q++) Ji[q] = ((q % 4 == 0) ? 1.0 : 0.0) - 0.5 * P[q] + D * T1[q];
  {
    double PR[9], RP[9], PRP[9];
    mul3(P, Rh, PR);
    mul3(Rh, P, RP);
    mul3(PR, P, PRP);
    mul3(P, PR, T1);   // P P R
    mul3(RP, P, T2);   // R P P
#pragma unroll
    for (int q = 0; q < 9; q++) Q[q] = 0.5 * Rh[q] + C * (PR[q] + RP[q] + PRP[q]) + c2 * (T1[q] + T2[q] - 3.0 * PRP[q]);
    mul3(PRP, P, T1);  // P R P P
    mul3(P, PRP, T2);  // P P R P
#pragma unroll
    for (int q = 0; q < 9; q++) Q[q] += c3 * (T1[q] + T2[q]);
  }
  double u[3];
#pragma unroll
  for (int r = 0; r < 3; r++) u[r] = -(Rjt[r * 3] * Xj[9] + Rjt[r * 3 + 1] * Xj[10] + Rjt[r * 3 + 2] * Xj[11]);
  hat3(u, T2);
  mul3(Q, Ji, T1);
#pragma unroll
  for (int q = 0; q < 9; q++) T2[q] -= T1[q];  // [u]x - Q Ji
  mul3(Ji, T2, T1);
  double Qb[9];
  mul3(T1, Rjt, Qb);
  mul3(Ji, Rjt, P);
  // column b of J: b < 3 -> (P[:,b], 0), b >= 3 -> (Qb[:,b-3], P[:,b-3])
#define PG_J(r, b) ((b) < 3 ? ((r) < 3 ? P[(r) * 3 + (b)] : 0.0) : ((r) < 3 ? Qb[(r) * 3 + (b) - 3] : P[((r) - 3) * 3 + (b) - 3]))
  double* Bo = a.B + (size_t)k * 21;
#pragma unroll
  for (int b = 0; b < 6; b++) {
    double v[6];
#pragma unroll
    for (int r = 0; r < 6; r++) {
      double acc = 0.0;
#pragma unroll
      for (int q = 0; q < 6; q++) acc += O[pu(r, q)] * PG_J(q, b);
      v[r] = acc;
    }
#pragma unroll
    for (int aa = 0; aa <= b; aa++) {
      double acc = 0.0;
#pragma unroll
      for (int r = 0; r < 6; r++) acc += PG_J(r, aa) * v[r];
      Bo[pu(aa, b)] = w * acc;
    }
  }
  double* go = a.gv + (size_t)k * 6;
#pragma unroll
  for (int aa = 0; aa < 6; aa++) {
    double acc = 0.0;
#pragma unroll
    for (int r = 0; r < 6; r++) acc += PG_J(r, aa) * y[r];
    go[aa] = w * acc;
  }
#undef PG_J
}

// One block of 256 threads: thread t reduces elements [256 t, 256 t + 256) in order, thread 0 the 256 partials in order.
// OP 0: sum, OP 1: max.  n <= 65536.
template <int OP>
__global__ void __launch_bounds__(256) k_pg_reduce(const double* a, int n, double* out) {
  __shared__ double part[256];
  const int t = threadIdx.x;
  double acc = 0.0;
  for (int q = t * PG_CHUNK; q < n && q < (t + 1) * PG_CHUNK; q++) acc = OP == 0 ? acc + a[q] : fmax(acc, a[q]);
  part[t] = acc;
  __syncthreads();
  if (t == 0) {
    double r = 0.0;
    for (int q = 0; q < 256; q++) r = OP == 0 ? r + part[q] : fmax(r, part[q]);
    *out = r;
  }
}

struct PgNodeArgs {
  int nF;
  const int* rowptr;
  const int2* ent;     // (2 edge + side, other endpoint's free index or -1)
  const double *B, *gv;
  double *D, *g, *maxd; // phase 0 outputs
  double *Dd, *L;       // phase 1 outputs
  double* info;         // [6] max diagonal of A; [5] set to 1 when a damped block is not positive definite
  double lam;
};

// PHASE 0: D_n = sum of the incident blocks, g_n = sum of +-gv, in CSR order.  PHASE 1: damping and Cholesky.
template <int PHASE>
__global__ void __launch_bounds__(128) k_pg_nodes(PgNodeArgs a) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= a.nF) return;
  if (PHASE == 0) {
    double D[21], g[6];
#pragma unroll
    for (int q = 0; q < 21; q++) D[q] = 0.0;
#pragma unroll
    for (int q = 0; q < 6; q++) g[q] = 0.0;
    for (int p = a.rowptr[f]; p < a.rowptr[f + 1]; p++) {
      const int2 en = a.ent[p];
      const int k = en.x >> 1;
      const double* B = a.B + (size_t)k * 21;
      const double* gv = a.gv + (size_t)k * 6;
#pragma unroll
      for (int q = 0; q < 21; q++) D[q] += B[q];
      if (en.x & 1) {
#pragma unroll
        for (int q = 0; q < 6; q++) g[q] -= gv[q];
      } else {
#pragma unroll
        for (int q = 0; q < 6; q++) g[q] += gv[q];
      }
    }
    double m = D[pu(0, 0)];
#pragma unroll
    for (int q = 0; q < 21; q++) a.D[(size_t)f * 21 + q] = D[q];
#pragma unroll
    for (int q = 0; q < 6; q++) {
      a.g[(size_t)f * 6 + q] = g[q];
      m = fmax(m, D[pu(q, q)]);
    }
    a.maxd[f] = m;
  } else {
    double M[21];
    const double floor_d = 1e-9 * a.info[6];
#pragma unroll
    for (int q = 0; q < 21; q++) M[q] = a.D[(size_t)f * 21 + q];
#pragma unroll
    for (int q = 0; q < 6; q++) M[pu(q, q)] += a.lam * fmax(M[pu(q, q)], floor_d);
#pragma unroll
    for (int q = 0; q < 21; q++) a.Dd[(size_t)f * 21 + q] = M[q];
    double L[21];
    bool ok = true;
#pragma unroll
    for (int r = 0; r < 6; r++) {
#pragma unroll
      for (int c = 0; c <= r; c++) {
        double v = M[pu(r, c)];
#pragma unroll
        for (int q = 0; q < c; q++) v -= L[pl(r, q)] * L[pl(c, q)];
        if (r == c) {
          ok = ok && v > 0.0;
          L[pl(r, r)] = sqrt(fmax(v, 0.0));
        } else {
          L[pl(r, c)] = ok ? v / L[pl(c, c)] : 0.0;
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 21; q++) a.L[(size_t)f * 21 + q] = L[q];
    if (!ok) a.info[5] = 1.0;
  }
}

struct PgPcgArgs {
  int nF, nchunks, max_cg;
  double tol;
  const int* rowptr;
  const int2* ent;
  const double *B, *Dd, *L, *g;
  double *x, *r, *z, *p, *q;
  double *part_pq, *part_rr, *part_rz;  // [nchunks]
  double* info;                         // [3] iterations, [4] final relative residual; [5] checked first
};

__device__ __forceinline__ void pg_chol_solve(const double* L, const double* b, double* z) {
  double y[6];
#pragma unroll
  for (int r = 0; r < 6; r++) {
    double v = b[r];
#pragma unroll
    for (int q = 0; q < r; q++) v -= L[pl(r, q)] * y[q];
    y[r] = v / L[pl(r, r)];
  }
#pragma unroll
  for (int r = 5; r >= 0; r--) {
    double v = y[r];
#pragma unroll
    for (int q = r + 1; q < 6; q++) v -= L[pl(q, r)] * z[q];
    z[r] = v / L[pl(r, r)];
  }
}

__device__ __forceinline__ double pg_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double pg_chunk_total(const double* part, int n) {
  double s = 0.0;
  for (int c = 0; c < n; c++) s += part[c];
  return s;
}

// Every CG iteration of one LM step.  Free node f = 32 c + lane belongs to chunk c, handled by warp c mod (grid warps).
__global__ void __launch_bounds__(PG_CG_BLOCK) k_pg_pcg(PgPcgArgs a) {
  cg::grid_group grid = cg::this_grid();
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  if (a.info[5] != 0.0) {  // a damped block is not positive definite: no step
    for (int c = gw; c < a.nchunks; c += nw) {
      const int f = c * 32 + lane;
      if (f < a.nF)
#pragma unroll
        for (int q = 0; q < 6; q++) a.x[(size_t)f * 6 + q] = 0.0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) a.info[3] = a.info[4] = 0.0;
    return;
  }
  for (int c = gw; c < a.nchunks; c += nw) {
    const int f = c * 32 + lane;
    double rr = 0.0, rz = 0.0;
    if (f < a.nF) {
      double r[6], z[6];
#pragma unroll
      for (int q = 0; q < 6; q++) r[q] = -a.g[(size_t)f * 6 + q];
      pg_chol_solve(a.L + (size_t)f * 21, r, z);
#pragma unroll
      for (int q = 0; q < 6; q++) {
        a.x[(size_t)f * 6 + q] = 0.0;
        a.r[(size_t)f * 6 + q] = r[q];
        a.z[(size_t)f * 6 + q] = z[q];
        a.p[(size_t)f * 6 + q] = z[q];
        rr += r[q] * r[q];
        rz += r[q] * z[q];
      }
    }
    rr = pg_warp_sum(rr);
    rz = pg_warp_sum(rz);
    if (lane == 0) {
      a.part_rr[c] = rr;
      a.part_rz[c] = rz;
    }
  }
  grid.sync();
  const double rr0 = pg_chunk_total(a.part_rr, a.nchunks);
  double rr = rr0, rz = pg_chunk_total(a.part_rz, a.nchunks);
  const double stop = a.tol * sqrt(rr0);
  int it = 0;
  while (it < a.max_cg && !(sqrt(rr) <= stop)) {
    for (int c = gw; c < a.nchunks; c += nw) {
      const int f = c * 32 + lane;
      double pq = 0.0;
      if (f < a.nF) {
        double pf[6], qv[6];
        const double* Dd = a.Dd + (size_t)f * 21;
#pragma unroll
        for (int q = 0; q < 6; q++) pf[q] = a.p[(size_t)f * 6 + q];
#pragma unroll
        for (int rw = 0; rw < 6; rw++) {
          double v = 0.0;
#pragma unroll
          for (int q = 0; q < 6; q++) v += Dd[pu(rw, q)] * pf[q];
          qv[rw] = v;
        }
        for (int e = a.rowptr[f]; e < a.rowptr[f + 1]; e++) {
          const int2 en = a.ent[e];
          if (en.y < 0) continue;
          const double* B = a.B + (size_t)(en.x >> 1) * 21;
          const double* po = a.p + (size_t)en.y * 6;
          double pm[6];
#pragma unroll
          for (int q = 0; q < 6; q++) pm[q] = po[q];
#pragma unroll
          for (int rw = 0; rw < 6; rw++) {
            double v = 0.0;
#pragma unroll
            for (int q = 0; q < 6; q++) v += B[pu(rw, q)] * pm[q];
            qv[rw] -= v;
          }
        }
#pragma unroll
        for (int q = 0; q < 6; q++) {
          a.q[(size_t)f * 6 + q] = qv[q];
          pq += pf[q] * qv[q];
        }
      }
      pq = pg_warp_sum(pq);
      if (lane == 0) a.part_pq[c] = pq;
    }
    grid.sync();
    const double pq = pg_chunk_total(a.part_pq, a.nchunks);
    if (!(pq > 0.0)) break;
    const double alpha = rz / pq;
    for (int c = gw; c < a.nchunks; c += nw) {
      const int f = c * 32 + lane;
      double prr = 0.0, prz = 0.0;
      if (f < a.nF) {
        double r[6], z[6];
#pragma unroll
        for (int q = 0; q < 6; q++) {
          a.x[(size_t)f * 6 + q] += alpha * a.p[(size_t)f * 6 + q];
          r[q] = a.r[(size_t)f * 6 + q] - alpha * a.q[(size_t)f * 6 + q];
          a.r[(size_t)f * 6 + q] = r[q];
        }
        pg_chol_solve(a.L + (size_t)f * 21, r, z);
#pragma unroll
        for (int q = 0; q < 6; q++) {
          a.z[(size_t)f * 6 + q] = z[q];
          prr += r[q] * r[q];
          prz += r[q] * z[q];
        }
      }
      prr = pg_warp_sum(prr);
      prz = pg_warp_sum(prz);
      if (lane == 0) {
        a.part_rr[c] = prr;
        a.part_rz[c] = prz;
      }
    }
    grid.sync();
    rr = pg_chunk_total(a.part_rr, a.nchunks);
    const double rzn = pg_chunk_total(a.part_rz, a.nchunks);
    const double beta = rzn / rz;
    rz = rzn;
    for (int c = gw; c < a.nchunks; c += nw) {
      const int f = c * 32 + lane;
      if (f < a.nF)
#pragma unroll
        for (int q = 0; q < 6; q++) a.p[(size_t)f * 6 + q] = a.z[(size_t)f * 6 + q] + beta * a.p[(size_t)f * 6 + q];
    }
    grid.sync();  // p complete before the next SpMV reads neighbours
    it++;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.info[3] = (double)it;
    a.info[4] = rr0 > 0.0 ? sqrt(rr / rr0) : 0.0;
  }
}

// Trial poses: free nodes exp(x_f) X, fixed nodes copied bit for bit; per free node max |rho|, max |phi|.
__global__ void __launch_bounds__(128) k_pg_step(int N, const int* free_of, const double* x, const double* X, double* Xt,
                                                 double* mrho, double* mphi) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const int f = free_of[n];
  const double* Xn = X + (size_t)n * 12;
  double* Xo = Xt + (size_t)n * 12;
  if (f < 0) {
#pragma unroll
    for (int q = 0; q < 12; q++) Xo[q] = Xn[q];
    return;
  }
  double xi[6], Xi[12], Xr[12];
#pragma unroll
  for (int q = 0; q < 6; q++) xi[q] = x[(size_t)f * 6 + q];
#pragma unroll
  for (int q = 0; q < 12; q++) Xi[q] = Xn[q];
  pg_update(xi, Xi, Xr);
#pragma unroll
  for (int q = 0; q < 12; q++) Xo[q] = Xr[q];
  mrho[f] = fmax(fmax(fabs(xi[0]), fabs(xi[1])), fabs(xi[2]));
  mphi[f] = fmax(fmax(fabs(xi[3]), fabs(xi[4])), fabs(xi[5]));
}

bool pg_finite(const double* a, int n) {
  for (int q = 0; q < n; q++)
    if (!std::isfinite(a[q])) return false;
  return true;
}

bool pg_orthonormal(const double* R) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 3; c++) {
      const double v = R[r] * R[c] + R[3 + r] * R[3 + c] + R[6 + r] * R[6 + c] - (r == c ? 1.0 : 0.0);
      if (!(std::fabs(v) <= 1e-6)) return false;
    }
  return true;
}

int pg_find(std::vector<int>& par, int a) {
  while (par[a] != a) {
    par[a] = par[par[a]];
    a = par[a];
  }
  return a;
}

size_t pg_al(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace

extern "C" int tslam_pose_graph_solve(int32_t N, const double* R, const double* T, const uint8_t* fixed, int32_t E,
                                      const int32_t* ij, const double* ZR, const double* ZT, const double* omega,
                                      const double* cauchy, const tslam_pg_params_t* prm, double* R_out, double* T_out,
                                      double* chi2, double* weight, double* f3, int64_t* info5, void* stream) {
  static const char* fn = "tslam_pose_graph_solve";
  if (N < 2 || N > PG_MAX_N || E < 1 || E > PG_MAX_E) {
    ts_set_error("%s: n_nodes %d outside [2, %d] or n_edges %d outside [1, %d]", fn, N, PG_MAX_N, E, PG_MAX_E);
    return TSLAM_E_INVALID;
  }
  if (!R || !T || !fixed || !ij || !ZR || !ZT || !omega || !cauchy || !prm || !R_out || !T_out || !chi2 || !weight || !f3 ||
      !info5) {
    ts_set_error("%s: NULL array or params", fn);
    return TSLAM_E_INVALID;
  }
  const tslam_pg_params_t P = *prm;
  if (!(std::isfinite(P.eps_t) && P.eps_t >= 0.0 && std::isfinite(P.eps_r) && P.eps_r >= 0.0 && std::isfinite(P.cg_tol) &&
        P.cg_tol >= 0.0 && P.cg_tol < 1.0) ||
      P.max_iters < 0 || P.max_iters > TSLAM_PG_MAX_ITERS || P.max_cg < 1 || P.max_cg > TSLAM_PG_MAX_ITERS || P.pcg_grid < 0) {
    ts_set_error("%s: solver parameters out of range (eps_t, eps_r finite >= 0; cg_tol in [0, 1); max_iters in [0, %d]; "
                 "max_cg in [1, %d]; pcg_grid >= 0)", fn, TSLAM_PG_MAX_ITERS, TSLAM_PG_MAX_ITERS);
    return TSLAM_E_INVALID;
  }
  for (int n = 0; n < N; n++) {
    if (!pg_finite(R + (size_t)n * 9, 9) || !pg_finite(T + (size_t)n * 3, 3)) {
      ts_set_error("%s: node %d: pose not finite", fn, n);
      return TSLAM_E_INVALID;
    }
    if (!pg_orthonormal(R + (size_t)n * 9)) {
      ts_set_error("%s: node %d: rotation not orthonormal (max |R^T R - I| > 1e-6)", fn, n);
      return TSLAM_E_INVALID;
    }
  }
  for (int k = 0; k < E; k++) {
    const int i = ij[2 * k], j = ij[2 * k + 1];
    if (i < 0 || i >= N || j < 0 || j >= N || i == j) {
      ts_set_error("%s: edge %d: endpoints (%d, %d) out of range or equal", fn, k, i, j);
      return TSLAM_E_INVALID;
    }
    const double* O = omega + (size_t)k * 36;
    bool fin = pg_finite(ZR + (size_t)k * 9, 9) && pg_finite(ZT + (size_t)k * 3, 3) && std::isfinite(cauchy[k]);
    for (int r = 0; r < 6; r++)
      for (int c = r; c < 6; c++) fin = fin && std::isfinite(O[r * 6 + c]);
    if (!fin) {
      ts_set_error("%s: edge %d: measurement, information or Cauchy scale not finite", fn, k);
      return TSLAM_E_INVALID;
    }
    if (cauchy[k] < 0.0) {
      ts_set_error("%s: edge %d: Cauchy scale %g < 0", fn, k, cauchy[k]);
      return TSLAM_E_INVALID;
    }
    if (!pg_orthonormal(ZR + (size_t)k * 9)) {
      ts_set_error("%s: edge %d: rotation not orthonormal (max |R^T R - I| > 1e-6)", fn, k);
      return TSLAM_E_INVALID;
    }
    for (int r = 0; r < 6; r++)
      if (O[r * 7] < 0.0) {
        ts_set_error("%s: edge %d: negative diagonal entry of the information matrix", fn, k);
        return TSLAM_E_INVALID;
      }
  }
  std::vector<int> par(N);
  for (int n = 0; n < N; n++) par[n] = n;
  for (int k = 0; k < E; k++) par[pg_find(par, ij[2 * k])] = pg_find(par, ij[2 * k + 1]);
  std::vector<char> anchored(N, 0);
  for (int n = 0; n < N; n++)
    if (fixed[n]) anchored[pg_find(par, n)] = 1;
  for (int n = 0; n < N; n++)
    if (!anchored[pg_find(par, n)]) {
      ts_set_error("%s: node %d: its connected component has no fixed node (no gauge)", fn, n);
      return TSLAM_E_INVALID;
    }

  // ---- host set-up: free index, incidence CSR (a free node's edges ascending), packed inputs
  std::vector<int> free_of(N, -1), free_nodes;
  for (int n = 0; n < N; n++)
    if (!fixed[n]) {
      free_of[n] = (int)free_nodes.size();
      free_nodes.push_back(n);
    }
  const int nF = (int)free_nodes.size();
  std::vector<int> rowptr(nF + 1, 0);
  for (int k = 0; k < E; k++) {
    if (free_of[ij[2 * k]] >= 0) rowptr[free_of[ij[2 * k]] + 1]++;
    if (free_of[ij[2 * k + 1]] >= 0) rowptr[free_of[ij[2 * k + 1]] + 1]++;
  }
  for (int f = 0; f < nF; f++) rowptr[f + 1] += rowptr[f];
  const int nnz = rowptr[nF];
  std::vector<int2> ent(nnz > 0 ? nnz : 1);
  {
    std::vector<int> fill(rowptr.begin(), rowptr.end() - 1);
    for (int k = 0; k < E; k++) {
      const int fi = free_of[ij[2 * k]], fj = free_of[ij[2 * k + 1]];
      if (fi >= 0) ent[fill[fi]++] = make_int2(2 * k, fj);
      if (fj >= 0) ent[fill[fj]++] = make_int2(2 * k + 1, fi);
    }
  }
  std::vector<double> hX((size_t)N * 12), hZ((size_t)E * 12), hO((size_t)E * 21);
  for (int n = 0; n < N; n++) {
    for (int q = 0; q < 9; q++) hX[(size_t)n * 12 + q] = R[(size_t)n * 9 + q];
    for (int q = 0; q < 3; q++) hX[(size_t)n * 12 + 9 + q] = T[(size_t)n * 3 + q];
  }
  for (int k = 0; k < E; k++) {
    for (int q = 0; q < 9; q++) hZ[(size_t)k * 12 + q] = ZR[(size_t)k * 9 + q];
    for (int q = 0; q < 3; q++) hZ[(size_t)k * 12 + 9 + q] = ZT[(size_t)k * 3 + q];
    for (int r = 0; r < 6; r++)
      for (int c = r; c < 6; c++) hO[(size_t)k * 21 + pu(r, c)] = omega[(size_t)k * 36 + r * 6 + c];
  }
  const int nchunks = (nF + 31) / 32, nFa = nF > 0 ? nF : 1, nca = nchunks > 0 ? nchunks : 1;

  // ---- one stream-ordered scratch allocation
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += pg_al(bytes); return o; };
  const size_t oX = take((size_t)N * 96), oXt = take((size_t)N * 96), oIJ = take((size_t)E * 8), oZ = take((size_t)E * 96),
               oO = take((size_t)E * 168), oC = take((size_t)E * 8), oS = take((size_t)E * 8), oW = take((size_t)E * 8),
               oTm = take((size_t)E * 8), oB = take((size_t)E * 168), oGv = take((size_t)E * 48),
               oRp = take((size_t)(nF + 1) * 4), oEnt = take((size_t)(nnz > 0 ? nnz : 1) * 8), oFo = take((size_t)N * 4),
               oD = take((size_t)nFa * 168), oDd = take((size_t)nFa * 168), oL = take((size_t)nFa * 168),
               oG = take((size_t)nFa * 48), oV = take((size_t)nFa * 48 * 5), oMd = take((size_t)nFa * 8),
               oMr = take((size_t)nFa * 8), oMp = take((size_t)nFa * 8), oPt = take((size_t)nca * 24), oInfo = take(64);
  cudaStream_t st = (cudaStream_t)stream;
  char* w = nullptr;
  TS_CUDA(cudaMallocAsync((void**)&w, off, st));
  double* dX = (double*)(w + oX);
  double* dXt = (double*)(w + oXt);
  double* info = (double*)(w + oInfo);
  PgEdgeArgs ea{E, (const int2*)(w + oIJ), dX, (const double*)(w + oZ), (const double*)(w + oO), (const double*)(w + oC),
                (double*)(w + oS), (double*)(w + oW), (double*)(w + oTm), (double*)(w + oB), (double*)(w + oGv)};
  PgNodeArgs na{nF, (const int*)(w + oRp), (const int2*)(w + oEnt), ea.B, ea.gv, (double*)(w + oD), (double*)(w + oG),
                (double*)(w + oMd), (double*)(w + oDd), (double*)(w + oL), info, 0.0};
  double* V = (double*)(w + oV);
  PgPcgArgs pa{nF, nchunks, P.max_cg, P.cg_tol, na.rowptr, na.ent, ea.B, na.Dd, na.L, na.g,
               V, V + (size_t)nFa * 6, V + (size_t)nFa * 12, V + (size_t)nFa * 18, V + (size_t)nFa * 24,
               (double*)(w + oPt), (double*)(w + oPt) + nca, (double*)(w + oPt) + 2 * nca, info};
  double* mrho = (double*)(w + oMr);
  double* mphi = (double*)(w + oMp);
  const int eb = (E + 127) / 128, fb = (nFa + 127) / 128, nb = (N + 127) / 128;
  double hinfo[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  double F0 = 0.0, F = 0.0, cg_res = 0.0;
  int64_t evals = 0, accepted = 0, cg_iters = 0;
  int status = 1;  // max_iters
  int grid = 1;
  cudaError_t e = cudaSuccess;
#define PG_TRY(x)                     \
  do {                                \
    if (e == cudaSuccess) e = (x);    \
  } while (0)
#define PG_KCHECK() PG_TRY(cudaGetLastError())
  PG_TRY(cudaMemcpyAsync(dX, hX.data(), (size_t)N * 96, cudaMemcpyHostToDevice, st));
  PG_TRY(cudaMemcpyAsync((void*)ea.ij, ij, (size_t)E * 8, cudaMemcpyHostToDevice, st));
  PG_TRY(cudaMemcpyAsync((void*)ea.Z, hZ.data(), (size_t)E * 96, cudaMemcpyHostToDevice, st));
  PG_TRY(cudaMemcpyAsync((void*)ea.om, hO.data(), (size_t)E * 168, cudaMemcpyHostToDevice, st));
  PG_TRY(cudaMemcpyAsync((void*)ea.c, cauchy, (size_t)E * 8, cudaMemcpyHostToDevice, st));
  PG_TRY(cudaMemcpyAsync((void*)na.rowptr, rowptr.data(), (size_t)(nF + 1) * 4, cudaMemcpyHostToDevice, st));
  PG_TRY(cudaMemcpyAsync((void*)na.ent, ent.data(), (size_t)ent.size() * 8, cudaMemcpyHostToDevice, st));
  PG_TRY(cudaMemcpyAsync(w + oFo, free_of.data(), (size_t)N * 4, cudaMemcpyHostToDevice, st));
  PG_TRY(cudaMemsetAsync(info, 0, 64, st));
  if (e == cudaSuccess && nF > 0) {
    int dev = 0, sms = 0, per_sm = 0;
    PG_TRY(cudaGetDevice(&dev));
    PG_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PG_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pg_pcg, PG_CG_BLOCK, 0));
    const int need = (nchunks * 32 + PG_CG_BLOCK - 1) / PG_CG_BLOCK, most = per_sm * sms;
    grid = P.pcg_grid > 0 ? P.pcg_grid : need;
    if (grid > most) grid = most;
    if (grid < 1) grid = 1;
  }
  // linearise at X: terms, blocks, gradient pieces, node sums, max diagonal
  auto linearise = [&]() {
    ea.X = dX;
    k_pg_edges<1><<<eb, 128, 0, st>>>(ea);
    PG_KCHECK();
    k_pg_reduce<0><<<1, 256, 0, st>>>(ea.term, E, info);
    PG_KCHECK();
    if (nF > 0) {
      k_pg_nodes<0><<<fb, 128, 0, st>>>(na);
      PG_KCHECK();
      k_pg_reduce<1><<<1, 256, 0, st>>>(na.maxd, nF, info + 6);
      PG_KCHECK();
    }
  };
  linearise();
  PG_TRY(cudaMemcpyAsync(hinfo, info, 64, cudaMemcpyDeviceToHost, st));
  PG_TRY(cudaStreamSynchronize(st));
  F0 = F = 0.5 * hinfo[0];
  double lam = 1e-4;
  while (e == cudaSuccess && evals < P.max_iters) {
    na.lam = lam;
    if (nF > 0) {
      k_pg_nodes<1><<<fb, 128, 0, st>>>(na);
      PG_KCHECK();
      void* args[] = {&pa};
      PG_TRY(cudaLaunchCooperativeKernel((void*)k_pg_pcg, dim3(grid), dim3(PG_CG_BLOCK), args, 0, st));
    }
    k_pg_step<<<nb, 128, 0, st>>>(N, (const int*)(w + oFo), pa.x, dX, dXt, mrho, mphi);
    PG_KCHECK();
    ea.X = dXt;
    k_pg_edges<0><<<eb, 128, 0, st>>>(ea);
    PG_KCHECK();
    k_pg_reduce<0><<<1, 256, 0, st>>>(ea.term, E, info);
    PG_KCHECK();
    if (nF > 0) {
      k_pg_reduce<1><<<1, 256, 0, st>>>(mrho, nF, info + 1);
      PG_KCHECK();
      k_pg_reduce<1><<<1, 256, 0, st>>>(mphi, nF, info + 2);
      PG_KCHECK();
    }
    PG_TRY(cudaMemcpyAsync(hinfo, info, 64, cudaMemcpyDeviceToHost, st));
    PG_TRY(cudaStreamSynchronize(st));
    if (e != cudaSuccess) break;
    evals++;
    cg_iters += (int64_t)hinfo[3];
    cg_res = std::fmax(cg_res, hinfo[4]);
    if (hinfo[5] != 0.0) {
      status = 3;  // a damped diagonal block is not positive definite
      break;
    }
    const double Ft = 0.5 * hinfo[0];
    if (Ft < F) {
      std::swap(dX, dXt);
      F = Ft;
      lam /= 10.0;
      accepted++;
      if (hinfo[1] < P.eps_t && hinfo[2] < P.eps_r) {
        status = 0;
        break;
      }
      linearise();
    } else {
      lam *= 10.0;
      if (lam > 1e16) {
        status = 2;
        break;
      }
    }
  }
  // s, w at the final poses
  ea.X = dX;
  k_pg_edges<0><<<eb, 128, 0, st>>>(ea);
  PG_KCHECK();
  PG_TRY(cudaMemcpyAsync(hX.data(), dX, (size_t)N * 96, cudaMemcpyDeviceToHost, st));
  std::vector<double> hs((size_t)E), hw((size_t)E);
  PG_TRY(cudaMemcpyAsync(hs.data(), ea.s, (size_t)E * 8, cudaMemcpyDeviceToHost, st));
  PG_TRY(cudaMemcpyAsync(hw.data(), ea.w, (size_t)E * 8, cudaMemcpyDeviceToHost, st));
  PG_TRY(cudaStreamSynchronize(st));
#undef PG_TRY
#undef PG_KCHECK
  const cudaError_t fe = cudaFreeAsync(w, st);
  if (e == cudaSuccess) e = fe;
  if (e != cudaSuccess) {
    ts_set_error("%s: %s", fn, cudaGetErrorString(e));
    return TSLAM_E_CUDA;
  }
  for (int n = 0; n < N; n++) {
    for (int q = 0; q < 9; q++) R_out[(size_t)n * 9 + q] = fixed[n] ? R[(size_t)n * 9 + q] : hX[(size_t)n * 12 + q];
    for (int q = 0; q < 3; q++) T_out[(size_t)n * 3 + q] = fixed[n] ? T[(size_t)n * 3 + q] : hX[(size_t)n * 12 + 9 + q];
  }
  for (int k = 0; k < E; k++) {
    chi2[k] = hs[k];
    weight[k] = hw[k];
  }
  f3[0] = F0;
  f3[1] = F;
  f3[2] = cg_res;
  info5[0] = evals;
  info5[1] = accepted;
  info5[2] = cg_iters;
  info5[3] = status == 0 ? 1 : 0;
  info5[4] = status;
  return TSLAM_OK;
}
