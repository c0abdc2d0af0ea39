// Pieces shared by the two ESDFs of libtslam.so: the TSDF ESDF (tslam_esdf.cu, 16^3 blocks) and the occupancy ESDF of
// the log-odds Octomap (tslam_octo_esdf.cu, 8^3 blocks).  Both run the same scheme - a block-parallel wavefront with
// per-block epochs, a raise wave flagged by an exact f32 derivation test, re-init, and a lower wave - and answer
// queries with the same trilinear interpolant, so the sweep-group driver and the query arithmetic live here once.
#pragma once
#include "tslam_internal.cuh"

#define ES_GROUP 6       // sweeps enqueued per host synchronisation (full update)
#define ES_MAX_SWEEPS 4096
#define ES_CH 0x40   // class-byte flags of an incremental update: CHANGED (detect) / SUSPECT (raise wave)
#define ES_SU 0x80
#define ES_CLS 0x0F

// One wave (raise or lower) to convergence: sweeps are enqueued in groups, a sweep whose predecessor changed nothing
// returns at once; the host reads ONE flag per group.  Returns the number of sweeps that did something + 1 in *n_out.
// M = tslam_tsdf or tslam_octo (anything with a launch counter).
template <class M, class Launch>
static int es_wave(M* m, cudaStream_t st, int* flags, int group, Launch launch, int* n_out) {
  int sweeps = 0;
  for (;;) {
    for (int q = 0; q < group && sweeps < ES_MAX_SWEEPS; q++) { sweeps++; launch(sweeps); TS_LAUNCH_CHECK(m); }
    int changed = 0;
    TS_CUDA(cudaMemcpyAsync(&changed, flags + sweeps, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
    if (!changed || sweeps >= ES_MAX_SWEEPS) break;
  }
  if (n_out) {
    static int h_changed[ES_MAX_SWEEPS + 2];
    TS_CUDA(cudaMemcpy(h_changed, flags, (size_t)(sweeps + 1) * 4, cudaMemcpyDeviceToHost));
    int k = 1;
    while (k <= sweeps && h_changed[k]) k++;
    *n_out = k;
  }
  return TSLAM_OK;
}

// lerp(a, b, t) = a + t*(b - a), rounded step by step (never contracted to an FMA): tests/esdf_query_reference.py
__device__ __forceinline__ float esq_lerp(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a))); }

// Trilinear interpolant of the 8 corner values e[dx*4 + dy*2 + dz] at fractions (fx, fy, fz) of the cell, and its
// exact partial derivatives (tests/esdf_query_reference.py states the same arithmetic operation by operation).
__device__ __forceinline__ void esq_interp(const float e[8], float fx, float fy, float fz, float vs, float& d, float& gx, float& gy,
                                           float& gz) {
  // dist: along x, then y, then z
  const float c00 = esq_lerp(e[0], e[4], fx), c01 = esq_lerp(e[1], e[5], fx);
  const float c10 = esq_lerp(e[2], e[6], fx), c11 = esq_lerp(e[3], e[7], fx);
  d = esq_lerp(esq_lerp(c00, c10, fy), esq_lerp(c01, c11, fy), fz);
  // d/dx: the four x-differences along y, then z
  const float ax00 = __fsub_rn(e[4], e[0]), ax01 = __fsub_rn(e[5], e[1]), ax10 = __fsub_rn(e[6], e[2]), ax11 = __fsub_rn(e[7], e[3]);
  gx = __fdiv_rn(esq_lerp(esq_lerp(ax00, ax10, fy), esq_lerp(ax01, ax11, fy), fz), vs);
  // d/dy: the four y-differences along x, then z
  const float ay00 = __fsub_rn(e[2], e[0]), ay01 = __fsub_rn(e[3], e[1]), ay10 = __fsub_rn(e[6], e[4]), ay11 = __fsub_rn(e[7], e[5]);
  gy = __fdiv_rn(esq_lerp(esq_lerp(ay00, ay10, fx), esq_lerp(ay01, ay11, fx), fz), vs);
  // d/dz: the four z-differences along x, then y
  const float az00 = __fsub_rn(e[1], e[0]), az01 = __fsub_rn(e[3], e[2]), az10 = __fsub_rn(e[5], e[4]), az11 = __fsub_rn(e[7], e[6]);
  gz = __fdiv_rn(esq_lerp(esq_lerp(az00, az10, fx), esq_lerp(az01, az11, fx), fy), vs);
}
