// libtslam.so - the plan rule of the incremental global fusions (host): what an update does with each submap.
// tslam_tsdf_fuse_update (tslam_fuse.cu, single and tiled maps) and tslam_octo_fuse_update (tslam_octo_fuse.cu) share it,
// so `include`, `tolerance` and the full-update reasons mean the same thing for both map types.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

// full-update reasons (stats8[0]; 0 = incremental)
// 7, 8: tiled updates only (tslam_tsdf_fuse_update_tiled_*)
enum { FZ_INCR = 0, FZ_FIRST = 1, FZ_ASKED = 2, FZ_OTHER_SRC = 3, FZ_DST_WRITTEN = 4, FZ_CONTENT = 5, FZ_COST = 6, FZ_CUTS = 7,
       FZ_INVALID = 8 };
enum { FZ_NONE = 0, FZ_ADD, FZ_REMOVE, FZ_MOVE, FZ_KEEP };  // what an update does with a submap

struct FzJob {        // one placement of one submap: sign +1 adds, -1 removes
  float R[9], T[3];
  int sign, pad;
};
struct FzSub {        // what a submap contributes to dst
  int fused;          // 1: its voxels are in dst, at (R, T)
  float R[9], T[3];
  unsigned long long ver;  // src content version at that time
  int nblk;           // its source blocks then
};
struct FzPlan {        // one update, from its plan to its record
  int reason;         // FZ_*
  bool full;
  std::vector<unsigned char> want, act;  // per submap: included with source blocks; FZ_NONE .. FZ_KEEP
  std::vector<int> nblk;
  std::vector<float> rad, pR, pT;        // radius, dst pose table
  long long n_add, n_move, n_remove, n_tol, cost, cost_full;  // cost: source blocks an incremental update splats
  unsigned long long ghosts;             // dst ghost blocks (TSDF)
};

// rotation angle of R0^T R (row-major 3x3), in double
static inline double fz_angle(const float* R0, const float* R) {
  double tr = 0.0;
  for (int i = 0; i < 3; i++)
    for (int k = 0; k < 3; k++) tr += (double)R0[3 * k + i] * (double)R[3 * k + i];  // trace(R0^T R) = sum R0_ki R_ki
  double c = (tr - 1.0) * 0.5;
  c = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);
  return std::acos(c);
}

// The per-submap decisions of an update, from P.nblk (source blocks per submap), P.rad (radius of each submap's blocks
// about its origin), P.pR / P.pT (dst's pose table), the records `sub` of the last update and src's content versions.
// `reason` is the full-update reason found from the handles; when it is FZ_INCR the actions of an incremental update
// are planned: unchanged or moved within tolerance (|T - T0| + angle(R0^T R) r_s <= tolerance; 0: iff the pose bits
// are equal) -> KEEP, newly included -> ADD, excluded or now empty -> REMOVE, moved -> MOVE.  A fused submap whose
// content changed makes the update full (FZ_CONTENT).  Returns the reason; the cost rule is the caller's (fz_settle).
static inline int fz_decide(FzPlan& P, const std::vector<FzSub>& sub, const unsigned long long* content_ver, const uint8_t* include,
                            float tolerance, int reason) {
  const int S = (int)P.nblk.size();
  P.want.assign(S, 0);
  P.act.assign(S, FZ_NONE);
  P.n_add = P.n_move = P.n_remove = P.n_tol = P.cost = P.cost_full = 0;
  const std::vector<int>& nblk = P.nblk;
  for (int s = 0; s < S; s++) {
    const bool want = (!include || include[s]) && nblk[s] > 0;
    P.want[s] = want;
    if (want) P.cost_full += nblk[s];
    if (reason != FZ_INCR) continue;
    const FzSub& r = sub[s];
    if (!r.fused) {
      if (want) { P.act[s] = FZ_ADD; P.cost += nblk[s]; }
      continue;
    }
    if (r.ver != content_ver[s]) { reason = FZ_CONTENT; continue; }  // its old content is gone: cannot be subtracted
    if (!want) { P.act[s] = FZ_REMOVE; P.cost += r.nblk; continue; }
    const float* R = &P.pR[(size_t)9 * s];
    const float* T = &P.pT[(size_t)3 * s];
    if (!memcmp(R, r.R, 36) && !memcmp(T, r.T, 12)) { P.act[s] = FZ_KEEP; continue; }
    if (tolerance > 0.0f) {
      const double dx = (double)T[0] - r.T[0], dy = (double)T[1] - r.T[1], dz = (double)T[2] - r.T[2];
      const double move = std::sqrt(dx * dx + dy * dy + dz * dz) + fz_angle(r.R, R) * (double)P.rad[s];
      if (move <= (double)tolerance) { P.act[s] = FZ_KEEP; P.n_tol++; continue; }
    }
    P.act[s] = FZ_MOVE;
    P.cost += r.nblk + nblk[s];
  }
  P.reason = reason;
  return reason;
}

// the update's final reason: a full update adds every included submap
static inline void fz_settle(FzPlan& P, int reason) {
  P.reason = reason;
  P.full = reason != FZ_INCR;
  if (P.full) {
    P.n_tol = 0;
    for (size_t s = 0; s < P.act.size(); s++) P.act[s] = P.want[s] ? FZ_ADD : FZ_NONE;
  }
  P.n_add = P.n_move = P.n_remove = 0;
  for (size_t s = 0; s < P.act.size(); s++) {
    P.n_add += P.act[s] == FZ_ADD;
    P.n_move += P.act[s] == FZ_MOVE;
    P.n_remove += P.act[s] == FZ_REMOVE;
  }
}

// the submaps' records after a successful update (act / pose table / nblk of P, content versions of src)
static inline void fz_record_subs(std::vector<FzSub>& sub, const FzPlan& P, const unsigned long long* content_ver) {
  for (size_t s = 0; s < sub.size(); s++) {
    FzSub& r = sub[s];
    if (P.full) r.fused = 0;
    if (P.act[s] == FZ_REMOVE) r.fused = 0;
    if (P.act[s] == FZ_ADD || P.act[s] == FZ_MOVE) {
      r.fused = 1;
      memcpy(r.R, &P.pR[(size_t)9 * s], 36);
      memcpy(r.T, &P.pT[(size_t)3 * s], 12);
      r.ver = content_ver[s];
      r.nblk = P.nblk[s];
    }
  }
}

// a process-unique handle number (tslam_fuse.cu), for the "other source" rule
unsigned long long ts_next_serial();
