// libtslam.so - occupancy ESDF of a log-odds Octomap (DESIGN.md section 7, "Occupancy ESDF"), kept incrementally.
//
// Per submap, as of one update.  Classes come from the cnt plane: OCC = known and L > l_occ, FREE = known and
// L <= l_occ, UNKNOWN = not known.  A FREE voxel starts at +D, an OCC voxel at -D; UNKNOWN voxels are neither sources
// nor targets.  Relaxation over the known 26-neighbours h of v (edge cost c = vs * {1, sqrt 2, sqrt 3}):
//   FREE v: E(v) = min(E(v), h OCC  ?  c : E(h) + c)
//   OCC  v: E(v) = max(E(v), h FREE ? -c : E(h) - c)
// to the fixed point (f32 min/+ is monotone: unique, independent of the schedule).
//
// The wavefront - full and incremental update, raise and lower waves, queries - is the one both ESDFs share
// (tslam_esdf_common.cuh), on 8^3 blocks (10^3 tiles, 128 threads, 8 CTAs per SM).  This ESDF's rules (EsOcto):
//   targets     FREE (min side) and OCC (max side); every known neighbour is a source, as above
//   detect      (blocks k_octo_lo_apply updated since the last update) a voxel whose class changed -> CHANGED
//   raise test  a target whose value EQUALS the candidate a flagged known neighbour offered it at the old fixed point
//               (old class, old value; the cross-class candidates are the constants +-c)
//   queries     a corner has a value when it was known at the last update
//   extras      the host clears the dirty flags before a full update; an incremental update resets the blocks allocated
//               since the last one to UNKNOWN (prepare)
// DESIGN.md section 7 gives the argument that the lower wave ends at the full recompute's fixed point, bit for bit.
#include <cmath>
#include <cstring>
#include "tslam_esdf_common.cuh"
#include "tslam_traj.cuh"

struct OeAux {
  float* e;            // [max_blocks*512] the field
  unsigned char* cls;  // [max_blocks*512] class at the last update (+ flags during an update)
  int* nbr;            // [max_blocks*27] neighbour block indices (-1 = absent)
  int* epoch;          // [max_blocks] lower wave: last sweep in which the block changed (< -1: block of another submap)
  int* repoch;         // [max_blocks] raise wave: last raise sweep in which the block gained flags (-1: none)
  int* changed;        // [ES_MAX_SWEEPS+2] changed[k] != 0 <=> lower sweep k changed something
  int* rchanged;       // [ES_MAX_SWEEPS+2]
  int* counts;         // [8] changed voxels, suspect voxels, re-initialised blocks, (spare), nb_seen, nb_prev
  int* nb_seen;        // blocks in the pool when the last update ran (bump allocation: higher indices are newer)
  int* nb_prev;        // nb_seen of the update before (incremental update: blocks >= it are new)
};

__device__ __forceinline__ float oe_seed(unsigned char c, float D) { return c == OC_FREE ? D : (c == OC_OCC ? -D : 0.0f); }

// The occupancy ESDF's rules for the shared wavefront (tslam_esdf_common.cuh).  Classes come from the cnt plane at
// init / detect / re-init and from the class bytes in the waves; the field is OeAux::e.
struct EsOcto {
  static constexpr int SHIFT = OC_BSHIFT, THREADS = 128, GRID = 8;
  static constexpr int COUNTS_CLEARED = 4;  // nb_seen and nb_prev are kept
  static constexpr bool GHOSTS = false;
  static constexpr unsigned char NONE = OC_UNK, MIN_SIDE = OC_FREE, MAX_SIDE = OC_OCC;
  OcGrid g;
  OeAux a;
  int submap;
  int l_occ;
  float D, vs;      // seeds +-D, voxel size
  int* esdf_dirty;  // tslam_octo::esdf_dirty
  __device__ float* field() const { return a.e; }
  __device__ int* dirty() const { return esdf_dirty; }
  __device__ float seed(size_t off, unsigned char& c) const {
    c = oc_class(g.cnt[off], l_occ);
    return oe_seed(c, D);
  }
  __device__ bool moved(size_t off, unsigned char oc) const { return oc_class(g.cnt[off], l_occ) != oc; }
  __device__ void stage(size_t off, float& e, unsigned char& c) const {
    c = *(volatile unsigned char*)&a.cls[off];
    e = *(volatile float*)&a.e[off];
  }
  __device__ static bool target(unsigned char c) { return c != OC_UNK; }
  __device__ static bool source(unsigned char, unsigned char h) { return h != OC_UNK; }
  __device__ static bool raise_source(unsigned char h) { return h != OC_UNK; }
  __device__ static float cand_min(unsigned char h, float he, float d) { return h == OC_OCC ? d : he + d; }
  __device__ static float cand_max(unsigned char h, float he, float d) { return h == OC_FREE ? -d : he - d; }
  __device__ static bool valid(unsigned char c) { return c != OC_UNK; }
  __device__ void init_done(int) const {}
  // a block allocated since the last update starts UNKNOWN (whatever its pool slot held before a reset), so detect sees
  // each of its known voxels change
  __device__ void prepare_block(int b, int lane) const {
    if (b >= *a.nb_prev) {
      const size_t base = (size_t)b * OC_B3;
      for (int v = lane; v < OC_B3; v += 32) { a.cls[base + v] = OC_UNK; a.e[base + v] = 0.0f; }
    }
  }
};

// (ijk, E) of every voxel known at the last update, in the blocks that update saw
__global__ void __launch_bounds__(EsOcto::THREADS) k_octo_esdf_gather(OcGrid g, OeAux a, int submap, long long cap, int32_t* idx, float* esdf,
                                                                 unsigned long long* counter) {
  const int nb = min(*a.nb_seen, g.max_blocks);
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap) continue;  // (uniform per CTA)
    const size_t base = (size_t)b * OC_B3;
    for (int v = threadIdx.x; v < OC_B3; v += blockDim.x) {
      const bool want = (a.cls[base + v] & ES_CLS) != OC_UNK;
      const long long row = warp_append_u64(want, counter);
      if (want && row < cap) {
        idx[3 * row] = bx * OC_B + (v >> 6);
        idx[3 * row + 1] = by * OC_B + ((v >> 3) & 7);
        idx[3 * row + 2] = bz * OC_B + (v & 7);
        esdf[row] = a.e[base + v];
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_octo_esdf_query(OcGrid g, OeAux a, int submap, long long n, const float* __restrict__ xyz, float vs,
                                                         float* __restrict__ dist, float* __restrict__ grad, uint8_t* __restrict__ valid) {
  es_query(EsOcto{g, a, submap, 0, 0.0f, vs, nullptr}, n, xyz, dist, grad, valid);
}

// ---- host side -----------------------------------------------------------------------------------------------------
// bytes per pool block: field 2048 + class 512 + neighbour table 108 + epoch, raise epoch, dirty flag 12 = 2680
static size_t oe_bytes(size_t nb) { return nb * (OC_B3 * 5 + 30 * 4) + (2 * (ES_MAX_SWEEPS + 2) + 8) * 4; }

static OeAux oe_aux(tslam_octo* m) {
  const size_t nb = (size_t)m->g.max_blocks;
  OeAux a;
  a.e = (float*)m->esdf_mem;
  a.nbr = (int*)(a.e + nb * OC_B3);
  a.epoch = a.nbr + nb * 27;
  a.repoch = a.epoch + nb;
  // (esdf_dirty = a.repoch + nb)
  a.changed = a.repoch + 2 * nb;
  a.rchanged = a.changed + (ES_MAX_SWEEPS + 2);
  a.counts = a.rchanged + (ES_MAX_SWEEPS + 2);
  a.nb_seen = a.counts + 4;
  a.nb_prev = a.counts + 5;
  a.cls = (unsigned char*)(a.counts + 8);
  return a;
}

static int oe_alloc(tslam_octo* m) {
  if (m->esdf_mem) return TSLAM_OK;
  const size_t bytes = oe_bytes((size_t)m->g.max_blocks);
  TS_CUDA(cudaMalloc(&m->esdf_mem, bytes));
  TS_CUDA(cudaMemset(m->esdf_mem, 0, bytes));
  m->esdf_dirty = oe_aux(m).repoch + m->g.max_blocks;
  return TSLAM_OK;
}

static EsOcto oe_rules(tslam_octo* m, int submap, float D) {
  return EsOcto{m->g, oe_aux(m), submap, m->lo.l_occ, D, m->in.vs, m->esdf_dirty};
}

int oc_esdf_free(tslam_octo* m) {
  if (m->esdf_mem) cudaFree(m->esdf_mem);
  m->esdf_mem = nullptr;
  m->esdf_dirty = nullptr;
  return TSLAM_OK;
}

int oc_esdf_field(tslam_octo* m, int32_t submap, const char* what, OcEsdfField* f) {
  int rc = oc_track_readable(m, m->esdf_track, submap, what, "tslam_octo_esdf_update");
  if (rc) return rc;
  const OeAux a = oe_aux(m);
  f->e = a.e;
  f->cls = a.cls;
  f->nb_seen = a.nb_seen;
  f->D = m->esdf_D;
  f->free_cls = OC_FREE;
  f->cls_mask = ES_CLS;
  return TSLAM_OK;
}

// mode 0 = incremental when the state allows it (same submap and D as the last update, no reset / fusion in between),
// 1 = full recompute.  stats4 (HOST, may be NULL): lower sweeps, raise sweeps (-1 = full), changed voxels, suspect voxels.
extern "C" int tslam_octo_esdf_update(tslam_octo_t* m, int32_t submap, float max_dist, int32_t mode, int32_t* stats4, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  int rc = oc_logodds_submap(m, submap, "tslam_octo_esdf_update", "the occupancy ESDF");
  if (rc) return rc;
  if (!(std::isfinite(max_dist) && max_dist > 0.0f)) {
    ts_set_error("tslam_octo_esdf_update: max_dist must be finite and > 0 (got %g)", (double)max_dist);
    return TSLAM_E_INVALID;
  }
  if (mode != 0 && mode != 1) { ts_set_error("tslam_octo_esdf_update: mode must be 0 (incremental) or 1 (full)"); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  rc = oe_alloc(m);
  if (rc) return rc;
  const EsOcto p = oe_rules(m, submap, max_dist);
  const bool full = mode == 1 || !m->esdf_track.ready || m->esdf_track.submap != submap ||
                    memcmp(&m->esdf_D, &max_dist, sizeof(float)) != 0;
  m->esdf_track.ready = 0;  // until this update has completed
  if (full) TS_CUDA(cudaMemsetAsync(m->esdf_dirty, 0, (size_t)m->g.max_blocks * 4, st));
  else TS_CUDA(cudaMemcpyAsync(p.a.nb_prev, p.a.nb_seen, 4, cudaMemcpyDeviceToDevice, st));
  rc = es_update(m, p, full, st, stats4);
  if (rc) return rc;
  m->esdf_track = OcTrack{1, submap};
  m->esdf_D = max_dist;
  return TSLAM_OK;
}

extern "C" int tslam_octo_esdf_gather(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, float* esdf, int64_t* n_out,
                                      void* stream) {
  if (!m || !n_out || cap < 0 || (cap > 0 && (!idx || !esdf))) return TSLAM_E_INVALID;
  const char* what = "tslam_octo_esdf_gather";
  int rc = oc_track_readable(m, m->esdf_track, submap, what, "tslam_octo_esdf_update");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return oc_counted_gather(m, st, [&](unsigned long long* ctr) {
    k_octo_esdf_gather<<<m->sm_count * EsOcto::GRID, EsOcto::THREADS, 0, st>>>(m->g, oe_aux(m), submap, cap, idx, esdf, ctr);
  }, cap, n_out, what);
}

extern "C" int tslam_octo_esdf_query(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, float* dist, float* grad,
                                     uint8_t* valid, void* stream) {
  if (!m || n < 0 || (n && (!xyz || !dist || !grad || !valid))) return TSLAM_E_INVALID;
  int rc = oc_track_readable(m, m->esdf_track, submap, "tslam_octo_esdf_query", "tslam_octo_esdf_update");
  if (rc || n == 0) return rc;
  k_octo_esdf_query<<<oc_grid(n, 256, m->sm_count * 16), 256, 0, (cudaStream_t)stream>>>(m->g, oe_aux(m), submap, n, xyz, m->in.vs, dist,
                                                                                         grad, valid);
  TS_LAUNCH_CHECK(m);
  return TSLAM_OK;
}

// Trajectories against the occupancy ESDF (tslam_traj.cuh), read as tslam_octo_esdf_query reads it
extern "C" int tslam_octo_esdf_trajectory(tslam_octo_t* m, int32_t submap, int32_t T, const int32_t* n_ctrl, const double* ctrl_in,
                                          const tslam_traj_params_t* params, double* ctrl_out, double* cost, int32_t* info,
                                          void* stream) {
  const char* what = "tslam_octo_esdf_trajectory";
  long long sum_n = 0;
  int rc = tj_check_args(what, T, n_ctrl, ctrl_in, params, ctrl_out, cost, info, &sum_n);
  if (rc) return rc;
  if (!m) { ts_set_error("%s: NULL handle", what); return TSLAM_E_INVALID; }
  rc = oc_track_readable(m, m->esdf_track, submap, what, "tslam_octo_esdf_update");
  if (rc) return rc;
  if (params->clearance > (double)m->esdf_D) {
    ts_set_error("%s: clearance %g above the max_dist %g of the last ESDF update", what, params->clearance, (double)m->esdf_D);
    return TSLAM_E_INVALID;
  }
  const EsOcto p{m->g, oe_aux(m), submap, 0, 0.0f, m->in.vs, nullptr};
  return tj_run(m, p, m->in.vs, what, &m->traj_mem, &m->traj_mem_bytes, T, n_ctrl, sum_n, ctrl_in, params, ctrl_out, cost, info,
                (cudaStream_t)stream);
}
