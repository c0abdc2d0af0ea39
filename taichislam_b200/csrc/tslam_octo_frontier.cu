// libtslam.so - exploration frontiers of a log-odds Octomap (DESIGN.md section 7, "Frontiers of the log-odds Octomap").
//
// Per submap, as of one update.  Classes come from the cnt plane as the occupancy ESDF defines them: OCC = known and
// L > l_occ, FREE = known and L <= l_occ, UNKNOWN = not known (every cell of an absent block).  A frontier voxel is a
// FREE cell with at least one 6-neighbour that is inside the volume and UNKNOWN.  Clusters are the 26-connected
// components of the frontier voxels; a cluster's label is the smallest linear key ((i+hN)*N + (j+hN))*Nz + (k+hNz) of
// its voxels, and clusters are listed in ascending label order.
//
// The frontier set is kept as a 512-bit mask per pool block.  An update runs
//   1. prepare   clear the masks of blocks allocated since the last update, and list the blocks to re-examine: every
//                block of the submap (full), or the blocks k_octo_lo_apply flagged plus their existing face neighbours;
//   2. classify  one CTA per listed block: the block and a one-cell face halo in shared memory -> its new mask;
//   3. compact   popcount per block and an exclusive scan: voxel v of block b has the compact index
//                off[b] + popc(mask bits of b below v), so no per-voxel index plane is needed;
//   4. link      one lane per frontier voxel: union with its 13 backward 26-neighbours that are frontier voxels
//                (lock-free union-find, the larger root hooked under the smaller one by atomicCAS);
//   5. compress  every voxel points at its root; roots take a cluster slot;
//   6. stats     the slot's record by integer atomics, aggregated per root within a warp;
//   7. order     radix sort of the slots by label.
// A cell's status depends only on its class and its 6 neighbours' classes, and a class changes only in the blocks
// k_octo_lo_apply updated, so after 2 the masks equal a full recompute's; 3-7 run over the whole set at every update.
#include <climits>
#include <cstring>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include "tslam_internal.cuh"

#define OF_WORDS 16  // mask words per block (bit v & 31 of word v >> 5 = voxel v)
#define OF_T 10      // staged tile edge: the block and a one-cell halo
#define OF_T3 (OF_T * OF_T * OF_T)
#define OF_THREADS 128
#define OF_REC 16    // int64 fields of a cluster record

#define OF_OUT 3     // halo class of a cell outside the volume, next to the OC_* classes

struct OfAux {
  uint32_t* mask;  // [max_blocks * 16] frontier bits as of the last update
  int* dirty;      // [max_blocks] = tslam_octo::fr_dirty
  int* rflag;      // [max_blocks] block is on this update's region list
  int* rlist;      // [max_blocks] blocks to re-examine
  int* pc;         // [max_blocks + 1] frontier voxels per block of the submap (0 elsewhere)
  int* off;        // [max_blocks + 1] exclusive scan of pc; off[nb] = frontier voxels
  int* ctr;        // [4] region blocks, clusters
};
struct OfVox {     // per frontier voxel (compact index)
  int* parent;     // union-find parent; after compress, the root
  int* slot;       // cluster slot (valid at roots)
};
struct OfClu {     // per cluster slot
  unsigned long long* key;    // label (smallest linear key)
  unsigned long long* key_s;  // labels in ascending order
  long long* rec;             // [16] per slot: field 0 unused (the label lives in key), 1..15 as the output record
  int* sid;                   // slot ids 0..nc-1
  int* sid_s;                 // slot of the q-th cluster in label order
  int* ord;                   // ordinal of each slot in label order
};

// index of the block holding local cell (lx, ly, lz), each in [-1, 8], in a 27-entry neighbour table (13 = the block)
__device__ __forceinline__ int of_nbr_slot(int lx, int ly, int lz) {
  return (((lx + 8) >> 3) * 3 + ((ly + 8) >> 3)) * 3 + ((lz + 8) >> 3);
}

__device__ __forceinline__ long long of_key(const OcGrid& g, int i, int j, int k) {
  return ((long long)(i + g.hN) * g.N + (j + g.hN)) * g.Nz + (k + g.hNz);
}

// 1. prepare: one thread per pool block
__global__ void __launch_bounds__(256) k_octo_frontier_prepare(OcGrid g, OfAux a, int submap, int nb, int nb_prev, int full) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb; b += gridDim.x * blockDim.x) {
    if (b >= nb_prev) {  // allocated since the last update: no frontier bits, whatever the slot held before a reset
      uint4* w = (uint4*)(a.mask + (size_t)b * OF_WORDS);
#pragma unroll
      for (int q = 0; q < OF_WORDS / 4; ++q) w[q] = make_uint4(0u, 0u, 0u, 0u);
    }
    const int flagged = a.dirty[b];
    if (flagged) a.dirty[b] = 0;
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    if (s != submap) continue;
    if (full) {
      a.rlist[atomicAdd(&a.ctr[0], 1)] = b;
      continue;
    }
    if (!flagged) continue;
    for (int f = 0; f < 7; ++f) {  // the block and its existing face neighbours
      const int ax = f >> 1, sg = (f & 1) ? 1 : -1;
      const int x = f == 6 ? b : ts_find(g, ts_pack_key(s, bx + (ax == 0) * sg, by + (ax == 1) * sg, bz + (ax == 2) * sg));
      if (x >= 0 && atomicExch(&a.rflag[x], 1) == 0) a.rlist[atomicAdd(&a.ctr[0], 1)] = x;
    }
  }
}

// 2. classify: one CTA per listed block
__global__ void __launch_bounds__(OF_THREADS) k_octo_frontier_classify(OcGrid g, OfAux a, int l_occ) {
  __shared__ unsigned char cls[OF_T3];
  __shared__ int fnb[6];  // face neighbours -x, +x, -y, +y, -z, +z (-1 = absent)
  const int n = a.ctr[0];
  for (int q = blockIdx.x; q < n; q += gridDim.x) {
    const int b = a.rlist[q];
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    __syncthreads();  // the previous block's tile is consumed
    if (threadIdx.x < 6) {
      const int ax = threadIdx.x >> 1, sg = (threadIdx.x & 1) ? 1 : -1;
      fnb[threadIdx.x] = ts_find(g, ts_pack_key(s, bx + (ax == 0) * sg, by + (ax == 1) * sg, bz + (ax == 2) * sg));
    }
    if (threadIdx.x == 0) a.rflag[b] = 0;
    __syncthreads();
    for (int c = threadIdx.x; c < OF_T3; c += blockDim.x) {
      const int lz = c % OF_T - 1, ly = (c / OF_T) % OF_T - 1, lx = c / (OF_T * OF_T) - 1;
      const int ox = lx < 0 ? -1 : (lx > 7 ? 1 : 0), oy = ly < 0 ? -1 : (ly > 7 ? 1 : 0), oz = lz < 0 ? -1 : (lz > 7 ? 1 : 0);
      if ((ox != 0) + (oy != 0) + (oz != 0) > 1) continue;  // edges and corners of the halo are never read
      const int blk = ox ? fnb[ox > 0] : (oy ? fnb[2 + (oy > 0)] : (oz ? fnb[4 + (oz > 0)] : b));
      const int i = bx * OC_B + lx, j = by * OC_B + ly, k = bz * OC_B + lz;
      unsigned char cl = OF_OUT;  // a cell outside the volume can never be observed: it does not count as UNKNOWN
      if (ts_in_bounds(g, i, j, k)) cl = blk < 0 ? OC_UNK : oc_class(g.cnt[(size_t)blk * OC_B3 + oc_voxel_off(i, j, k)], l_occ);
      cls[c] = cl;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < OC_B3 / OF_THREADS; ++r) {
      const int v = r * OF_THREADS + threadIdx.x;
      const int c0 = ((v >> 6) + 1) * OF_T * OF_T + (((v >> 3) & 7) + 1) * OF_T + ((v & 7) + 1);
      const bool f = cls[c0] == OC_FREE && (cls[c0 - OF_T * OF_T] == OC_UNK || cls[c0 + OF_T * OF_T] == OC_UNK ||
                                            cls[c0 - OF_T] == OC_UNK || cls[c0 + OF_T] == OC_UNK || cls[c0 - 1] == OC_UNK ||
                                            cls[c0 + 1] == OC_UNK);
      const unsigned word = __ballot_sync(0xffffffffu, f);
      if ((threadIdx.x & 31) == 0) a.mask[(size_t)b * OF_WORDS + (v >> 5)] = word;
    }
  }
}

// 3. compact: frontier voxels per block of the submap (pc[nb] = 0, so the exclusive scan's last entry is the total)
__global__ void __launch_bounds__(256) k_octo_frontier_count(OcGrid g, OfAux a, int submap, int nb) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b <= nb; b += gridDim.x * blockDim.x) {
    int n = 0;
    if (b < nb) {
      int s, bx, by, bz;
      ts_unpack_key(g.block_key[b], s, bx, by, bz);
      if (s == submap) {
        const uint4* w = (const uint4*)(a.mask + (size_t)b * OF_WORDS);
#pragma unroll
        for (int q = 0; q < OF_WORDS / 4; ++q) {
          const uint4 u = w[q];
          n += __popc(u.x) + __popc(u.y) + __popc(u.z) + __popc(u.w);
        }
      }
    }
    a.pc[b] = n;
  }
}

__global__ void __launch_bounds__(256) k_octo_frontier_iota(int* p, int n) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) p[t] = t;
}

// union-find over compact indices; parent[x] <= x always (a root is only ever hooked under a smaller one)
__device__ __forceinline__ int of_find(int* p, int x) {
  volatile int* vp = p;
  int px = vp[x];
  while (px != x) {
    const int ppx = vp[px];
    if (ppx != px) vp[x] = ppx;  // path halving: x now points at its grandparent (same set, still <= x)
    x = ppx;
    px = vp[x];
  }
  return x;
}

__device__ __forceinline__ void of_union(int* p, int a, int b) {
  a = of_find(p, a);
  b = of_find(p, b);
  while (a != b) {
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicCAS(&p[b], b, a);  // hook the larger root under the smaller
    if (old == b) return;
    b = of_find(p, old);  // b was hooked meanwhile: retry from the new roots
    a = of_find(p, a);
  }
}

// Warp-per-block traversal of the frontier voxels (link, stats, gather): the warp stages the block's mask and its 27
// neighbour blocks, then visits the voxels 32 at a time.  fn(t, v, has, bx, by, bz, nbr, mask) runs on every lane of
// every round (warp-uniform); t is the compact index of voxel v where the lane has a frontier voxel (has).
template <class F>
__device__ __forceinline__ void of_for_blocks(const OcGrid& g, const OfAux& a, int nb, F fn) {
  __shared__ int s_nbr[8][27];
  __shared__ uint32_t s_mk[8][OF_WORDS];
  const int wi = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int b = blockIdx.x * 8 + wi; b < nb; b += gridDim.x * 8) {
    const int o0 = a.off[b];
    if (a.off[b + 1] == o0) continue;  // no frontier voxel, or another submap's block (uniform per warp)
    int s, bx, by, bz;
    ts_unpack_key(g.block_key[b], s, bx, by, bz);
    __syncwarp();
    if (lane < 27) s_nbr[wi][lane] = lane == 13 ? b : ts_find(g, ts_pack_key(s, bx + lane / 9 - 1, by + (lane / 3) % 3 - 1, bz + lane % 3 - 1));
    if (lane < OF_WORDS) s_mk[wi][lane] = a.mask[(size_t)b * OF_WORDS + lane];
    __syncwarp();
    int before = 0;  // frontier voxels of the block in the words before this round's
    for (int r = 0; r < OF_WORDS; ++r) {
      const uint32_t mw = s_mk[wi][r];
      const bool has = (mw >> lane) & 1u;
      const int t = o0 + before + __popc(mw & ((1u << lane) - 1u));
      fn(t, r * 32 + lane, has, bx, by, bz, s_nbr[wi], s_mk[wi]);
      before += __popc(mw);
    }
  }
}

// compact index of voxel nv of block nbk, or -1 when it is not a frontier voxel
__device__ __forceinline__ int of_compact(const OfAux& a, int nbk, int nv, const uint32_t* own_mask, bool own) {
  const uint32_t* m = own ? own_mask : a.mask + (size_t)nbk * OF_WORDS;
  const int w = nv >> 5;
  const uint32_t mw = m[w];
  if (!((mw >> (nv & 31)) & 1u)) return -1;
  int t = a.off[nbk] + __popc(mw & ((1u << (nv & 31)) - 1u));
  for (int q = 0; q < w; ++q) t += __popc(m[q]);
  return t;
}

// 4. link: 13 backward neighbours (offsets before (0,0,0) in (dx, dy, dz) order) cover every 26-adjacent pair once
__global__ void __launch_bounds__(256) k_octo_frontier_link(OcGrid g, OfAux a, OfVox x, int nb) {
  of_for_blocks(g, a, nb, [&](int t, int v, bool has, int bx, int by, int bz, const int* nbr, const uint32_t* mk) {
    if (!has) return;
    const int lx = v >> 6, ly = (v >> 3) & 7, lz = v & 7;
    for (int o = 0; o < 13; ++o) {
      const int dx = o / 9 - 1, dy = (o / 3) % 3 - 1, dz = o % 3 - 1;
      const int nx = lx + dx, ny = ly + dy, nz = lz + dz;
      if (!ts_in_bounds(g, bx * OC_B + nx, by * OC_B + ny, bz * OC_B + nz)) continue;
      const int sl = of_nbr_slot(nx, ny, nz);
      const int nbk = nbr[sl];
      if (nbk < 0) continue;
      const int tn = of_compact(a, nbk, oc_voxel_off(nx, ny, nz), mk, sl == 13);
      if (tn >= 0) of_union(x.parent, t, tn);
    }
  });
}

// 5. compress: every voxel to its root; each root takes a cluster slot.  The walk to the root does not halve the path:
// a halving store to parent[t] computed before thread t stores the root could land after it and leave a non-root there.
__global__ void __launch_bounds__(256) k_octo_frontier_compress(OfAux a, OfVox x, int n) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
    int r = t, pr;
    while ((pr = x.parent[r]) != r) r = pr;  // every value read is an ancestor: stores of this kernel only shorten paths
    x.parent[t] = r;
    if (r == t) x.slot[t] = atomicAdd(&a.ctr[1], 1);
  }
}

__global__ void __launch_bounds__(256) k_octo_frontier_rec_init(OfClu c, int nc) {
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < nc; s += gridDim.x * blockDim.x) {
    c.key[s] = ULLONG_MAX;
    c.sid[s] = s;
    long long* r = c.rec + (size_t)s * OF_REC;
#pragma unroll
    for (int f = 0; f < OF_REC; ++f) r[f] = (f >= 5 && f <= 7) ? LLONG_MAX : ((f >= 8 && f <= 10) ? LLONG_MIN : 0);
  }
}

// 6. stats: per voxel n, i, j, k, bounds, and its (voxel, UNKNOWN in-volume 6-neighbour) pairs with their unit offsets;
// the lanes of a warp that share a cluster reduce first and one of them does the atomics
__global__ void __launch_bounds__(256) k_octo_frontier_stats(OcGrid g, OfAux a, OfVox x, OfClu c, int nb) {
  of_for_blocks(g, a, nb, [&](int t, int v, bool has, int bx, int by, int bz, const int* nbr, const uint32_t* mk) {
    const int lane = threadIdx.x & 31;
    const int lx = v >> 6, ly = (v >> 3) & 7, lz = v & 7;
    const int i = bx * OC_B + lx, j = by * OC_B + ly, k = bz * OC_B + lz;
    int sl = -1, faces = 0, d[3] = {0, 0, 0};
    unsigned long long key = ULLONG_MAX;
    if (has) {
      sl = x.slot[x.parent[t]];
      key = (unsigned long long)of_key(g, i, j, k);
#pragma unroll
      for (int f = 0; f < 6; ++f) {
        const int ax = f >> 1, sg = (f & 1) ? 1 : -1;
        const int nx = lx + (ax == 0) * sg, ny = ly + (ax == 1) * sg, nz = lz + (ax == 2) * sg;
        if (!ts_in_bounds(g, bx * OC_B + nx, by * OC_B + ny, bz * OC_B + nz)) continue;
        const int nbk = nbr[of_nbr_slot(nx, ny, nz)];
        if (nbk >= 0 && lo_known(g.cnt[(size_t)nbk * OC_B3 + oc_voxel_off(nx, ny, nz)])) continue;
        faces++;
        d[ax] += sg;
      }
    }
    unsigned todo = __ballot_sync(0xffffffffu, has);
    while (todo) {
      const int leader = __ffs(todo) - 1;
      const int ls = __shfl_sync(0xffffffffu, sl, leader);
      const unsigned peers = __ballot_sync(0xffffffffu, has && sl == ls);
      const bool in = (peers >> lane) & 1u;
      const int n_ = __reduce_add_sync(0xffffffffu, in ? 1 : 0);
      const int si = __reduce_add_sync(0xffffffffu, in ? i : 0), sj = __reduce_add_sync(0xffffffffu, in ? j : 0),
                sk = __reduce_add_sync(0xffffffffu, in ? k : 0);
      const int mi = __reduce_min_sync(0xffffffffu, in ? i : INT_MAX), mj = __reduce_min_sync(0xffffffffu, in ? j : INT_MAX),
                mk_ = __reduce_min_sync(0xffffffffu, in ? k : INT_MAX);
      const int xi = __reduce_max_sync(0xffffffffu, in ? i : INT_MIN), xj = __reduce_max_sync(0xffffffffu, in ? j : INT_MIN),
                xk = __reduce_max_sync(0xffffffffu, in ? k : INT_MIN);
      const int fa = __reduce_add_sync(0xffffffffu, in ? faces : 0);
      const int d0 = __reduce_add_sync(0xffffffffu, in ? d[0] : 0), d1 = __reduce_add_sync(0xffffffffu, in ? d[1] : 0),
                d2 = __reduce_add_sync(0xffffffffu, in ? d[2] : 0);
      unsigned long long kk = in ? key : ULLONG_MAX;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) kk = min(kk, __shfl_xor_sync(0xffffffffu, kk, o));
      if (lane == leader) {
        long long* r = c.rec + (size_t)ls * OF_REC;
        atomicMin(&c.key[ls], kk);
        atomicAdd((unsigned long long*)&r[1], (unsigned long long)(long long)n_);
        atomicAdd((unsigned long long*)&r[2], (unsigned long long)(long long)si);
        atomicAdd((unsigned long long*)&r[3], (unsigned long long)(long long)sj);
        atomicAdd((unsigned long long*)&r[4], (unsigned long long)(long long)sk);
        atomicMin(&r[5], (long long)mi); atomicMin(&r[6], (long long)mj); atomicMin(&r[7], (long long)mk_);
        atomicMax(&r[8], (long long)xi); atomicMax(&r[9], (long long)xj); atomicMax(&r[10], (long long)xk);
        atomicAdd((unsigned long long*)&r[11], (unsigned long long)(long long)fa);
        atomicAdd((unsigned long long*)&r[12], (unsigned long long)(long long)d0);
        atomicAdd((unsigned long long*)&r[13], (unsigned long long)(long long)d1);
        atomicAdd((unsigned long long*)&r[14], (unsigned long long)(long long)d2);
      }
      todo &= ~peers;
    }
  });
}

// 7. order: ordinal of each slot once the labels are sorted
__global__ void __launch_bounds__(256) k_octo_frontier_order(OfClu c, int nc) {
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nc; q += gridDim.x * blockDim.x) c.ord[c.sid_s[q]] = q;
}

// (ijk, cluster ordinal) of every frontier voxel, row = compact index (pool order of the blocks, then voxel order)
__global__ void __launch_bounds__(256) k_octo_frontier_gather(OcGrid g, OfAux a, OfVox x, OfClu c, int nb, long long cap,
                                                              int32_t* idx, int32_t* cluster) {
  of_for_blocks(g, a, nb, [&](int t, int v, bool has, int bx, int by, int bz, const int*, const uint32_t*) {
    if (!has || t >= cap) return;
    idx[3 * (size_t)t] = bx * OC_B + (v >> 6);
    idx[3 * (size_t)t + 1] = by * OC_B + ((v >> 3) & 7);
    idx[3 * (size_t)t + 2] = bz * OC_B + (v & 7);
    cluster[t] = c.ord[x.slot[x.parent[t]]];
  });
}

// cluster records in label order
__global__ void __launch_bounds__(256) k_octo_frontier_records(OfClu c, int n, int64_t* out) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < (long long)n * OF_REC; e += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(e / OF_REC), f = (int)(e % OF_REC);
    out[e] = f == 0 ? (int64_t)c.key_s[q] : c.rec[(size_t)c.sid_s[q] * OF_REC + f];
  }
}

// ---- host side -----------------------------------------------------------------------------------------------------
// bytes per pool block: mask 64 + dirty flag, region flag, region list, popcount, offset 20 = 84 (+ 8 + 16 once)
static size_t of_bytes(size_t nb) { return nb * (OF_WORDS * 4 + 5 * 4) + 2 * 4 + 4 * 4; }

static OfAux of_aux(tslam_octo* m) {
  const size_t nb = (size_t)m->g.max_blocks;
  OfAux a;
  a.mask = (uint32_t*)m->fr_mem;
  a.dirty = (int*)(a.mask + nb * OF_WORDS);
  a.rflag = a.dirty + nb;
  a.rlist = a.rflag + nb;
  a.pc = a.rlist + nb;
  a.off = a.pc + nb + 1;
  a.ctr = a.off + nb + 1;
  return a;
}

static OfVox of_vox(tslam_octo* m) {
  OfVox x;
  x.parent = (int*)m->fr_vox;
  x.slot = x.parent + m->fr_vox_cap;
  return x;
}

static OfClu of_clu(tslam_octo* m) {
  const size_t cap = (size_t)m->fr_clu_cap;
  OfClu c;
  c.rec = (long long*)m->fr_clu;
  c.key = (unsigned long long*)(c.rec + cap * OF_REC);
  c.key_s = c.key + cap;
  c.sid = (int*)(c.key_s + cap);
  c.sid_s = c.sid + cap;
  c.ord = c.sid_s + cap;
  return c;
}

static int of_alloc(tslam_octo* m) {
  if (m->fr_mem) return TSLAM_OK;
  const size_t bytes = of_bytes((size_t)m->g.max_blocks);
  TS_CUDA(cudaMalloc(&m->fr_mem, bytes));
  TS_CUDA(cudaMemset(m->fr_mem, 0, bytes));
  m->fr_dirty = of_aux(m).dirty;
  return TSLAM_OK;
}

// (re)allocate *p for at least `need` entries of `per` bytes (grown by half again, so a slowly growing set reallocates rarely)
static int of_grow(void** p, long long* cap, long long need, size_t per) {
  if (need <= *cap) return TSLAM_OK;
  const long long n = need + need / 2 + 1024;
  if (*p) cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  TS_CUDA(cudaMalloc(p, (size_t)n * per));
  *cap = n;
  return TSLAM_OK;
}

int oc_frontier_free(tslam_octo* m) {
  if (m->fr_mem) cudaFree(m->fr_mem);
  if (m->fr_vox) cudaFree(m->fr_vox);
  if (m->fr_clu) cudaFree(m->fr_clu);
  if (m->fr_tmp) cudaFree(m->fr_tmp);
  m->fr_mem = m->fr_vox = m->fr_clu = m->fr_tmp = nullptr;
  m->fr_dirty = nullptr;
  m->fr_vox_cap = m->fr_clu_cap = 0;
  m->fr_tmp_bytes = 0;
  return TSLAM_OK;
}

// mode 0 = incremental when the state allows it (same submap as the last update, no reset / fusion in between), 1 = full.
// stats4 (HOST, may be NULL): frontier voxels, clusters, blocks re-examined, 1 when the update was full.
extern "C" int tslam_octo_frontier_update(tslam_octo_t* m, int32_t submap, int32_t mode, int32_t* stats4, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  int rc = oc_logodds_submap(m, submap, "tslam_octo_frontier_update", "a frontier set");
  if (rc) return rc;
  if (mode != 0 && mode != 1) { ts_set_error("tslam_octo_frontier_update: mode must be 0 (incremental) or 1 (full)"); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  rc = of_alloc(m);
  if (rc) return rc;
  OfAux a = of_aux(m);
  const bool full = mode == 1 || !m->fr_track.ready || m->fr_track.submap != submap;
  m->fr_track.ready = 0;  // until this update has completed
  int nb = 0;
  TS_CUDA(cudaMemcpyAsync(&nb, m->g.n_blocks, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemsetAsync(a.ctr, 0, 4 * 4, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (nb > m->g.max_blocks) nb = m->g.max_blocks;
  const int cap_grid = m->sm_count * 16;
  k_octo_frontier_prepare<<<oc_grid(nb, 256, cap_grid), 256, 0, st>>>(m->g, a, submap, nb, full ? 0 : m->fr_nb, full ? 1 : 0);
  TS_LAUNCH_CHECK(m);
  k_octo_frontier_classify<<<m->sm_count * 8, OF_THREADS, 0, st>>>(m->g, a, m->lo.l_occ);
  TS_LAUNCH_CHECK(m);
  k_octo_frontier_count<<<oc_grid((long long)nb + 1, 256, cap_grid), 256, 0, st>>>(m->g, a, submap, nb);
  TS_LAUNCH_CHECK(m);
  size_t tb = 0;
  TS_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, a.pc, a.off, nb + 1, st));
  rc = oc_reserve(&m->fr_tmp, &m->fr_tmp_bytes, tb);
  if (rc) return rc;
  TS_CUDA(cub::DeviceScan::ExclusiveSum(m->fr_tmp, tb, a.pc, a.off, nb + 1, st));
  int n = 0, region = 0, nc = 0;
  TS_CUDA(cudaMemcpyAsync(&n, a.off + nb, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaMemcpyAsync(&region, a.ctr, 4, cudaMemcpyDeviceToHost, st));
  TS_CUDA(cudaStreamSynchronize(st));
  if (n > 0) {
    rc = of_grow(&m->fr_vox, &m->fr_vox_cap, n, 2 * sizeof(int));
    if (rc) return rc;
    OfVox x = of_vox(m);
    k_octo_frontier_iota<<<oc_grid(n, 256, cap_grid), 256, 0, st>>>(x.parent, n);
    TS_LAUNCH_CHECK(m);
    k_octo_frontier_link<<<oc_grid(nb, 8, cap_grid), 256, 0, st>>>(m->g, a, x, nb);
    TS_LAUNCH_CHECK(m);
    k_octo_frontier_compress<<<oc_grid(n, 256, cap_grid), 256, 0, st>>>(a, x, n);
    TS_LAUNCH_CHECK(m);
    TS_CUDA(cudaMemcpyAsync(&nc, a.ctr + 1, 4, cudaMemcpyDeviceToHost, st));
    TS_CUDA(cudaStreamSynchronize(st));
    rc = of_grow(&m->fr_clu, &m->fr_clu_cap, nc, OF_REC * 8 + 2 * 8 + 3 * 4);
    if (rc) return rc;
    OfClu c = of_clu(m);
    k_octo_frontier_rec_init<<<oc_grid(nc, 256, cap_grid), 256, 0, st>>>(c, nc);
    TS_LAUNCH_CHECK(m);
    k_octo_frontier_stats<<<oc_grid(nb, 8, cap_grid), 256, 0, st>>>(m->g, a, x, c, nb);
    TS_LAUNCH_CHECK(m);
    const long long keys = (long long)m->g.N * m->g.N * m->g.Nz;
    int end_bit = 1;
    while (end_bit < 64 && (1ll << end_bit) < keys) end_bit++;
    tb = 0;
    TS_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, c.key, c.key_s, c.sid, c.sid_s, nc, 0, end_bit, st));
    rc = oc_reserve(&m->fr_tmp, &m->fr_tmp_bytes, tb);
    if (rc) return rc;
    TS_CUDA(cub::DeviceRadixSort::SortPairs(m->fr_tmp, tb, c.key, c.key_s, c.sid, c.sid_s, nc, 0, end_bit, st));
    k_octo_frontier_order<<<oc_grid(nc, 256, cap_grid), 256, 0, st>>>(c, nc);
    TS_LAUNCH_CHECK(m);
    TS_CUDA(cudaStreamSynchronize(st));
  }
  m->fr_track = OcTrack{1, submap};
  m->fr_nb = nb;
  m->fr_n = n;
  m->fr_nc = nc;
  if (stats4) { stats4[0] = n; stats4[1] = nc; stats4[2] = region; stats4[3] = full ? 1 : 0; }
  return TSLAM_OK;
}

int oc_frontier_rows(tslam_octo* m, int32_t* idx, int32_t* cluster, cudaStream_t st) {
  if (m->fr_n > 0) {
    k_octo_frontier_gather<<<oc_grid(m->fr_nb, 8, m->sm_count * 16), 256, 0, st>>>(m->g, of_aux(m), of_vox(m), of_clu(m), m->fr_nb,
                                                                                   m->fr_n, idx, cluster);
    TS_LAUNCH_CHECK(m);
  }
  return TSLAM_OK;
}

int oc_frontier_records(tslam_octo* m, int64_t* rec16, cudaStream_t st) {
  if (m->fr_nc > 0) {
    k_octo_frontier_records<<<oc_grid((long long)m->fr_nc * OF_REC, 256, m->sm_count * 16), 256, 0, st>>>(of_clu(m), m->fr_nc, rec16);
    TS_LAUNCH_CHECK(m);
  }
  return TSLAM_OK;
}

extern "C" int tslam_octo_frontier_gather(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, int32_t* cluster, int64_t* n_out,
                                          void* stream) {
  if (!m || !n_out || cap < 0 || (cap > 0 && (!idx || !cluster))) return TSLAM_E_INVALID;
  int rc = oc_track_readable(m, m->fr_track, submap, "tslam_octo_frontier_gather", "tslam_octo_frontier_update");
  if (rc) return rc;
  *n_out = m->fr_n;
  if (m->fr_n > 0 && cap > 0) {
    k_octo_frontier_gather<<<oc_grid(m->fr_nb, 8, m->sm_count * 16), 256, 0, (cudaStream_t)stream>>>(
        m->g, of_aux(m), of_vox(m), of_clu(m), m->fr_nb, cap, idx, cluster);
    TS_LAUNCH_CHECK(m);
  }
  if (m->fr_n > cap) { ts_set_error("octo frontier gather: %d voxels > capacity %lld", m->fr_n, (long long)cap); return TSLAM_E_CAPACITY; }
  return TSLAM_OK;
}

extern "C" int tslam_octo_frontier_clusters(tslam_octo_t* m, int32_t submap, int64_t cap, int64_t* rec16, int64_t* n_out, void* stream) {
  if (!m || !n_out || cap < 0 || (cap > 0 && !rec16)) return TSLAM_E_INVALID;
  int rc = oc_track_readable(m, m->fr_track, submap, "tslam_octo_frontier_clusters", "tslam_octo_frontier_update");
  if (rc) return rc;
  *n_out = m->fr_nc;
  const int n = (int)(m->fr_nc < cap ? m->fr_nc : cap);
  if (n > 0) {
    k_octo_frontier_records<<<oc_grid((long long)n * OF_REC, 256, m->sm_count * 16), 256, 0, (cudaStream_t)stream>>>(of_clu(m), n, rec16);
    TS_LAUNCH_CHECK(m);
  }
  if (m->fr_nc > cap) { ts_set_error("octo frontier clusters: %d clusters > capacity %lld", m->fr_nc, (long long)cap); return TSLAM_E_CAPACITY; }
  return TSLAM_OK;
}
