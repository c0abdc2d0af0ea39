// libtslam.so - the per-frame queue of the TSDF map: frames handed over one at a time are staged on a copy stream
// (three hand-over modes) and integrated a batch at a time (ts_integrate_depth_impl, tslam_integrate.cu).  sm_90a.
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include "tslam_internal.cuh"

// ---------------------------------------------------------------------------
// per-frame queue: the reference API hands over ONE frame per call (recast_depth_to_map, dense_tsdf.py:162-165).
// tslam_tsdf_queue_depth copies the frame to a device staging slot on a copy stream (overlapping the kernels of
// the previous batch) and records its pose; a full queue (TSLAM_MAX_BATCH frames) or tslam_tsdf_flush launches
// the batch: bucket -> ray march -> commit.
// ---------------------------------------------------------------------------
// the queue's part of tslam_tsdf_create / tslam_tsdf_destroy: switches, copy stream, events
int ts_queue_init(tslam_tsdf* m) {
  {
    int prio_lo = 0, prio_hi = 0;  // highest priority: the gather kernel's few CTAs go first when SM slots free up
    TS_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
    TS_CUDA(cudaStreamCreateWithPriority(&m->copy_stream, cudaStreamNonBlocking, prio_hi));
  }
  {
    // Page-locked frames are COPIED at call time by default (the reference's semantics: recast_depth_to_map has
    // consumed the array when it returns).  Borrowing them instead - the GPU reads the sampled rows straight from
    // host memory a few calls later - is opt-in: tslam_tsdf_set_frame_mode(m, 1) or TSLAM_ZERO_COPY=1.
    const char* zc = getenv("TSLAM_ZERO_COPY");
    m->zero_copy = (zc && zc[0] == '1') ? 1 : 0;
    const char* fc = getenv("TSLAM_FRAME_COPY");  // "dma": pageable frames through cudaMemcpyAsync too (A/B against the ring)
    m->stage_mode = (fc && strcmp(fc, "dma") == 0) ? 0 : 1;
    // page-locked frames in copy mode: awaited cudaMemcpyAsync (default; A/B: "ring" = through the host ring like
    // pageable frames, "fetch" = awaited row fetch).  On one H100 SXM (400 W power limit, one rank,
    // bench.py e2e arms, three runs): dma 32.0-35.5 k, ring 13.4-14.8 k, fetch 25.1-27.6 k frames/s - the copy engine is the
    // one that neither depends on the host's memcpy bandwidth (8 ranks share it) nor on the PCIe read latency
    const char* pc = getenv("TSLAM_PINNED_COPY");
    m->pinned_mode = (pc && strcmp(pc, "ring") == 0) ? 0 : (pc && strcmp(pc, "fetch") == 0) ? 1 : 2;
    m->trace = getenv("TSLAM_TRACE") != nullptr;
    if (m->trace) {
      for (int i = 0; i < 2; i++)
        for (int k = 0; k < 4; k++) TS_CUDA(cudaEventCreate(&m->tr_ev[i][k]));
      TS_CUDA(cudaEventCreate(&m->tr_base));
      TS_CUDA(cudaEventRecord(m->tr_base, 0));
    }
    // frames per queue launch, alternating a, b, a, b, ...: half a batch each by default, so that the kernels of the
    // first half run while the caller is still handing over the second half.  (16,48 and 24,40 were measured too: with
    // page-locked frames the step is bound by the PCIe reads of the row gather, the split hardly matters.)
    m->queue_launch[0] = TSLAM_MAX_BATCH / 2;
    m->queue_launch[1] = TSLAM_MAX_BATCH / 2;
    const char* ql = getenv("TSLAM_QUEUE_LAUNCH");
    if (ql) {
      int a = 0, b = 0;
      const int k = sscanf(ql, "%d,%d", &a, &b);
      if (k == 1) b = a;
      if (k >= 1 && a >= 1 && a <= TSLAM_MAX_BATCH && b >= 1 && b <= TSLAM_MAX_BATCH) { m->queue_launch[0] = a; m->queue_launch[1] = b; }
    }
  }
  for (int i = 0; i < 2; i++) {
    TS_CUDA(cudaEventCreateWithFlags(&m->ev_copied[i], cudaEventDisableTiming));
    TS_CUDA(cudaEventCreateWithFlags(&m->ev_free[i], cudaEventDisableTiming));
  }
  return TSLAM_OK;
}
void ts_queue_free(tslam_tsdf* m) {
  cudaStreamDestroy(m->copy_stream);
  if (m->h_ring) cudaFreeHost(m->h_ring);
  for (int i = 0; i < 2; i++) { cudaEventDestroy(m->ev_copied[i]); cudaEventDestroy(m->ev_free[i]); }
}

// Pinned (page-locked) host frames: instead of a DMA copy of the whole 614 KB frame, a small kernel reads ONLY THE
// SAMPLED ROWS (every recast_step-th row, :192) straight from host memory over PCIe - 16-byte loads, a warp covers
// 512 contiguous bytes - and drops them at their place in the device staging frame.  Half the PCIe bytes for
// recast_step 2, one launch per TS_GATHER_GROUP frames instead of one copy call per frame.
#define TS_GATHER_GROUP 8
struct TsGatherArgs {
  const uint4* src[TS_GATHER_GROUP];
  uint4* dst[TS_GATHER_GROUP];
  int sstride[TS_GATHER_GROUP];  // source row stride (16-byte units): recast_step rows for a caller's frame, 1 row for the ring
};
__global__ void __launch_bounds__(256) k_gather_rows(const __grid_constant__ TsGatherArgs ga, int hh, int row_u4, int row_stride_u4) {
  const uint4* __restrict__ src = ga.src[blockIdx.y];
  uint4* __restrict__ dst = ga.dst[blockIdx.y];
  const int sstride = ga.sstride[blockIdx.y];
  const int total = hh * row_u4;
  const int base = (blockIdx.x * 256 + threadIdx.x) * 4;
  uint4 v[4];
  int off[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {  // 4 independent 16-byte PCIe reads in flight per thread
    const int i = base + k;
    off[k] = -1;
    if (i < total) {
      const int jj = i / row_u4, c = i - jj * row_u4;
      off[k] = jj * row_stride_u4 + c;
      v[k] = __ldcs(src + (jj * sstride + c));
    }
  }
#pragma unroll
  for (int k = 0; k < 4; k++)
    if (off[k] >= 0) dst[off[k]] = v[k];
}

// hand the queued zero-copy frames [q_gathered, q_n) to gather launches on the copy stream
static int ts_gather_pending(tslam_tsdf* m) {
  const int b = m->q_buf;
  const int step = m->cfg.recast_step;
  const int hh = (int)((double)m->q_h / step), row_u4 = m->q_w / 8;
  while (m->q_gathered < m->q_n) {
    TsGatherArgs ga;
    int k = 0;
    while (m->q_gathered < m->q_n && k < TS_GATHER_GROUP) {
      const int q = m->q_gathered++;
      if (!m->q_hptr[q]) continue;
      ga.src[k] = (const uint4*)m->q_hptr[q];
      ga.sstride[k] = m->q_sstride[q];
      ga.dst[k] = (uint4*)(m->depth_stage + (size_t)b * TSLAM_MAX_BATCH * m->cfg.max_image_pixels + (size_t)q * m->q_h * m->q_w);
      k++;
    }
    if (k == 0 || hh <= 0) continue;
    dim3 grid((hh * row_u4 + 1023) / 1024, k);
    k_gather_rows<<<grid, 256, 0, m->copy_stream>>>(ga, hh, row_u4, step * row_u4);
    TS_LAUNCH_CHECK(m);
  }
  return TSLAM_OK;
}

int ts_launch_queue(tslam_tsdf* m, cudaStream_t st) {
  if (m->q_open) {  // a hand-over that was begun and never ended (the caller failed in between): the frame is dropped
    m->q_open = 0;
    if (m->q_await) { m->q_await = 0; TS_CUDA(cudaStreamSynchronize(m->copy_stream)); }
  }
  m->q_phase = 0;  // any launch that is not the queue's own threshold (flush, reader, geometry change) restarts the pattern
  const int n = m->q_n;
  if (n == 0) return TSLAM_OK;
  const int b = m->q_buf;
  {
    int rcg = ts_gather_pending(m);
    if (rcg) return rcg;
  }
  m->q_gathered = 0;
  if (m->trace) TS_CUDA(cudaEventRecord(m->tr_ev[b][1], m->copy_stream));
  TS_CUDA(cudaEventRecord(m->ev_copied[b], m->copy_stream));
  TS_CUDA(cudaStreamWaitEvent(st, m->ev_copied[b], 0));
  if (m->trace) TS_CUDA(cudaEventRecord(m->tr_ev[b][2], st));
  const uint16_t* src = m->depth_stage + (size_t)b * TSLAM_MAX_BATCH * m->cfg.max_image_pixels;
  m->q_n = 0;  // (integrate may recurse into flush through readers; the queue is empty from here on)
  m->q_buf = b ^ 1;
  const uint8_t* tsrc = m->q_has_tex ? m->tex_stage + (size_t)b * TSLAM_MAX_BATCH * m->cfg.max_image_pixels * 3 : nullptr;
  int rc = ts_integrate_depth_impl(m, src, TSLAM_MEM_DEVICE, n, m->q_h, m->q_w, m->q_R, m->q_T, m->q_s, TSLAM_F_COMMIT, (void*)st, tsrc,
                                   m->q_th, m->q_tw);
  if (rc) return rc;
  TS_CUDA(cudaEventRecord(m->ev_free[b], st));
  m->ev_free_valid[b] = true;
  if (m->trace) { TS_CUDA(cudaEventRecord(m->tr_ev[b][3], st)); m->tr_have[b] = n; }
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_set_queue_launch(tslam_tsdf_t* m, int32_t frames_a, int32_t frames_b) {
  if (!m || frames_a < 1 || frames_a > TSLAM_MAX_BATCH || frames_b < 1 || frames_b > TSLAM_MAX_BATCH) { ts_set_error("queue launch sizes must be in [1, %d]", TSLAM_MAX_BATCH); return TSLAM_E_INVALID; }
  if (m->q_n > 0) { ts_set_error("frames are queued: flush before changing the launch size"); return TSLAM_E_INVALID; }
  m->queue_launch[0] = frames_a;
  m->queue_launch[1] = frames_b;
  m->q_phase = 0;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_set_frame_mode(tslam_tsdf_t* m, int borrow_pinned) {
  if (!m) return TSLAM_E_INVALID;
  if (m->q_n > 0) { ts_set_error("frames are queued: flush before changing the frame mode"); return TSLAM_E_INVALID; }
  m->zero_copy = borrow_pinned ? 1 : 0;
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_flush(tslam_tsdf_t* m, void* stream) {
  if (!m) return TSLAM_E_INVALID;
  m->q_phase = 0;
  int rc = ts_launch_queue(m, (cudaStream_t)stream);
  if (rc) return rc;
  return ts_check_deferred_async(m, (cudaStream_t)stream);
}

extern "C" int tslam_tsdf_queue_depth(tslam_tsdf_t* m, const uint16_t* depth_host, int32_t h, int32_t w, const float* R9,
                                      const float* T3, int32_t submap, void* stream) {
  return tslam_tsdf_queue_depth_tex(m, depth_host, nullptr, h, w, 0, 0, R9, T3, submap, stream);
}
#if defined(__SSE2__) || defined(__x86_64__)
#include <emmintrin.h>
static inline void ts_stream_copy_row(uint16_t* dst, const uint16_t* src, size_t bytes) {  // dst 16-byte aligned, bytes % 16 == 0
  __m128i* d = reinterpret_cast<__m128i*>(dst);
  const __m128i* s = reinterpret_cast<const __m128i*>(src);
  const size_t n = bytes / 16;
  size_t i = 0;
  for (; i + 4 <= n; i += 4) {
    const __m128i a = _mm_loadu_si128(s + i), b = _mm_loadu_si128(s + i + 1), c = _mm_loadu_si128(s + i + 2), e = _mm_loadu_si128(s + i + 3);
    _mm_stream_si128(d + i, a); _mm_stream_si128(d + i + 1, b); _mm_stream_si128(d + i + 2, c); _mm_stream_si128(d + i + 3, e);
  }
  for (; i < n; i++) _mm_stream_si128(d + i, _mm_loadu_si128(s + i));
}
static inline void ts_stream_fence() { _mm_sfence(); }
#else
static inline void ts_stream_copy_row(uint16_t* dst, const uint16_t* src, size_t bytes) { memcpy(dst, src, bytes); }
static inline void ts_stream_fence() {}
#endif

// first half of a per-frame hand-over: the frame's copy is STARTED (page-locked source: DMA on the copy stream;
// pageable source: sampled rows into the ring; borrowed: nothing).  ts_queue_end awaits it and records the pose.
static int ts_queue_begin(tslam_tsdf* m, const uint16_t* depth_host, const uint8_t* tex_host, int32_t h, int32_t w, int32_t th, int32_t tw,
                          void* stream) {
  if (m) { int rc0 = ts_check_tex(m, tex_host, th, tw); if (rc0) return rc0; }
  if (!m || !depth_host || h <= 0 || w <= 0) { ts_set_error("bad argument"); return TSLAM_E_INVALID; }
  if ((long long)h * w > m->cfg.max_image_pixels) { ts_set_error("frame %dx%d exceeds max_image_pixels=%d", h, w, m->cfg.max_image_pixels); return TSLAM_E_INVALID; }
  m->q_open = 0;
  m->q_await = 0;
  cudaStream_t st = (cudaStream_t)stream;
  const int has_tex = tex_host != nullptr;
  if (!has_tex) { th = 0; tw = 0; }
  // one batch = one frame geometry and either all or no frames textured
  if (m->q_n > 0 && (m->q_h != h || m->q_w != w || m->q_has_tex != has_tex || m->q_th != th || m->q_tw != tw)) {
    int rc = ts_launch_queue(m, st);
    if (rc) return rc;
  }
  const int b = m->q_buf, q = m->q_n;
  if (q == 0) {
    m->q_h = h; m->q_w = w;
    m->q_has_tex = has_tex; m->q_th = th; m->q_tw = tw;
    // the kernels that read this staging buffer (two batches ago) must be done.  Waiting on the HOST bounds how far
    // the caller can run ahead of the GPU: a pinned frame is consumed before 2*TSLAM_MAX_BATCH further frames are queued.
    if (m->ev_free_valid[b]) TS_CUDA(cudaEventSynchronize(m->ev_free[b]));
    m->q_gathered = 0;
    if (m->trace) {
      if (m->tr_have[b]) {  // timeline of the launch that used this buffer last (ms since handle creation)
        float t[4];
        for (int k = 0; k < 4; k++) cudaEventElapsedTime(&t[k], m->tr_base, m->tr_ev[b][k]);
        fprintf(stderr, "[tslam trace] buf %d frames %d: copy %.3f..%.3f  kernels %.3f..%.3f ms\n", b, m->tr_have[b], t[0], t[1], t[2], t[3]);
      }
      TS_CUDA(cudaEventRecord(m->tr_ev[b][0], m->copy_stream));
    }
  }
  // One linear copy of the whole frame.  (A strided 2-D copy of only the sampled rows halves the bytes but was
  // slower from pinned memory end to end - 240 row descriptors of 1280 B.)
  uint16_t* dst = m->depth_stage + (size_t)b * TSLAM_MAX_BATCH * m->cfg.max_image_pixels + (size_t)q * h * w;  // frames packed h*w apart
  m->q_hptr[q] = nullptr;
  const int step_q = m->cfg.recast_step;
  cudaPointerAttributes at;
  const bool src_pinned = cudaPointerGetAttributes(&at, depth_host) == cudaSuccess && at.type == cudaMemoryTypeHost;
  if (!src_pinned) cudaGetLastError();
  if (m->zero_copy && src_pinned && at.devicePointer && step_q >= 2 && (w % 8) == 0 && ((uintptr_t)depth_host % 16) == 0 && ((size_t)h * w % 8) == 0) {
    m->q_hptr[q] = (const uint16_t*)at.devicePointer;  // borrowed: the GPU reads the caller's frame itself, later
    m->q_sstride[q] = step_q * (w / 8);
  }
  if (!m->q_hptr[q] && (src_pinned ? m->pinned_mode == 0 : m->stage_mode != 0) && (w % 8) == 0) {
    // PAGEABLE source (what np.frombuffer(msg.data) gives the ROS node): the runtime would stage the whole frame through
    // its own bounce buffer inside cudaMemcpyAsync.  Instead the sampled rows (every
    // recast_step-th, :192 - half the bytes for step 2) are copied into the library's page-locked ring with streaming
    // stores - the caller's buffer is free when the call returns - and the GPU fetches them from there over PCIe while
    // the caller hands over the next frames.
    const int hh = (int)((double)h / step_q);
    if (!m->h_ring) {
      m->ring_frame_cap = ((size_t)m->cfg.max_image_pixels / (size_t)step_q + 8) & ~(size_t)7;
      TS_CUDA(cudaHostAlloc((void**)&m->h_ring, (size_t)2 * TSLAM_MAX_BATCH * m->ring_frame_cap * 2, cudaHostAllocMapped));
      TS_CUDA(cudaHostGetDevicePointer((void**)&m->h_ring_dev, m->h_ring, 0));
    }
    if ((size_t)hh * w <= m->ring_frame_cap) {
      const size_t slot = ((size_t)b * TSLAM_MAX_BATCH + (size_t)q) * m->ring_frame_cap;
      uint16_t* hdst = m->h_ring + slot;
      // streaming stores: the ring is read by the GPU over PCIe, never by this CPU - no read-for-ownership of the
      // destination lines, no cache pollution
      // (software prefetch of the rows ahead and 32-byte AVX2 stores were measured on the host: no gain / 2x slower)
      for (int j = 0; j < hh; j++) ts_stream_copy_row(hdst + (size_t)j * w, depth_host + (size_t)j * step_q * w, (size_t)w * 2);
      ts_stream_fence();
      m->q_hptr[q] = m->h_ring_dev + slot;
      m->q_sstride[q] = w / 8;
    }
  }
  if (m->q_hptr[q] && m->sm_count > 8) {
    // the persistent march kernels own every register of the SMs they run on: keep two SMs out of their grids so
    // that the row gather of the NEXT launch's frames can run (and keep PCIe busy) while they march
    m->rm_reserve = 2;
  }
  if (!m->q_hptr[q] && src_pinned && m->pinned_mode == 1 && at.devicePointer && step_q >= 2 && (w % 8) == 0 && ((uintptr_t)depth_host % 16) == 0 &&
      ((size_t)h * w % 8) == 0) {
    // page-locked source, copy mode: the SAMPLED ROWS are fetched right now by a small kernel (half the PCIe bytes of a
    // DMA copy of the frame for recast_step 2) and the fetch is awaited in ts_queue_end
    TsGatherArgs ga;
    ga.src[0] = (const uint4*)at.devicePointer;
    ga.dst[0] = (uint4*)dst;
    ga.sstride[0] = step_q * (w / 8);
    const int hh = (int)((double)h / step_q), row_u4 = w / 8;
    if (hh > 0) {
      dim3 grid((hh * row_u4 + 1023) / 1024, 1);
      k_gather_rows<<<grid, 256, 0, m->copy_stream>>>(ga, hh, row_u4, step_q * row_u4);
      TS_LAUNCH_CHECK(m);
    }
    m->q_await = 1;
    if (m->sm_count > 8) m->rm_reserve = 2;
  } else if (!m->q_hptr[q]) {
    TS_CUDA(cudaMemcpyAsync(dst, depth_host, (size_t)h * w * 2, cudaMemcpyHostToDevice, m->copy_stream));
    // a pageable source has been staged when the call returns; a page-locked one is read by the DMA engine later,
    // so the copy is awaited: the caller may reuse its buffer (camera drivers do)
    if (src_pinned) m->q_await = 1;
  }
  if (has_tex) {
    uint8_t* tdst = m->tex_stage + ((size_t)b * TSLAM_MAX_BATCH * m->cfg.max_image_pixels + (size_t)q * th * tw) * 3;
    TS_CUDA(cudaMemcpyAsync(tdst, tex_host, (size_t)th * tw * 3, cudaMemcpyHostToDevice, m->copy_stream));
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, tex_host) == cudaSuccess && at.type == cudaMemoryTypeHost) m->q_await = 1;
    else cudaGetLastError();
  }
  m->q_open = 1;
  return TSLAM_OK;
}

// second half: the copy started by ts_queue_begin is awaited (the caller's buffers are free when this returns), the pose
// recorded, the queue launched when it is full
static int ts_queue_end(tslam_tsdf* m, const float* R9, const float* T3, int32_t submap, void* stream) {
  if (!m || !R9 || !T3) { ts_set_error("bad argument"); return TSLAM_E_INVALID; }
  if (!m->q_open) { ts_set_error("tslam_tsdf_queue_depth_end without a successful tslam_tsdf_queue_depth_begin"); return TSLAM_E_INVALID; }
  m->q_open = 0;
  if (m->q_await) { m->q_await = 0; TS_CUDA(cudaStreamSynchronize(m->copy_stream)); }
  if (submap < 0 || submap >= m->cfg.max_submaps) { ts_set_error("bad submap id %d", submap); return TSLAM_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  const int q = m->q_n;
  memcpy(m->q_R + 9 * q, R9, 36);
  memcpy(m->q_T + 3 * q, T3, 12);
  m->q_s[q] = submap;
  fz_written(m->ver, submap);
  m->q_n = q + 1;
  if (m->q_n >= m->queue_launch[m->q_phase]) {
    const int ph = m->q_phase;
    int rc = ts_launch_queue(m, st);
    m->q_phase = ph ^ 1;
    return rc;
  }
  if (m->q_n - m->q_gathered >= TS_GATHER_GROUP) return ts_gather_pending(m);
  return TSLAM_OK;
}

extern "C" int tslam_tsdf_queue_depth_tex(tslam_tsdf_t* m, const uint16_t* depth_host, const uint8_t* tex_host, int32_t h, int32_t w,
                                          int32_t th, int32_t tw, const float* R9, const float* T3, int32_t submap, void* stream) {
  if (!R9 || !T3) { ts_set_error("bad argument"); return TSLAM_E_INVALID; }
  if (m && (submap < 0 || submap >= m->cfg.max_submaps)) { ts_set_error("bad submap id %d", submap); return TSLAM_E_INVALID; }
  int rc = ts_queue_begin(m, depth_host, tex_host, h, w, th, tw, stream);
  if (rc) return rc;
  return ts_queue_end(m, R9, T3, submap, stream);
}
extern "C" int tslam_tsdf_queue_depth_begin(tslam_tsdf_t* m, const uint16_t* depth_host, int32_t h, int32_t w, void* stream) {
  return ts_queue_begin(m, depth_host, nullptr, h, w, 0, 0, stream);
}
extern "C" int tslam_tsdf_queue_depth_end(tslam_tsdf_t* m, const float* R9, const float* T3, int32_t submap, void* stream) {
  return ts_queue_end(m, R9, T3, submap, stream);
}
