/* ============================================================================
 * tslam.h - C ABI of libtslam.so, the H100-native dense-mapping backend.
 *
 * The reference (xuhao1/TaichiSLAM) has no FFI layer: its callers use the Python
 * classes DenseTSDF / Octomap / MarchingCubeMesher directly, and those run Taichi
 * kernels.  This ABI is what a maintainer binds (ctypes, see INTEGRATION.md) to
 * replace each Taichi kernel launch; every entry point names the reference
 * method/kernel it stands in for (paths relative to taichi_slam/mapping/).
 *
 * Conventions
 *  - plain C types only; opaque handles; no exceptions cross the boundary.
 *  - every call returns TSLAM_OK (0) or a negative TSLAM_E_* code;
 *    tslam_last_error() gives a thread-local message for the last failure.
 *  - `stream` is a cudaStream_t passed as void* (0 = default stream).  Calls are
 *    ASYNCHRONOUS on that stream unless documented "synchronises".
 *  - `mem` arguments: TSLAM_MEM_DEVICE = the pointer is device memory on the
 *    handle's GPU (caller-owned, must stay alive until the stream reaches the
 *    call); TSLAM_MEM_HOST = host memory, the library copies it to the device
 *    itself (truly asynchronous only when the host memory is pinned).
 *  - handles are not thread-safe; distinct handles are independent.
 *  - voxel indices are signed and centred: valid i in [-N/2, N/2)
 *    (dense_tsdf.py:90).  Out-of-volume samples are skipped (the reference
 *    performs an unchecked access there, mapping_common.py:263-266).
 * ==========================================================================*/
#ifndef TSLAM_H
#define TSLAM_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define TSLAM_OK 0
#define TSLAM_E_INVALID (-1)   /* bad argument                                  */
#define TSLAM_E_CUDA (-2)      /* CUDA runtime error (see tslam_last_error)     */
#define TSLAM_E_POOL_FULL (-3) /* voxel-block pool exhausted; samples dropped   */
#define TSLAM_E_CAPACITY (-4)  /* caller buffer too small; output saturated     */
#define TSLAM_E_NOGPU (-5)     /* no CUDA device: there is NO CPU fallback      */

#define TSLAM_MEM_DEVICE 0
#define TSLAM_MEM_HOST 1

#define TSLAM_MAX_BATCH 64 /* frames per integrate launch (larger calls are split) */

const char* tslam_last_error(void);
int tslam_device_count(void);
/* ABI version of this header (tests check the library agrees). */
int tslam_abi_version(void);
#define TSLAM_ABI_VERSION 6

/* ----------------------------------------------------------------------------
 * TSDF map  (DenseTSDF, dense_tsdf.py)
 * --------------------------------------------------------------------------*/
typedef struct tslam_tsdf tslam_tsdf_t;

typedef struct tslam_tsdf_config {
  double voxel_scale;        /* dense_tsdf.py:13 voxel_scale                         */
  int32_t N, Nz;             /* grid edge in voxels, dense_tsdf.py:24-25             */
  double max_ray_length;     /* dense_tsdf.py:14                                     */
  double min_ray_length;     /* dense_tsdf.py:14                                     */
  int32_t internal_voxels;   /* dense_tsdf.py:15                                     */
  int32_t recast_step;       /* dense_tsdf.py:16                                     */
  double fx, fy, cx, cy;     /* K_cam_dep[0],[4],[2],[5]  mapping_common.py:33-36    */
  int32_t is_global_map;     /* dense_tsdf.py:15                                     */
  double disp_floor, disp_ceiling; /* dense_tsdf.py:16                               */
  int32_t max_submaps;       /* dense_tsdf.py:15 max_submap_num                      */
  int32_t max_blocks;        /* capacity of the 16^3 voxel-block pool (0 = derive)   */
  int32_t max_image_pixels;  /* largest h*w a depth frame may have (0 = 640*480)     */
  int32_t max_points;        /* largest point cloud for integrate_points (0 = 1<<20) */
  int32_t texture_enabled;   /* dense_tsdf.py:13 texture_enabled: colour planes + colour fusion        */
} tslam_tsdf_config_t;

/* DenseTSDF.__init__ / initialize_fields (dense_tsdf.py:13-118). */
int tslam_tsdf_create(const tslam_tsdf_config_t* cfg, tslam_tsdf_t** out);
int tslam_tsdf_destroy(tslam_tsdf_t* m);
/* DenseTSDF.reset(): B.parent().deactivate_all() (dense_tsdf.py:309-310). */
int tslam_tsdf_reset(tslam_tsdf_t* m, void* stream);
/* BaseMap.set_dep_camera_intrinsic (mapping_common.py:25-26). */
int tslam_tsdf_set_intrinsics(tslam_tsdf_t* m, double fx, double fy, double cx, double cy);
/* BaseMap.set_base_pose_submap_kernel (mapping_common.py:126-131): pose table row s. */
int tslam_tsdf_set_submap_pose(tslam_tsdf_t* m, int32_t s, const float* R9, const float* T3);

/* DenseTSDF.recast_depth_to_map -> recast_depth_to_map_kernel (dense_tsdf.py:162-165,
 * :188-214) for a batch of n_frames frames.  depth: uint16 [n_frames,h,w] millimetres;
 * R9s/T3s: HOST arrays [n_frames,9]/[n_frames,3] = input_R/input_T after set_pose's
 * convert_by_base + f32 cast (mapping_common.py:149-156); submap_ids: HOST int32
 * [n_frames] (active_submap_id per frame) or NULL for all-zero.
 * flags: TSLAM_F_COMMIT applies the pending weighted averages before returning
 * control to the stream (otherwise they stay pending until tslam_tsdf_commit or any
 * reader).  The per-frame bucket grid (PCLroot.deactivate_all, :163) is implicit. */
#define TSLAM_F_COMMIT 1
int tslam_tsdf_integrate_depth(tslam_tsdf_t* m, const uint16_t* depth, int mem, int32_t n_frames, int32_t h, int32_t w,
                               const float* R9s, const float* T3s, const int32_t* submap_ids, int flags, void* stream);
/* Per-frame form of the same call, for callers that hand over one frame at a time (the reference API):
 * copies ONE host frame to a device staging slot on an internal copy stream (overlapping the kernels of the
 * previous launch) and records its pose; every TSLAM_MAX_BATCH/2 queued frames (TSLAM_QUEUE_LAUNCH="a,b" in the
 * environment alternates other counts) - or tslam_tsdf_flush, which every reader calls implicitly - are integrated
 * and committed with one launch triple, so the kernels of one half run while the caller hands over the next.
 * The frame has been consumed when the call returns (the reference's semantics: its kernel launch copies the array
 * synchronously): a page-locked source is DMA-copied and the copy awaited; of a pageable source the sampled rows (every
 * recast_step-th row) are copied into a page-locked ring of the library with streaming stores, from where the GPU
 * fetches them.  (Environment, A/B only: TSLAM_FRAME_COPY=dma hands pageable frames to cudaMemcpyAsync;
 * TSLAM_PINNED_COPY=ring|fetch sends page-locked frames through the ring / awaits a row fetch inside the call.)
 * tslam_tsdf_set_frame_mode(m, 1) (or TSLAM_ZERO_COPY=1 in the environment) opts into BORROWING page-locked frames
 * instead: they are not copied at all, the GPU fetches their sampled rows (every recast_step-th row) straight from
 * host memory a few calls later - half the PCIe bytes for recast_step 2, no wait per frame - and they must then stay
 * valid and unchanged until tslam_tsdf_flush has returned and the stream has been synchronised, or until
 * 2*TSLAM_MAX_BATCH further frames have been queued (the call blocks rather than letting the host run further ahead). */
int tslam_tsdf_queue_depth(tslam_tsdf_t* m, const uint16_t* depth_host, int32_t h, int32_t w, const float* R9,
                           const float* T3, int32_t submap, void* stream);
int tslam_tsdf_flush(tslam_tsdf_t* m, void* stream);
int tslam_tsdf_set_frame_mode(tslam_tsdf_t* m, int borrow_pinned);
/* The same hand-over in two halves, so that the caller's own per-frame work (DenseTSDF.recast_depth_to_map: the f64 pose
 * arithmetic of convert_by_base, mapping_common.py:91-100) runs while the frame's DMA copy is in flight: _begin starts
 * the copy, _end awaits it (the frame has been consumed when _end returns), records the pose and launches a full
 * queue.  No other call on the handle between the two. */
int tslam_tsdf_queue_depth_begin(tslam_tsdf_t* m, const uint16_t* depth_host, int32_t h, int32_t w, void* stream);
int tslam_tsdf_queue_depth_end(tslam_tsdf_t* m, const float* R9, const float* T3, int32_t submap, void* stream);
/* Frames per queue launch, alternating a, b, a, ... (default TSLAM_MAX_BATCH/2 each).  Every launch ends with a commit:
 * the granule of the Wmax clamp (dense_tsdf.py:267).  (1, 1) = one commit per frame - what a frame-by-frame caller of
 * the reference sees below Wmax, and the closest a summed update gets to its per-sample clamp at Wmax
 * (tests/test_oracle_vs_reference_exec.py::test_commit_granularity_vs_per_sample_clamp_at_wmax) - at the price of
 * one launch sequence per frame. */
int tslam_tsdf_set_queue_launch(tslam_tsdf_t* m, int32_t frames_a, int32_t frames_b);
/* Textured maps (texture_enabled).  set_color_camera_intrinsic (mapping_common.py:28-29) + color_same_proj
 * (dense_tsdf.py:16).  The *_tex / *_rgb forms take the colour image uint8 [n_frames,th,tw,3] (channel order as
 * given - DenseTSDF does not swap BGR) or per-point colours uint8 [n,3]; tex == NULL integrates geometry only.
 * Colour semantics: the reference overwrites color[xi] at every sample, racing rays, last writer wins
 * (dense_tsdf.py:268-269); here the winner is deterministic: latest frame, then the sample closest to its ray's
 * surface point (DESIGN.md "Texture"). */
int tslam_tsdf_set_color_intrinsics(tslam_tsdf_t* m, double fx, double fy, double cx, double cy, int color_same_proj);
int tslam_tsdf_integrate_depth_tex(tslam_tsdf_t* m, const uint16_t* depth, const uint8_t* tex, int mem, int32_t n_frames, int32_t h,
                                   int32_t w, int32_t th, int32_t tw, const float* R9s, const float* T3s, const int32_t* submap_ids,
                                   int flags, void* stream);
int tslam_tsdf_queue_depth_tex(tslam_tsdf_t* m, const uint16_t* depth_host, const uint8_t* tex_host, int32_t h, int32_t w, int32_t th,
                               int32_t tw, const float* R9, const float* T3, int32_t submap, void* stream);
int tslam_tsdf_integrate_points_rgb(tslam_tsdf_t* m, const float* xyz, const uint8_t* rgb, int mem, int32_t n, const float* R9,
                                    const float* T3, int32_t submap, int flags, void* stream);
/* to_numpy / load_numpy with the colour column (dense_tsdf.py:437-440, :450-453): color f32[cap,3] DEVICE or NULL. */
int tslam_tsdf_gather2(tslam_tsdf_t* m, int32_t submap, int64_t cap, int32_t* idx, float* tsdf, float* w, int8_t* occ, float* color,
                       int64_t* n_out, void* stream);
int tslam_tsdf_scatter2(tslam_tsdf_t* m, int32_t submap, int64_t n, const int32_t* idx, const float* tsdf, const float* w,
                        const int8_t* occ, const float* color, void* stream);
/* DenseTSDF.recast_pcl_to_map -> recast_pcl_to_map_kernel (dense_tsdf.py:157-160, :167-186).
 * xyz: float32 [n,3]. */
int tslam_tsdf_integrate_points(tslam_tsdf_t* m, const float* xyz, int mem, int32_t n, const float* R9, const float* T3,
                                int32_t submap, int flags, void* stream);
/* Apply pending per-voxel weighted averages: T' = (T*W + sum w*d)/(W + sum w),
 * W' = min(W + sum w, Wmax=1000)  (dense_tsdf.py:264-267 applied once per voxel). */
int tslam_tsdf_commit(tslam_tsdf_t* m, void* stream);

/* DenseTSDF.count_active (dense_tsdf.py:412-423).  Synchronises. */
int tslam_tsdf_count_active(tslam_tsdf_t* m, int32_t submap, int64_t* n_out);
/* DenseTSDF.to_numpy (dense_tsdf.py:425-440): observed voxels of `submap` into
 * caller DEVICE arrays idx int32[cap,3], tsdf f32[cap], w f32[cap], occ int8[cap]
 * (row order unspecified, like the reference's atomic counter).  *n_out = demand.
 * Synchronises.  Returns TSLAM_E_CAPACITY (outputs saturated) when demand > cap. */
int tslam_tsdf_gather(tslam_tsdf_t* m, int32_t submap, int64_t cap, int32_t* idx, float* tsdf, float* w, int8_t* occ,
                      int64_t* n_out, void* stream);
/* DenseTSDF.load_numpy (dense_tsdf.py:442-454): DEVICE arrays, n rows. */
int tslam_tsdf_scatter(tslam_tsdf_t* m, int32_t submap, int64_t n, const int32_t* idx, const float* tsdf, const float* w,
                       const int8_t* occ, void* stream);
/* DenseTSDF.fuse_submaps -> reset() + fuse_submaps_kernel (dense_tsdf.py:272-318):
 * trilinear splat (7 corners, :300) of every observed voxel of every submap of `src`
 * into submap 0 of `dst`, using dst's pose table.  No Wmax clamp (:274-278). */
int tslam_tsdf_fuse(tslam_tsdf_t* dst, tslam_tsdf_t* src, void* stream);
/* Incremental fusion of the submaps of `src` into the global map `dst` (DESIGN.md section 7, "Incremental global
 * fusion"): an opt-in alternative to tslam_tsdf_fuse that keeps exact int64 sums (24 B per voxel, 48 B textured, grown
 * with the pool blocks in use) of the terms k_fuse splats, each quantised to llrint(f * 2^24), and re-reads only the
 * blocks a call changed.  After the call dst equals the fusion of every submap s with include[s] != 0 (include: host,
 * max_submaps bytes; NULL = all) at its fused pose: dst's base pose of s, unless s was fused before with the same
 * content and |T - T0| + angle(R0^T R) * r_s <= tolerance (r_s: farthest allocated block corner of s from its origin;
 * tolerance 0: iff the pose bits are unchanged).  The result does not depend on the history of calls.  A full update
 * (reset, then add every included submap) runs on the first call, when full != 0, for another src, after any other
 * write of dst, when a fused submap's content changed, and when subtracting and re-adding would splat more source
 * blocks than a rebuild; both paths give the same bits.  Differences from tslam_tsdf_fuse: the quantisation, occ
 * saturates once on the total, and blocks left empty by removals stay allocated (a full update compacts them).
 * stats8 (may be NULL): full-update reason (0 incremental, 1 first call, 2 full requested, 3 other src, 4 dst written,
 * 5 content changed, 6 cheaper than subtract and re-add), submaps added, moved, removed, left within tolerance, source
 * voxels splatted (adds + subtracts), source voxels skipped (a term not finite or >= 2^23), blocks committed.
 * Refused (TSLAM_E_INVALID, nothing written), before the handles are looked at: tolerance not finite or < 0, a NULL
 * handle, dst == src; then a dst that is not a global map, different max_submaps, voxel size or texture setting,
 * and a tiled dst (tile cuts set or ghost blocks).  TSLAM_E_CUDA (byte count in tslam_last_error) when the sum planes
 * cannot grow; TSLAM_E_POOL_FULL when dst's pool runs out (nothing added; the next call is a full update).
 * Synchronises with `stream`. */
int tslam_tsdf_fuse_update(tslam_tsdf_t* dst, tslam_tsdf_t* src, const uint8_t* include, float tolerance, int32_t full,
                           int64_t* stats8, void* stream);
/* Reclaim pool blocks (DESIGN.md section 7, "Reclaiming pool blocks"): drop blocks and compact the pool in place.
 * Queued frames are integrated and pending sums committed first.  A block is a candidate when submaps[s] != 0 for its
 * submap s (submaps: host, max_submaps bytes; NULL = every submap).  A candidate is dropped when
 *   TSLAM_RECLAIM_ALL is set, or
 *   TSLAM_RECLAIM_EMPTY is set and the block is empty: no voxel has obs != 0, no commit is pending for it, and, on a
 *     fusion destination whose sums are valid, every sum word of the block is zero (obs 0 with a non-zero sum is kept), or
 *   TSLAM_RECLAIM_OUTSIDE is set and the block lies outside the sphere (center3, radius): with the voxel positions
 *     p = (double)((float)i * vs) of the frame the map stores the submap in (the map frame of a global map; the submap's
 *     own frame, before its base pose, in a collection), the block (b, voxels 16 b .. 16 b + 15 per axis) is outside iff
 *     (d_x^2 + d_y^2) + d_z^2 > radius^2 in f64, d = c - clamp(c, p(16 b), p(16 b + 15)) per axis.  A block that touches
 *     the sphere exactly is kept.
 * Compaction: n_keep = kept blocks.  Holes (dropped slots below n_keep) and movers (kept slots at or above n_keep) are
 * paired in ascending order, and the k-th mover moves to the k-th hole with every per-block state: key, acc, tw, obs,
 * occ, colour word and colour, ESDF, dirty flags, commit stamp and the fusion sum planes.  Kept blocks below n_keep stay
 * put.  [n_keep, n_old) of every plane is zeroed, n_blocks = n_keep, and the hash table is rebuilt from the kept keys
 * (keys that failed on a full pool can allocate again).  When a block was dropped, the next tslam_mesh_update and ESDF
 * update are full ones, and every submap that lost a non-empty block counts as written for tslam_tsdf_fuse_update
 * (dropping empty blocks does not; an EMPTY reclaim of a fusion destination keeps its next update incremental).  When
 * nothing is dropped, nothing is moved or invalidated.
 * stats6 (host, may be NULL): blocks before, candidates, dropped, dropped non-empty, moved, blocks after.
 * Refused (TSLAM_E_INVALID, nothing written, before the handle is read): rules 0 or with unknown bits; with OUTSIDE a
 * radius that is negative or not finite, or a NULL or non-finite centre; a NULL handle.  Then: a tiled map (tile cuts
 * set, or ghost blocks), an open tiled ESDF exchange, a tiled fusion update in progress.  Synchronises with `stream`. */
#define TSLAM_RECLAIM_ALL 1
#define TSLAM_RECLAIM_EMPTY 2
#define TSLAM_RECLAIM_OUTSIDE 4
int tslam_tsdf_reclaim(tslam_tsdf_t* m, int32_t rules, const uint8_t* submaps, const double* center3, double radius,
                       int64_t* stats6, void* stream);
/* The pool in slot order: keys4 (DEVICE int32[cap, 4]) row b = (submap, bx, by, bz) of pool block b, b < n_blocks.
 * Pending work is flushed first.  *n_out = n_blocks; TSLAM_E_CAPACITY (rows saturated) when it exceeds cap.  Synchronises. */
int tslam_tsdf_block_keys(tslam_tsdf_t* m, int64_t cap, int32_t* keys4, int64_t* n_out, void* stream);
/* cvt_TSDF_surface_to_voxels_kernel (dense_tsdf.py:339-365): append |TSDF|<1.8*vs
 * voxels of `submap` to xyz/rgb f32[cap,3] (DEVICE) starting at *count_dev (DEVICE
 * int32 counter, incremented; entries beyond cap are counted but not written). */
int tslam_tsdf_extract_surface(tslam_tsdf_t* m, int32_t submap, int64_t cap, float* xyz, float* rgb, int32_t* count_dev,
                               void* stream);
/* cvt_TSDF_to_voxels_slice_kernel (dense_tsdf.py:367-385). val = TSDF value. */
int tslam_tsdf_extract_slice(tslam_tsdf_t* m, int32_t submap, float z, float dz, int64_t cap, float* xyz, float* val,
                             float* rgb, int32_t* count_dev, void* stream);
/* Counters since the last clear: [0] sampled pixels, [1] valid pixels (range filter),
 * [2] rays (live buckets), [3] voxel updates applied, [4] out-of-volume samples,
 * [5] allocated voxel blocks, [6] device error flags, [7] integrate launches.
 * Synchronises. */
int tslam_tsdf_get_stats(tslam_tsdf_t* m, int64_t* out8, int clear);
/* Block until all work enqueued on `stream` for this map is done and report a
 * deferred device error (TSLAM_E_POOL_FULL) if one was raised. */
int tslam_tsdf_sync(tslam_tsdf_t* m, void* stream);
/* Kernels launched by this handle since creation (bench.py `gpu_launches`). */
int64_t tslam_tsdf_launch_count(tslam_tsdf_t* m);
/* Timing of the integrate kernels when profiling is on (ring of the last 512 integrate launches): each kernel
 * stamps the GPU's global timer at the entry of its first CTA and the exit of its last one; nothing is recorded on
 * the stream.  A stage is charged from the later of its first kernel's start and the end of the stage before it,
 * to its last kernel's end, so the columns of a launch never sum to more than its span.  tslam_tsdf_kernel_ms writes
 * ms3[3*i+{0,1,2}] = bucket / ray-march / commit time of the i-th most recent launch (commit 0 for a launch
 * without one), i < min(n, recorded); *n_out = rows written.  Synchronises. */
int tslam_tsdf_set_profiling(tslam_tsdf_t* m, int on);
int tslam_tsdf_kernel_ms(tslam_tsdf_t* m, int32_t n, float* ms3, int32_t* n_out);
/* Same ring, 7 columns per launch: bucket, ray march (all its kernels), commit, 0, then the ray march split into
 * ray set-up + counting walk + class + scan / scattering walk / block march (tslam_march.cu; zeros for textured
 * maps, which march with one thread per ray). */
int tslam_tsdf_kernel_ms2(tslam_tsdf_t* m, int32_t n, float* ms7, int32_t* n_out);
/* Diagnostics of the block-binned ray march (process_new_pcl, dense_tsdf.py:236-270) since the last clear of
 * tslam_tsdf_get_stats: out6 = segments, work items, samples that took the exact-index path (fraction within
 * near_eps of .5), samples applied through a global reduction because their exact voxel lies outside the work
 * item's block, samples of the generic path, fast-path indices that disagreed with the exact index
 * (TSLAM_MARCH_VERIFY=1 only; must be 0).  Synchronises. */
int tslam_tsdf_get_march_stats(tslam_tsdf_t* m, int64_t* out6);
/* The same six, then out7[6] = segments the counting and the scattering walk of the binned march disagreed about:
 * routed to the generic path by a guard of the scattering walk, or counted but never placed.  Must be 0. */
int tslam_tsdf_get_march_stats2(tslam_tsdf_t* m, int64_t* out7);

/* ----------------------------------------------------------------------------
 * Map queries for planners - batched forms of the @ti.func helpers of BaseMap (mapping_common.py:165-204) that
 * TopoGraphGen calls from its kernels (topo_graph.py:444-507).  All arrays DEVICE, n entries.
 * --------------------------------------------------------------------------*/
/* flags[i]: bit0 = is_pos_occupy (TSDF < 1.8*vs, dense_tsdf.py:152-155 - unobserved space reads 0, i.e. occupied),
 * bit1 = is_pos_unobserved (dense_tsdf.py:148-150). */
int tslam_tsdf_query_points(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* xyz, uint8_t* flags, void* stream);
/* is_near_pos_occupy (mapping_common.py:193-204): any occupied cell in [-voxel, voxel)^3 around the point. */
int tslam_tsdf_query_near_occupy(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* xyz, int32_t voxel, uint8_t* out, void* stream);
/* raycast (mapping_common.py:165-178): step voxel_scale along dir until an occupied cell; hit, last position, length. */
int tslam_tsdf_raycast(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* pos, const float* dir, float max_dist, uint8_t* hit,
                       float* xyz_out, float* len_out, void* stream);

/* ----------------------------------------------------------------------------
 * Multi-GPU: spatially tiled global map (one process per GPU; SURVEY.md section 8e).  The global volume is cut into
 * tiles3[0] x tiles3[1] x tiles3[2] == world tiles of whole 16^3 blocks, tile t owned by rank t.  The library
 * packs / unpacks voxel blocks into caller DEVICE buffers; the caller exchanges them (NCCL all-to-all).
 * Keys are the library's packed block keys (opaque int64).  Planes per block: 4096 voxels.
 * --------------------------------------------------------------------------*/
/* fuse_submaps_kernel (dense_tsdf.py:282-307) of this rank's submaps, sums left PENDING (no commit). */
int tslam_tsdf_fuse_pending(tslam_tsdf_t* dst, tslam_tsdf_t* src, void* stream);
/* Fold pending fusion sums (no Wmax clamp, dense_tsdf.py:274-278). */
int tslam_tsdf_commit_fused(tslam_tsdf_t* m, void* stream);
/* Owner rank of block (bx,by,bz). */
int tslam_tiling_owner(tslam_tsdf_t* m, const int32_t* tiles3, int32_t world, int32_t bx, int32_t by, int32_t bz, int32_t* owner);
/* Tile boundaries.  By default the volume is cut into equal slices; tslam_tiling_set_cuts installs block-coordinate
 * cuts per axis (cuts_a[k] .. cuts_a[k+1]-1 = tile k, tiles3[a]+1 strictly increasing values; NULL tiles3 = back to
 * the default) - the host layer derives them from the occupied blocks (tslam_tsdf_dirty_hist: HOST int32[3][1024],
 * histogram of the block coordinates + 512 of the blocks touched since the last commit, per axis) so that a flat
 * flight volume does not leave half the ranks without surface.  Every rank must install the same cuts. */
int tslam_tiling_set_cuts(tslam_tsdf_t* m, const int32_t* tiles3, const int32_t* cuts_x, const int32_t* cuts_y, const int32_t* cuts_z);
int tslam_tsdf_dirty_hist(tslam_tsdf_t* m, int32_t* hist3x1024, void* stream);
/* counts_out[world] (HOST): touched blocks owned by every other rank.  Synchronises. */
int tslam_tsdf_foreign_count(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, int32_t* counts_out, void* stream);
/* Pack those blocks grouped by destination rank and clear them locally: keys int64[cap], acc f32[cap,4096,2]
 * (pending sums), obs u8[cap,4096], occ i8[cap,4096].  Synchronises. */
int tslam_tsdf_foreign_pack(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts,
                            int64_t cap, int64_t* keys, float* acc, uint8_t* obs, int8_t* occ, void* stream);
/* Add received blocks into the local map (sums stay pending until tslam_tsdf_commit_fused). */
int tslam_tsdf_unpack_add(tslam_tsdf_t* m, int64_t n, const int64_t* keys, const float* acc, const uint8_t* obs, const int8_t* occ,
                          void* stream);
/* Halo for meshing: blocks of the one-block boundary layer of this rank's tile, once per neighbouring tile. */
int tslam_tsdf_halo_count(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, int32_t* counts_out, void* stream);
int tslam_tsdf_halo_pack(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts, int64_t cap,
                         int64_t* keys, float* tw, uint8_t* obs, void* stream);
/* Insert received halo blocks as GHOSTS: read by marching cubes, never counted / exported / meshed as owners. */
int tslam_tsdf_ghost_unpack(tslam_tsdf_t* m, int64_t n, const int64_t* keys, const float* tw, const uint8_t* obs, void* stream);
/* Textured maps (colour is fused with the geometry, dense_tsdf.py:276-277): the same four calls with the colour
 * plane f32[cap,4096,4] riding along (pending sum of w*colour for the fusion exchange, committed colour for the halo).
 * col must be given for a textured map and NULL for an untextured one. */
int tslam_tsdf_foreign_pack2(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts,
                             int64_t cap, int64_t* keys, float* acc, uint8_t* obs, int8_t* occ, float* col, void* stream);
int tslam_tsdf_unpack_add2(tslam_tsdf_t* m, int64_t n, const int64_t* keys, const float* acc, const uint8_t* obs, const int8_t* occ,
                           const float* col, void* stream);
int tslam_tsdf_halo_pack2(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts, int64_t cap,
                          int64_t* keys, float* tw, uint8_t* obs, float* col, void* stream);
int tslam_tsdf_ghost_unpack2(tslam_tsdf_t* m, int64_t n, const int64_t* keys, const float* tw, const uint8_t* obs, const float* col,
                             void* stream);
/* Query routing: owner[n] (DEVICE int32) = owner rank of the block that holds the low interpolation corner of each
 * point xyz f32[n,3] (DEVICE) - the corner tslam_esdf_query starts from, computed by the same f32 expression - or -1
 * for a point that is not finite or whose low corner lies outside the volume (any rank answers those: invalid). */
int tslam_tiling_owner_points(tslam_tsdf_t* m, const int32_t* tiles3, int32_t world, int64_t n, const float* xyz, int32_t* owner,
                              void* stream);
/* Planner queries of the tiled map (DESIGN.md section 6).  Every answer is bit-identical to the same query on one map
 * holding every tile; the host layer routes the points / rays (TiledGlobalMap.raycast, is_pos_occupy, ...).
 * tslam_tiling_owner_cells: owner[n] (DEVICE int32) = owner rank of the block holding the cell round(x / vs) of each
 * point xyz f32[n,3] (DEVICE) - the cell tslam_tsdf_query_points / _query_near_occupy read, by the same f32 expression -
 * or -1 for a cell outside the volume (it reads occupied and unobserved on any rank). */
int tslam_tiling_owner_cells(tslam_tsdf_t* m, const int32_t* tiles3, int32_t world, int64_t n, const float* xyz, int32_t* owner,
                             void* stream);
/* One round of tslam_tsdf_raycast on a tiled map.  ray f32[n,8] (DEVICE, in/out) = pos[3], dir[3], max_dist, next
 * sample j (int32 bits; 0 for a new ray).  Marches each ray from sample j while the sample's cell lies in a block this
 * rank owns (ghosts are not read).  A ray that reaches a block of another rank gets dest[i] = that rank and its j
 * written back into row i; route the row there and call again.  A ray that hits, leaves the volume or runs out of
 * steps (int)(max_dist / vs) gets dest[i] = -1 and the answer of tslam_tsdf_raycast in row i of hit u8[n] /
 * xyz_out f32[n,3] / len_out f32[n]; those rows are untouched for a handed-over ray.  A batch is done after at most
 * tx+ty+tz-2 hand-over rounds (DESIGN.md section 6).  Does not synchronise. */
int tslam_tsdf_raycast_tiled(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, int32_t submap, int64_t n, float* ray,
                             int32_t* dest, uint8_t* hit, float* xyz_out, float* len_out, void* stream);
/* tslam_tsdf_query_near_occupy that also reads ghost blocks, for points routed to the owner of their centre cell
 * (tslam_tiling_owner_cells).  The answer is exact when the ghosts carry the current TSDF - a halo exchange after the
 * last fusion, which the host layer runs first - and voxel is in [0, 16]: the window then stays within the blocks next
 * to the centre cell's block, all of which the halo brings.  TSLAM_E_INVALID for voxel outside [0, 16]. */
int tslam_tsdf_query_near_occupy_tiled(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* xyz, int32_t voxel, uint8_t* out,
                                       void* stream);
/* ESDF of the tiled map (DESIGN.md section 6).  Always a full recompute of `submap`, exact: the result is bit-identical
 * to tslam_esdf_update2 on one map holding every tile.  Run a TSDF halo exchange first (ghosts must carry the current
 * TSDF), then on every rank:
 *   tslam_esdf_tiled_begin                  seed owned and ghost blocks, local wave to convergence; ghost blocks are
 *                                           read-only sources.  Synchronises.
 *   repeat: tslam_esdf_halo_count / _pack   owned boundary blocks (the TSDF halo's blocks and destinations) whose ESDF
 *                                           changed since they were last packed - after begin, all of them - into
 *                                           keys int64[cap] / esdf f32[cap,4096] (DEVICE) grouped by destination;
 *                                           packing clears the mark.  Synchronises.  TSLAM_E_CAPACITY: saturated,
 *                                           the blocks that did not fit stay marked.
 *           exchange (all-to-all), then tslam_esdf_ghost_unpack: overwrite the ESDF of existing ghost blocks (never
 *                                           allocates).  A key that is not a ghost block of the submap writes nothing
 *                                           and makes the call return TSLAM_E_INVALID.  Synchronises.
 *           tslam_esdf_tiled_relax          the wave from the ghosts unpacked since the last relax.  Synchronises.
 *   until every rank packed 0 blocks;  tslam_esdf_tiled_end.
 * n_sweeps_out (HOST, may be NULL) as tslam_esdf_update.  Between begin and end tslam_esdf_query / _extract_slice
 * return TSLAM_E_INVALID; after end tslam_esdf_query also reads corners in ghost blocks (after a plain update they stay
 * invalid), until the next reset, load, fusion, ghost import or update.  An update after a tiled ESDF is full. */
int tslam_esdf_tiled_begin(tslam_tsdf_t* m, int32_t submap, int32_t* n_sweeps_out, void* stream);
int tslam_esdf_halo_count(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, int32_t* counts_out, void* stream);
int tslam_esdf_halo_pack(tslam_tsdf_t* m, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts, int64_t cap,
                         int64_t* keys, float* esdf, void* stream);
int tslam_esdf_ghost_unpack(tslam_tsdf_t* m, int64_t n, const int64_t* keys, const float* esdf, void* stream);
int tslam_esdf_tiled_relax(tslam_tsdf_t* m, int32_t* n_sweeps_out, void* stream);
int tslam_esdf_tiled_end(tslam_tsdf_t* m);
/* Incremental fusion of a tiled global map (DESIGN.md section 6, "Incremental tiled fusion"): tslam_tsdf_fuse_update
 * over the ranks.  Rank r's `src` holds the submaps r contributes; every rank's dst has the pose table of all of them.
 * Terms, quantisation, skip rule, int64 sums and readout are tslam_tsdf_fuse_update's.  The sums of a dst block live
 * on its owner only (tile_owner with the current cuts); the other ranks send the integer deltas of the blocks their
 * added, moved or removed submaps touch.  Integer sums commute, so after an update the union of the ranks' owned
 * blocks is bit for bit tslam_tsdf_fuse_update of all ranks' submaps into one map, for any world size, cuts and
 * history.  The host layer (TiledGlobalMap.update_fused_submaps) calls, on every rank:
 *   _plan     the single-map plan of this rank's submaps.  plan3 (HOST int64[3]) = local full-update reason (as
 *             tslam_tsdf_fuse_update's stats8[0], without 6; plus 7 = tile cuts changed since the last update, 8 = the
 *             sums are not valid, e.g. after a failed update), cost and cost_full (source blocks an incremental and a
 *             full update would splat); present (HOST u8[max_submaps]) = src holds blocks of the submap.  Synchronises.
 *   merge     over the ranks: a submap present on two ranks is refused; include must be the same everywhere; the
 *             update is full when any rank's reason is, or when the summed cost exceeds the summed cost_full (6); the
 *             reason is the smallest non-zero one.
 *   _splat    with the merged reason: a full update resets dst, zeroes the sums and adds every included submap; an
 *             incremental one subtracts and adds as planned, removals also activating their FOREIGN dst blocks (a
 *             removal that misses an owned block raises TSLAM_E_CUDA at the commit).  Synchronises.
 *   (full update with balanced cuts: tslam_tsdf_dirty_hist of the activated blocks, summed, new cuts installed)
 *   tslam_tsdf_foreign_count, then _pack: the sum rows of the foreign dirty blocks into rows int64[cap, 1 + planes *
 *             4096] (DEVICE; key, then planes S_wT, S_w, count * 2^32 + S_occ and, textured, S_c[3]) grouped by owner;
 *             they are zeroed here.  An incremental update refuses cuts that changed since _plan.  Synchronises.
 *   exchange (all-to-all of the rows), then
 *   _unpack   n received rows: activate their blocks (TSLAM_E_POOL_FULL when the pool runs out), add them into the
 *             sums with wrapping int64 adds, read the touched owned blocks out of the sums (stamped for
 *             tslam_mesh_update, ESDF-dirty).  A voxel whose count decodes as negative: TSLAM_E_CUDA.  Synchronises.
 *   _finish   ok != 0 on every rank when every rank's phases succeeded: record the submaps' new state; stats8 as
 *             tslam_tsdf_fuse_update's (this rank's part).  ok = 0: nothing recorded, and when the update got past its
 *             plan the sums are invalid (the next update is full on every rank).
 * A halo exchange and a tiled ESDF between two updates do not force a full update; any other write of dst does.  A
 * removal or move makes the next ESDF update full.  Refused (TSLAM_E_INVALID) before the handles are looked at: tolerance
 * not finite or < 0, a NULL handle or plan buffer, dst == src, tiles3 NULL or not a factorisation of world (1..24, at
 * most 16 per axis), rank outside [0, world); then what tslam_tsdf_fuse_update refuses except a tiled dst, and a phase
 * called out of order or with another src than the plan. */
int tslam_tsdf_fuse_update_tiled_plan(tslam_tsdf_t* dst, tslam_tsdf_t* src, const int32_t* tiles3, int32_t rank, int32_t world,
                                      const uint8_t* include, float tolerance, int32_t full, int64_t* plan3, uint8_t* present, void* stream);
int tslam_tsdf_fuse_update_tiled_splat(tslam_tsdf_t* dst, tslam_tsdf_t* src, int32_t reason, void* stream);
int tslam_tsdf_fuse_update_tiled_pack(tslam_tsdf_t* dst, const int32_t* tiles3, int32_t rank, int32_t world, const int32_t* counts,
                                      int64_t cap, int64_t* rows, void* stream);
int tslam_tsdf_fuse_update_tiled_unpack(tslam_tsdf_t* dst, int64_t n, const int64_t* rows, void* stream);
int tslam_tsdf_fuse_update_tiled_finish(tslam_tsdf_t* dst, tslam_tsdf_t* src, int32_t ok, int64_t* stats8, void* stream);

/* ----------------------------------------------------------------------------
 * Marching cubes  (MarchingCubeMesher, marching_cube_mesher.py)
 * --------------------------------------------------------------------------*/
/* generate_mesh_kernel (marching_cube_mesher.py:127-187): two-pass (count, scan,
 * emit) marching cubes over every active block of `m`.  verts/normals: DEVICE
 * f32 [3*cap_tri,3]; *n_tri_out = true triangle demand (host).  Synchronises. */
int tslam_mc_generate(tslam_tsdf_t* m, int32_t step, float tsdf_surface_thres, int64_t cap_tri, float* verts,
                      float* normals, int64_t* n_tri_out, void* stream);
/* ... with vertex colours (vertexInterp_color / add_triangle_color, marching_cube_mesher.py:62-82, :104-108):
 * colors f32[3*cap_tri,3] DEVICE or NULL. */
int tslam_mc_generate2(tslam_tsdf_t* m, int32_t step, float tsdf_surface_thres, int64_t cap_tri, float* verts, float* normals,
                       float* colors, int64_t* n_tri_out, void* stream);
/* Incremental mesh of one map (step 1 only).  The cache keeps the mesh of its last update on the device and, on the next
 * update, remeshes only the blocks whose output a commit or ghost import since then could have changed; the rest of the
 * mesh is copied.  tslam_mesh_update has the output contract of tslam_mc_generate2(m, 1, ...): the same *n_tri_out
 * (demand), the same first min(demand, cap_tri) triangles bit for bit, the same TSLAM_E_CAPACITY and deferred
 * TSLAM_E_POOL_FULL.  It rebuilds fully on the first call, after a reset, load (scatter), fusion or fusion exchange of
 * the map, and when thres or the colour mode (colors NULL or not) changes.  stats4 (HOST, may be NULL) = pool blocks,
 * stamped blocks, touched blocks, remeshed blocks (a full rebuild: 0 stamped and touched, every block remeshed).
 * Synchronises.  A cache belongs to its map and must be destroyed before it. */
typedef struct tslam_mesh tslam_mesh_t;
int tslam_mesh_create(tslam_tsdf_t* m, tslam_mesh_t** out);
int tslam_mesh_destroy(tslam_mesh_t* c);
int tslam_mesh_update(tslam_mesh_t* c, float tsdf_surface_thres, int64_t cap_tri, float* verts, float* normals, float* colors,
                      int64_t* n_tri_out, int32_t* stats4, void* stream);
/* The blocks remeshed by the last update, in pool order: blk4 int32[cap,4] = submap, bx, by, bz; first_tri int64[cap] and
 * n_tri int32[cap] = their range in the update's output (demand numbering: a range may reach past a saturated cap_tri)
 * (all DEVICE).  n_tri 0: the block's mesh is now empty.  The list is a superset of the blocks whose triangles changed.
 * *full_out (HOST, may be NULL) = 1 after a full rebuild: every block is listed and the consumer drops what it kept.
 * *n_out (HOST) = blocks; rows beyond cap are not written (TSLAM_E_CAPACITY).  TSLAM_E_INVALID before the first
 * completed update.  Synchronises. */
int tslam_mesh_updated_blocks(tslam_mesh_t* c, int64_t cap, int32_t* blk4, int64_t* first_tri, int32_t* n_tri, int64_t* n_out,
                              int32_t* full_out, void* stream);

/* ----------------------------------------------------------------------------
 * ESDF  (DenseSDF.propogate_esdf semantics, dense_esdf.py:228-333; see DESIGN.md)
 * --------------------------------------------------------------------------*/
/* Converged 26-neighbour signed distance wavefront over the observed voxels of
 * `submap`.  *n_sweeps_out (host, optional) = global sweeps until no change. */
int tslam_esdf_update(tslam_tsdf_t* m, int32_t submap, int32_t* n_sweeps_out, void* stream);
/* Same with control and statistics.  mode 0: INCREMENTAL when the kept state allows it (same submap as the previous
 * update, no reset / load_numpy / ghost import since) - only the voxels that changed since the last update, the voxels
 * whose value may have been derived from them (raise wave) and whatever those lower again are recomputed; the result
 * is bit-identical to a full recompute.  mode 1: full recompute.  stats4 (HOST, may be NULL): lower sweeps,
 * raise sweeps (-1 = the update was full), changed voxels, suspect voxels.  Synchronises. */
int tslam_esdf_update2(tslam_tsdf_t* m, int32_t submap, int32_t mode, int32_t* stats4, void* stream);
/* ESDF of observed voxels: idx int32[cap,3], esdf f32[cap] (DEVICE). Synchronises. */
int tslam_esdf_gather(tslam_tsdf_t* m, int32_t submap, int64_t cap, int32_t* idx, float* esdf, int64_t* n_out,
                      void* stream);
/* Reading the field.  Both calls answer from the field as of the last tslam_esdf_update* of `submap`: integrating
 * more frames does not change their answers until the next update, and voxels of blocks allocated since then count
 * as unknown.  Both return TSLAM_E_INVALID when no update has completed, when the last update was for another
 * submap, or when a reset, load (scatter), fusion or ghost import has happened since.  Neither synchronises.
 *
 * Batched distance and gradient queries (what Voxblox answers for planners).  xyz f32[n,3] (DEVICE) are points in
 * the submap's own map frame - voxel i is centred at i*voxel_scale, no submap base pose is applied - like the other
 * planner queries.  Per point: dist f32[n] = trilinear interpolation of the ESDF over the 8 voxels around the point,
 * grad f32[n,3] = the exact partial derivatives of that interpolant (m/m), valid u8[n] = 1 when it is defined.
 * Undefined (valid 0, dist and grad NaN): a non-finite coordinate, a corner outside the volume, a corner that was
 * unobserved at the last update or whose TSDF was NaN.  n == 0 is a no-op. */
int tslam_esdf_query(tslam_tsdf_t* m, int32_t submap, int64_t n, const float* xyz, float* dist, float* grad,
                     uint8_t* valid, void* stream);
/* cvt_ESDF_to_voxels_slice (dense_esdf.py:498-509): the voxels of `submap` that were observed at the last update
 * and whose uncentred index k + Nz/2 lies strictly within 0.5 of _index = (z + map_size_z/2)/voxel_scale (f32),
 * appended to xyz f32[cap,3] / val f32[cap] (ESDF) at *count_dev (DEVICE int32 counter, incremented; rows beyond
 * cap are counted but not written).  Positions as tslam_tsdf_extract_slice. */
int tslam_esdf_extract_slice(tslam_tsdf_t* m, int32_t submap, float z, int64_t cap, float* xyz, float* val,
                             int32_t* count_dev, void* stream);

/* ----------------------------------------------------------------------------
 * Octomap = per-voxel hit counter  (Octomap, taichi_octomap.py)
 * --------------------------------------------------------------------------*/
typedef struct tslam_octo tslam_octo_t;
typedef struct tslam_octo_config {
  double voxel_scale;       /* the CONSTRUCTOR's voxel_scale (mapping_common.py:22-23) */
  int32_t N, Nz, K;         /* taichi_octomap.py:19-27                                 */
  double max_ray_length, min_ray_length;
  int32_t recast_step;
  double fx, fy, cx, cy;
  int32_t min_occupy_thres; /* taichi_octomap.py:30,86-88                              */
  int32_t max_submaps;
  int32_t max_blocks;       /* capacity of the 8^3 counter-block pool (0 = derive)     */
  int32_t max_image_pixels;
  int32_t max_points;
  int32_t texture_enabled;  /* taichi_octomap.py:34,77-79: per-voxel colour                */
} tslam_octo_config_t;

int tslam_octo_create(const tslam_octo_config_t* cfg, tslam_octo_t** out);
int tslam_octo_destroy(tslam_octo_t* m);
int tslam_octo_reset(tslam_octo_t* m, void* stream); /* root.deactivate_all() taichi_octomap.py:210-211 */
int tslam_octo_set_submap_pose(tslam_octo_t* m, int32_t s, const float* R9, const float* T3);
/* BaseMap.set_dep_camera_intrinsic (mapping_common.py:25-26). */
int tslam_octo_set_intrinsics(tslam_octo_t* m, double fx, double fy, double cx, double cy);
/* recast_pcl_to_map_kernel (taichi_octomap.py:134-145): occupy[round((R p + T)/vs)] += 1. */
int tslam_octo_integrate_points(tslam_octo_t* m, const float* xyz, int mem, int32_t n, const float* R9, const float* T3,
                                int32_t submap, void* stream);
/* recast_depth_to_map_kernel (taichi_octomap.py:147-169). */
int tslam_octo_integrate_depth(tslam_octo_t* m, const uint16_t* depth, int mem, int32_t h, int32_t w, const float* R9,
                               const float* T3, int32_t submap, void* stream);
/* Textured octomaps (texture_enabled): process_point overwrites color[ijk] with the point's colour, channels swapped
 * BGR -> RGB, /255 (taichi_octomap.py:120-124); racing points, last writer wins.  Deterministic here: the latest
 * integrate call wins, inside a call the largest packed RGB.  rgb uint8 [n,3] / tex uint8 [th,tw,3] in `mem` space;
 * NULL colours integrate hits only.  Fusion copies the colour of the most recently integrated source voxel (:189). */
int tslam_octo_set_color_intrinsics(tslam_octo_t* m, double fx, double fy, double cx, double cy, int color_same_proj);
int tslam_octo_integrate_points_rgb(tslam_octo_t* m, const float* xyz, const uint8_t* rgb, int mem, int32_t n, const float* R9,
                                    const float* T3, int32_t submap, void* stream);
int tslam_octo_integrate_depth_tex(tslam_octo_t* m, const uint16_t* depth, const uint8_t* tex, int mem, int32_t h, int32_t w,
                                   int32_t th, int32_t tw, const float* R9, const float* T3, int32_t submap, void* stream);
/* gather / LoD export with the colour column: color f32[cap,3] / rgb f32[cap,3] DEVICE or NULL (:101-102, :113-114). */
int tslam_octo_gather2(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, uint32_t* count, float* color, int64_t* n_out,
                       void* stream);
int tslam_octo_extract2(tslam_octo_t* m, int32_t submap, int32_t level, int64_t cap, float* xyz, float* rgb, int32_t* count_dev,
                        void* stream);
/* every (i,j,k,count>0) of `submap`: idx int32[cap,3], count uint32[cap] (DEVICE). Synchronises. */
int tslam_octo_gather(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, uint32_t* count, int64_t* n_out,
                      void* stream);
/* cvt_occupy_to_voxels(level) / cvt_occupy_voxels_to (taichi_octomap.py:90-114): append to
 * xyz f32[cap,3] at *count_dev. */
int tslam_octo_extract(tslam_octo_t* m, int32_t submap, int32_t level, int64_t cap, float* xyz, int32_t* count_dev,
                       void* stream);
/* fuse_submaps_kernel (taichi_octomap.py:171-189) after reset(). */
int tslam_octo_fuse(tslam_octo_t* dst, tslam_octo_t* src, void* stream);
/* Incremental fusion of the submaps of `src` into the Octomap global map `dst` (DESIGN.md section 7, "Incremental
 * Octomap fusion"), hit counters and log-odds maps alike: an opt-in alternative to tslam_octo_fuse that re-places only
 * the submaps a call added, moved or removed.
 * Result: after the call every voxel word (cnt plane) and colour word of dst is bit for bit what tslam_octo_fuse gives
 * when src holds only the submaps s with include[s] != 0 (include: host, max_submaps bytes; NULL = all), each at its
 * fused pose, with k_octo_fuse's placement and dst's rule (hit threshold / l_occ).  Pool order may differ (it does
 * between two tslam_octo_fuse calls too): compare sorted gathered rows (ijk, word, colour).  An allocated block whose
 * words are all zero (left so by removals) reads like an absent one to every reader: gather, extract, queries, raycast,
 * the occupancy ESDF and the frontiers.
 * Fused pose of s: dst's pose-table row of s, unless s was fused before with the same content and
 * |T - T0| + angle(R0^T R) * r_s <= tolerance (r_s: farthest allocated 8^3 block corner of s from its origin; tolerance 0:
 * iff the pose bits are unchanged) - tslam_tsdf_fuse_update's rule.  The result does not depend on the history of calls.
 * Hit counter: dst.cnt = u32 sum (mod 2^32) of c over contributing source voxels (c > min_occupy_thres); removals
 * subtract in the cnt plane, exact under wrapping.
 * Log-odds: one int64 sum word per voxel, count * 2^32 + sum L (4 KB per 8^3 block, grown geometrically with the pool
 * blocks in use, log-odds dst only); a touched voxel reads count > 0 ? lo_word(clamp(sum L, l_min, l_max)) : 0.
 * Bound: a rigid placement puts at most 27 source voxels into one dst cell (27 sub-cubes of side vs / 3, plus f32
 * rounding, each of diameter < vs), so a cell takes at most 27 * max_submaps contributions and |sum L| <= 27 *
 * max_submaps * max(|l_min|, l_max) of src; the call refuses maps where that reaches 2^30 (OctoMap's defaults with 1024
 * submaps: 27 * 1024 * 3595 < 2^27).  Then count and sum L fit their 32-bit halves, and the readout equals
 * k_octo_fuse's: its wrapped u32 sum of L << 1 is 2 sum L exactly (|2 sum L| < 2^31, low bit 0), the OR'd known bit
 * makes it lo_word(sum L), and k_octo_lo_clamp clamps it once, as the readout does.
 * Colour (textured maps): additions raise colour words with a max, as k_octo_fuse does; every dst block a removal (or
 * the old pose of a move) touches has its colour words cleared and raised again from the included submaps at their
 * fused poses that can reach it (host filter on each submap's placed bounding sphere).
 * Plan: unchanged or moved within tolerance: nothing; newly included: add; excluded or now empty: subtract; moved:
 * subtract then add.  A full update (reset dst, then add every included submap) runs on the first call, when full != 0,
 * for another src, after any other write of dst (integrate, reset, tslam_octo_fuse into it), when a fused submap's
 * content changed (integrate into it, reset or tslam_octo_fuse of src), and when subtracting and re-adding would place
 * more source blocks than a rebuild; both paths give the same bits.
 * Trackers: an incremental update flags every dst block it touched for the next occupancy-ESDF and frontier update
 * (which stay incremental, and readable as of their last update); a full update resets dst and so invalidates them.
 * stats8 (may be NULL; tslam_tsdf_fuse_update's layout): full-update reason (0 incremental, 1 first call, 2 full
 * requested, 3 other src, 4 dst written, 5 content changed, 6 cheaper than subtract and re-add), submaps added, moved,
 * removed, left within tolerance, source voxels placed (adds + subtracts), voxels recoloured, dst blocks committed.
 * Refused (TSLAM_E_INVALID, nothing written), before the handles are looked at: tolerance not finite or < 0, a NULL
 * handle, dst == src; then maps that differ in occupancy model, max_submaps, voxel size or texture setting, and the
 * log-odds bound above.  N / Nz may differ (a large global map of small submaps): placement tests only dst's bounds, as
 * tslam_octo_fuse does.  An error flag of earlier work on dst is reported first.  TSLAM_E_POOL_FULL when dst's pool runs
 * out, with nothing added: an incremental update returns before any sum or word changes (dst as before the call); a
 * full update has already reset dst, which comes back empty.  Either way the next call is a full update.  TSLAM_E_CUDA
 * when the sums cannot grow; a removal that finds no dst block is reported as TSLAM_E_INVALID and makes the next call
 * full.  Synchronises. */
int tslam_octo_fuse_update(tslam_octo_t* dst, tslam_octo_t* src, const uint8_t* include, float tolerance, int32_t full,
                           int64_t* stats8, void* stream);
/* Octomap.is_occupy (taichi_octomap.py:86-88: occupy > min_occupy_thres) for points, and BaseMap.raycast. */
int tslam_octo_query_points(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, uint8_t* flags, void* stream);
int tslam_octo_raycast(tslam_octo_t* m, int32_t submap, int64_t n, const float* pos, const float* dir, float max_dist, uint8_t* hit,
                       float* xyz_out, float* len_out, void* stream);
int tslam_octo_sync(tslam_octo_t* m, void* stream);
int64_t tslam_octo_launch_count(tslam_octo_t* m);

/* ----------------------------------------------------------------------------
 * Log-odds occupancy (OctoMap's probabilistic model; DESIGN.md section 7).  Log-odds are Q10 integers,
 * l = round_half_away(logit(p) * 1024); with OctoMap's defaults l_hit = 868, l_miss = -415, l_min = -2048, l_max = 3595,
 * l_occ = 0.  A voxel is unknown until its first update and occupied iff known and L > l_occ.  Each integrate call is one
 * frame: a ray from the sensor position T3 to every endpoint; the end cell gets one hit update, every other cell of the
 * 6-connected voxel path one miss update (a hit wins), L <- clamp(L + l, l_min, l_max) once per voxel and frame.  Depth
 * pixels beyond max_ray_length (points beyond it in range |R p|) are cut there and give misses only.  The mode is fixed
 * for the map's life; integrate / extract / query / raycast / fuse follow it.  Extra memory: 128 B per pool block (the
 * per-frame hit / miss marks) + 8 B per pool block + 16 B per ray record.
 * --------------------------------------------------------------------------*/
typedef struct tslam_octo_logodds {
  int32_t l_hit, l_miss, l_min, l_max, l_occ;  /* need l_miss < 0 < l_hit, l_min <= 0 <= l_max, l_occ in [l_min, l_max] */
} tslam_octo_logodds_t;
int tslam_octo_create_logodds(const tslam_octo_config_t* cfg, const tslam_octo_logodds_t* lp, tslam_octo_t** out);
/* is_near_pos_occupy (mapping_common.py:193-204) for both modes: out[q] = 1 iff a cell of [-voxel, voxel)^3 around the
 * cell of xyz[q] is occupied.  xyz / out DEVICE. */
int tslam_octo_query_near_occupy(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, int32_t voxel, uint8_t* out,
                                 void* stream);
/* every known voxel of `submap` of a log-odds map: idx int32[cap,3], L int32[cap], color f32[cap,3] or NULL (DEVICE).
 * Synchronises. */
int tslam_octo_gather_logodds(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, int32_t* L, float* color,
                              int64_t* n_out, void* stream);
/* out4 = rays cast, miss-cell visits inside the volume, hit voxels, voxels updated, summed over the frames since the
 * last clear (zeros for a hit counter).  Synchronises the device. */
int tslam_octo_get_stats(tslam_octo_t* m, int64_t* out4, int clear);

/* ----------------------------------------------------------------------------
 * Occupancy ESDF of a log-odds map (DESIGN.md section 7): per submap, a FREE voxel (known, L <= l_occ) holds its 26-
 * neighbour chamfer distance to the nearest OCC voxel centre (known, L > l_occ), an OCC voxel minus its distance to the
 * nearest FREE voxel centre, both truncated at D = max_dist; paths run through known voxels only.  Edge costs are
 * vs * {1, sqrtf(2), sqrtf(3)} in f32 with vs = f32(voxel_scale).  Every call refuses a hit-counter map
 * (TSLAM_E_INVALID).  State (allocated by the first update): about 2.7 KB per pool block.
 * --------------------------------------------------------------------------*/
/* Bring the field of `submap` up to date.  mode 0: incremental when the last update was for the same submap and the
 * same max_dist (bit for bit) and no reset or fusion came since, else full; mode 1: full.  Either gives the same bits.
 * max_dist must be finite and > 0.  stats4 (HOST, may be NULL): lower sweeps, raise sweeps (-1 = full), changed voxels,
 * suspect voxels.  Synchronises. */
int tslam_octo_esdf_update(tslam_octo_t* m, int32_t submap, float max_dist, int32_t mode, int32_t* stats4, void* stream);
/* (ijk, ESDF) of every voxel known at the last update: idx int32[cap,3], esdf f32[cap] (DEVICE); n_out = the number of
 * such voxels (TSLAM_E_CAPACITY when it exceeds cap).  Refused before an update, for another submap than the last
 * update's, and after a reset or fusion until the next update.  Synchronises. */
int tslam_octo_esdf_gather(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, float* esdf, int64_t* n_out, void* stream);
/* tslam_esdf_query on the occupancy ESDF, as of the last update: trilinear distance and its exact gradient; dist, grad
 * NaN and valid 0 where a coordinate is not finite or a corner is outside the volume, in a block newer than the update,
 * or was unknown at the update.  xyz f32[n,3], dist f32[n], grad f32[n,3], valid u8[n] (DEVICE); n == 0 is a no-op.
 * Refused like tslam_octo_esdf_gather. */
int tslam_octo_esdf_query(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, float* dist, float* grad, uint8_t* valid,
                          void* stream);

/* ----------------------------------------------------------------------------
 * Frontiers of a log-odds map (DESIGN.md section 7): per submap, a frontier voxel is a FREE cell (known, L <= l_occ)
 * with at least one 6-neighbour that is inside the volume and UNKNOWN (not known; every cell of an absent block).
 * Clusters are the 26-connected components of the frontier voxels, labelled by the smallest linear key
 * ((i+hN)*N + (j+hN))*Nz + (k+hNz) of their voxels and listed in ascending label order.  Every call refuses a
 * hit-counter map (TSLAM_E_INVALID).  State (allocated by the first update): 84 B per pool block, plus 8 B per
 * frontier voxel and 156 B per cluster, grown on demand.
 * --------------------------------------------------------------------------*/
/* Bring the frontier set of `submap` up to date.  mode 0: incremental (re-examine the blocks updated since the last
 * update and their face neighbours) when the last update was for the same submap and no reset or fusion came since,
 * else full; mode 1: full.  Either gives the same frontier set and records.  stats4 (HOST, may be NULL): frontier
 * voxels, clusters, blocks re-examined, 1 when the update was full.  Synchronises. */
int tslam_octo_frontier_update(tslam_octo_t* m, int32_t submap, int32_t mode, int32_t* stats4, void* stream);
/* (ijk, cluster ordinal) of every frontier voxel of the last update: idx int32[cap,3], cluster int32[cap] (DEVICE);
 * n_out = the number of frontier voxels (TSLAM_E_CAPACITY when it exceeds cap; the first cap rows are written).
 * Refused before an update, for another submap than the last update's, and after a reset or fusion until the next
 * update. */
int tslam_octo_frontier_gather(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, int32_t* cluster, int64_t* n_out,
                               void* stream);
/* The cluster records of the last update in label order, sixteen int64 each (DEVICE rec16[cap,16]): label, voxels,
 * sum i, sum j, sum k, min i, min j, min k, max i, max j, max k, faces (voxel / UNKNOWN in-volume 6-neighbour pairs),
 * the sums of the unit offsets towards those neighbours (x, y, z), 0.  n_out = the number of clusters
 * (TSLAM_E_CAPACITY when it exceeds cap).  Refused like tslam_octo_frontier_gather. */
int tslam_octo_frontier_clusters(tslam_octo_t* m, int32_t submap, int64_t cap, int64_t* rec16, int64_t* n_out, void* stream);

/* ----------------------------------------------------------------------------
 * Viewpoint gain of a log-odds map (DESIGN.md section 7): what a depth camera would see from each of n candidate views
 * of `submap`.  A view is a position pos[3] and a row-major rotation R9[9] in the submap's map frame, with the
 * convention of integrate_depth's R, T (camera x right, y down, z forward).  A view is valid iff its 12 numbers are
 * finite and its cell round_half_away(pos / voxel_scale) is inside the volume and FREE; an invalid view gets valid = 0
 * and zero in every output.  Arrays are DEVICE, n == 0 is a no-op.  Neither call changes the map or any tracker state.
 * Both refuse (TSLAM_E_INVALID) a NULL handle or camera, n < 0, NULL arrays when n > 0, a hit-counter map, fx, fy or
 * max_range not finite and > 0, non-finite cx or cy, width, height or step not > 0, width / step or height / step
 * rounding down to 0, and a camera whose farthest ray spans more than 2^22 cells.
 * --------------------------------------------------------------------------*/
typedef struct tslam_view_camera {
  float fx, fy, cx, cy;          /* pinhole intrinsics of the simulated depth camera                        */
  int32_t width, height, step;   /* image size; rays at pixels (ii * step, jj * step), ii < width / step    */
  float max_range;               /* every simulated pixel lies beyond it: rays are cut at depth max_range    */
} tslam_view_camera_t;
/* Unknown gain: gain[v] (int64) = the number of distinct UNKNOWN cells among the cells the view's rays see - each ray
 * walks integrate_depth's path of an all-far pixel up to its first OCC cell; out-of-volume cells are skipped.
 * Asynchronous: a walk that leaves its view's bitmap window (only possible when R is not a rotation) is reported as
 * TSLAM_E_INVALID by the next synchronising call (tslam_octo_sync). */
int tslam_octo_view_gain_unknown(tslam_octo_t* m, int32_t submap, int64_t n, const float* pos, const float* R9,
                                 const tslam_view_camera_t* cam, uint8_t* valid, int64_t* gain, void* stream);
/* Frontier gain: the frontier voxels of the last tslam_octo_frontier_update inside the view's frustum whose line of sight
 * from the view crosses FREE cells only (classes as of the call).  per_cluster[v * n_clusters + c] (int32, may be NULL)
 * counts them per cluster ordinal, total[v] is the row sum.  Also refused where tslam_octo_frontier_gather is, and when
 * n_clusters differs from the last update's cluster count. */
int tslam_octo_view_gain_frontier(tslam_octo_t* m, int32_t submap, int64_t n, const float* pos, const float* R9,
                                  const tslam_view_camera_t* cam, int64_t n_clusters, uint8_t* valid, int32_t* total,
                                  int32_t* per_cluster, void* stream);

/* Frontier viewpoints: candidate sensor poses around each frontier cluster of the last tslam_octo_frontier_update, the
 * best top_k per cluster (DESIGN.md section 7).  Classes as of the call.  Candidate (c, s) for cluster ordinal c and
 * sample s < n_samples: m = (float)((double)sum / (double)voxels * (double)vs) per axis from c's record, p = m +
 * offsets[s] (f32), and the level camera facing m: (dx, dy) = (m - p)_xy, h = sqrtf(dx*dx + dy*dy), (ux, uy) =
 * (dx, dy) / h, R = [[uy, 0, ux], [-ux, 0, uy], [0, -1, 0]] row-major (the view-gain convention).  A candidate is valid
 * iff p is finite, h > 0 and its cell round_half_away(p / vs) is traversable under the travel-cost rule with `clearance`;
 * an invalid candidate is not an error.  Its score is the number of cluster c's frontier voxels the frontier gain would
 * count for (p, R) with `cam`.  Kept: valid and score >= min_visible, ordered by score descending, then s ascending.
 * Outputs (DEVICE): count int32[nc] = min(top_k, kept); per slot j < top_k of cluster c (index c * top_k + j): sample
 * int32, visible int32, pos f32[3], R9 f32[9]; slots at and beyond count hold sample -1, visible 0 and a zero pose.
 * offsets f32[n_samples,3] (DEVICE), 1 <= n_samples, top_k <= TSLAM_OCTO_VIEWPOINT_MAX_SAMPLES, min_visible >= 1.
 * Refused (TSLAM_E_INVALID): a NULL handle, camera or offsets, NULL outputs when n_clusters > 0, n_samples or top_k out
 * of range, min_visible < 1, the camera checks of the view-gain calls, clearance as tslam_octo_travel_update refuses it,
 * where tslam_octo_frontier_gather is refused, n_clusters different from the last update's cluster count, and more than
 * 2^31 - 1 scoring items.  n_clusters == 0 is a no-op.  Asynchronous; changes neither the map nor any tracker state.
 * Scratch (in the handle, grown on demand, freed by tslam_octo_destroy): 152 B per cluster, 28 B per frontier voxel, 4 B per candidate
 * and 8 B per scoring item (n_samples * (ceil(frontier voxels / 64) + n_clusters) of them). */
#define TSLAM_OCTO_VIEWPOINT_MAX_SAMPLES 1024
int tslam_octo_frontier_viewpoints(tslam_octo_t* m, int32_t submap, const tslam_view_camera_t* cam, int32_t n_samples,
                                   const float* offsets, float clearance, int32_t min_visible, int32_t top_k, int64_t n_clusters,
                                   int32_t* count, int32_t* sample, int32_t* visible, float* pos, float* R9, void* stream);

/* ----------------------------------------------------------------------------
 * Travel cost on a log-odds map (DESIGN.md section 7): per submap, as of one update, the geodesic cost G from a start
 * cell through known free space.  A cell is traversable iff it is inside the volume and FREE (known, L <= l_occ), and,
 * when clearance > 0, was FREE at the last tslam_octo_esdf_update of the submap, in a block that update saw, with ESDF
 * value >= clearance.  Steps join 26-neighbours at the ESDF's f32 edge costs vs * {1, sqrtf(2), sqrtf(3)} and are
 * allowed iff every cell of the box their two cells span is traversable (no corner cutting).  G(start) = 0 when the
 * start cell round_half_away(start / voxel_scale) is traversable; every other cell holds the least f32 path sum, added
 * one step at a time; a cell above max_cost is unreachable (+inf).  Every call refuses a hit-counter map and a submap out
 * of range (TSLAM_E_INVALID).  The field is the S = 1 case of the many-source fields below, in a state of its own: 68 B
 * per pool block plus ~4.2 KB per submap block with a traversable cell, allocated by the first update, grown
 * geometrically and freed by tslam_octo_destroy.
 * --------------------------------------------------------------------------*/
/* Compute the field of `submap` from start3 (HOST, finite).  clearance finite and >= 0 (> 0 needs a readable occupancy
 * ESDF of the submap whose max_dist is >= clearance); max_cost finite, > 0 and <= 2^22 * vs.  A start that is not
 * traversable is not an error: start_ok = 0 and nothing is reachable.  stats4 (HOST, may be NULL): reachable cells,
 * sweeps, traversable cells, start_ok.  A wave still changing after the last sweep is refused, and so are the readers
 * until the next update.  Synchronises. */
int tslam_octo_travel_update(tslam_octo_t* m, int32_t submap, const float* start3, float clearance, float max_cost,
                             int32_t* stats4, void* stream);
/* (ijk, G) of every reachable cell: idx int32[cap,3], cost f32[cap] (DEVICE); n_out = the number of such cells
 * (TSLAM_E_CAPACITY when it exceeds cap).  Refused before an update, for another submap than the last update's, and
 * after a reset or fusion until the next update.  Synchronises. */
int tslam_octo_travel_gather(tslam_octo_t* m, int32_t submap, int64_t cap, int32_t* idx, float* cost, int64_t* n_out,
                             void* stream);
/* cost f32[n] = G of the cell of xyz[n,3] as of the last update; +inf where unreachable, outside the volume, in a block
 * newer than the update, or not finite (DEVICE, asynchronous, n == 0 a no-op).  Refused like tslam_octo_travel_gather. */
int tslam_octo_travel_query(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, float* cost, void* stream);
/* Path from the cell of each target xyz[n,3] to the start: cells int32[n,max_len,3] target -> start, each cell's
 * predecessor being the reachable 26-neighbour with an allowed step and G(h) + c == G(v), smallest G(h), ties to the
 * first in dx, dy, dz = -1, 0, 1 order (dx outermost); len int32[n] = the full number of cells, 0 when unreachable (only
 * the first max_len are written).  max_len >= 1.  DEVICE, asynchronous.  Refused like tslam_octo_travel_gather. */
int tslam_octo_travel_path(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, int32_t max_len, int32_t* cells,
                           int32_t* len, void* stream);

/* Many-source travel costs: S fields of one submap in one update, field s exactly the single-source field from starts[s]
 * (same traversability, steps, f32 sums and max_cost cut).  G_s(p_t) and G_t(p_s) add the same steps in opposite orders
 * and may differ in the last bits; nothing symmetrises them.  Under the default max_cost (2^22 * vs) reachability is
 * symmetric.  The fields are separate from the single-source field: an update of either changes nothing the other's
 * readers return.  State: 68 B per pool block, plus ~2.1 KB per submap block with a traversable cell (B_t) and ~2 KB per
 * (block, source) pair, grown geometrically (at least x2 per growth) and freed by tslam_octo_destroy. */
#define TSLAM_OCTO_TRAVEL_MAX_STARTS 1024
/* Compute the fields from starts[n_starts,3] (HOST, finite, 1 <= n_starts <= TSLAM_OCTO_TRAVEL_MAX_STARTS, duplicates
 * allowed); clearance and max_cost as for tslam_octo_travel_update.  stats2 (HOST, may be NULL): sweeps, traversable
 * cells; reachable[n_starts] (HOST, may be NULL): reachable cells per start; start_ok[n_starts] (HOST, may be NULL): 1
 * when the start's cell is traversable, else 0 and its row is all +inf (not an error).  Synchronises. */
int tslam_octo_travel_multi_update(tslam_octo_t* m, int32_t submap, int32_t n_starts, const float* starts, float clearance,
                                   float max_cost, int32_t* stats2, int32_t* reachable, uint8_t* start_ok, void* stream);
/* cost f32[S,n] row-major: cost[s*n + q] = G_s of the cell of xyz[q] as of the last multi update, with the rules of
 * tslam_octo_travel_query (DEVICE, asynchronous).  Passing the starts as xyz gives the S x S matrix.  Refused before a
 * multi update, for another submap, after a reset or fusion, and after a failed update. */
int tslam_octo_travel_multi_query(tslam_octo_t* m, int32_t submap, int64_t n, const float* xyz, float* cost, void* stream);
/* Path of pair q from the cell of xyz[q] back to starts[source[q]] with the rule and the len / max_len semantics of
 * tslam_octo_travel_path (DEVICE, asynchronous).  A source outside [0, S) writes len 0 and makes the next
 * tslam_octo_sync return TSLAM_E_INVALID.  Refused like tslam_octo_travel_multi_query. */
int tslam_octo_travel_multi_path(tslam_octo_t* m, int32_t submap, int64_t n, const int32_t* source, const float* xyz,
                                 int32_t max_len, int32_t* cells, int32_t* len, void* stream);

/* ----------------------------------------------------------------------------
 * Exploration tours (DESIGN.md section 7): the order in which to visit goals, from a cost matrix such as the S x S
 * matrix of tslam_octo_travel_multi_query.  Stateless.  cost f32[n,n] (DEVICE), 1 <= n <= TSLAM_OCTO_TRAVEL_MAX_STARTS:
 * node 0 is the start, nodes 1..n-1 the goals, the diagonal is ignored and every other entry is +inf, zero or a
 * positive normal f32 (a NaN, a negative value or a subnormal is refused).  Costs are exact: with e_lo / e_hi the least /
 * greatest floor(log2 x) over the positive finite off-diagonal entries (0 / 0 when there are none), e_hi - e_lo <= 28 is
 * required, every finite entry is the integer q(x) = x / U units of U = 2^(e_lo - 23), and a leg weighs (inf, q) =
 * (1, 0) for +inf, (0, q(x)) otherwise.  A tour's cost is the sum of its legs, compared lexicographically (fewer
 * infinite legs first).  The kept goals K are the g >= 1 with cost[0][g] finite, m = |K|; the others are unreachable.
 * A tour is open: t[0] = 0, t[1..m] a permutation of K, cost sum_{p<m} w(t[p], t[p+1]).
 * Restart 0 starts from the nearest-neighbour tour (least w, ties to the smaller node); restart r >= 1 from a
 * Fisher-Yates shuffle of K ascending: for i = m-1 down to 1, j = mix64(seed ^ (r << 32) ^ i) % (i + 1) in uint64, swap
 * a[i], a[j] (mix64: the SplitMix64 finaliser).  Each step applies the move giving the cheapest tour if it is strictly
 * cheaper, ties to the first in the order 2-opt (reverse t[i..j], 1 <= i < j <= m, reversed legs charged in their new
 * direction) by (i, j), then Or-opt (move t[i..i+L-1], L in {1,2,3}, orientation kept, to follow t[p], p in [0, m] minus
 * [i-1, i+L-1]) by (L, i, p).  A restart ends when no move improves (converged 1) or when a further move would exceed
 * max_passes applied moves (converged 0).
 * --------------------------------------------------------------------------*/
/* restarts in [1, 4096], max_passes >= 0.  Outputs (DEVICE): tours int32[R,n] (row r: t[0..m], then -1), cost2
 * int64[R,2] (infinite legs, q), passes int32[R] (moves applied), converged uint8[R], best int32[1] (the least cost,
 * ties to the smallest r); info2 (HOST): m, e_lo - 23 (U = 2^info2[1]).  Reads the matrix's scan once (synchronises),
 * then runs asynchronously on `stream`. */
int tslam_tour_open(int32_t n, const float* cost, int32_t restarts, uint64_t seed, int32_t max_passes, int32_t* tours,
                    int64_t* cost2, int32_t* passes, uint8_t* converged, int32_t* best, int32_t* info2, void* stream);

/* ----------------------------------------------------------------------------
 * SDF-to-SDF registration of TSDF submap pairs (DESIGN.md section 7, "Submap registration").  Pair p registers reference
 * submap ref_submaps[p] of map A against reading submap read_submaps[p] of map B (A == B allowed; the voxel scales must
 * be the same f32 bits).  T_p = (R, t) maps points of the reference submap's local frame into the reading submap's local
 * frame (a global map's local frame is the world frame).
 *   points     the voxels v of the reference submap in non-ghost blocks of A with obs = 1, W > 0, W >= min_weight and
 *              |TSDF| <= band; p_v = (f32(i) vs, f32(j) vs, f32(k) vs), d_v = TSDF(v)
 *   residual   x = R p_v + t in f32 (R, t rounded to f32 once per evaluation; pose_apply's operation order); D_B(x) the
 *              trilinear interpolant of B's committed TSDF of the reading submap with the ESDF queries' low-corner and
 *              interpolation rules, g its exact gradient; valid iff all 8 corners lie in the volume, in present
 *              non-ghost blocks, with obs = 1 and W > 0; r = D_B(x) - d_v (f32); J = [g, x cross g] (f64, left
 *              perturbation T <- exp(xi) T, xi = (rho, phi)); Huber weight w = 1 if |r| <= huber else huber / |r|
 *   sums       H = sum w J J^T, b = sum w J r, cost = sum rho_huber(r), n_valid (f64, fixed order per pair)
 *   solver     Levenberg-Marquardt (f64, host): (H + lam diag(max(H_ii, 1e-9 max_j H_jj))) xi = -b by Cholesky, lam
 *              from 1e-4; a step is accepted when n_valid >= min_points and cost / n_valid decreases (lam / 10), else
 *              rejected (lam * 10, pose kept).  Stops when |rho| < 1e-4 vs and |phi| < 1e-6 (converged), after
 *              max_iters evaluations, or when the damped matrix is not positive definite.  max_iters = 0 returns the
 *              normal equations at T0.
 * Inputs (HOST): R0 f64[P,9] row-major, T0 f64[P,3], finite.  1 <= P <= TSLAM_REG_MAX_PAIRS; submaps in range; band and
 * huber finite and > 0; min_weight finite; max_iters, min_points >= 0.  Outputs (HOST): R_out f64[P,9], T_out f64[P,3]
 * (final pose), H_out f64[P,36], b_out f64[P,6] (at the final pose), cost2 f64[P,2] (initial, final cost), info5
 * int64[P,5] (n_points, n_valid at the final pose, evaluations after the first, converged, status: 0 ok, 1 fewer than
 * min_points valid points at T0 - not a call error).  A pair's result does not depend on the other pairs of the call.
 * Flushes both maps, synchronises once per iteration, and writes no map word, flag, ESDF, mesh state or statistic other
 * than A's kernel-launch counter (tslam_tsdf_launch_count), which counts the call's launches as it does every call's.
 * Scratch in A's handle, grown geometrically, freed by tslam_tsdf_destroy: 28 B per pool block of A, 16 B per selected
 * point, 232 B per 1024-point chunk of every pair, ~300 B per pair. */
#define TSLAM_REG_MAX_PAIRS 1024
int tslam_tsdf_register(tslam_tsdf_t* A, tslam_tsdf_t* B, int32_t n_pairs, const int32_t* ref_submaps, const int32_t* read_submaps,
                        const double* R0, const double* T0, float band, float min_weight, float huber, int32_t max_iters,
                        int32_t min_points, double* R_out, double* T_out, double* H_out, double* b_out, double* cost2,
                        int64_t* info5, void* stream);

/* ----------------------------------------------------------------------------
 * Frame tracking against the TSDF (DESIGN.md section 7, "Frame tracking"): the pose at which a depth frame's or a point
 * cloud's points lie on the zero level of the map's committed TSDF, found before the frame is integrated (point-to-SDF
 * alignment, Bylow et al. 2013).
 *   pose       T_f = (R, t), f64 in and out, is the pose of frame f in the local frame of submap submaps[f] (a global map's
 *              local frame is the world frame): the (R, T) tslam_tsdf_integrate_depth takes for that frame, so integrating
 *              at the returned pose integrates at the tracked pose.
 *   depth      n frames uint16 [n, height, width] mm in `mem`.  Frame f's candidates are the sampled pixels (i, j) =
 *              (step ii, step jj), ii < width / step, jj < height / step (integer quotients: the pixels integrate samples
 *              at recast_step = step).  A pixel of d mm is kept when d != 0 && !(f32(d) > dmax_mm || f32(d) < dmin_mm)
 *              (dmin_mm, dmax_mm = f32(min_ray_length 1000), f32(max_ray_length 1000)); its point is (x, y, dep) with
 *              the bucket kernel's f32 operations: dep = f32(d) / 1000, x = ((f32(i) - cx) dep) / fx, y = ((f32(j) - cy)
 *              dep) / fy, each correctly rounded.  submaps: HOST int32 [n], or NULL for all zero.
 *   points     one cloud f32 [n_points, 3] in the sensor frame, in `mem`, tracked against `submap`.  A point is kept when
 *              x, y, z are finite and min_ray_length <= r < max_ray_length (f32 bounds) with r = sqrtf((x x + y y) + z z)
 *              in f32: integrate's upper bound, applied before the rotation (the unknown), and a lower bound that drops
 *              the (0, 0, 0) a LiDAR driver reports for a missing return.
 *   records    (x, y, z, 0): a frame's records are contiguous, in row-major sampled-pixel order (depth) or input order
 *              (points), whatever else the call holds.
 *   residual, sums, solver   those of tslam_tsdf_register with d_v = 0 and the reading submap submaps[f] of this map: the
 *              same corner validity, Huber weight, f64 sums, LM schedule, stopping rules and max_iters = 0 semantics.  H
 *              and b are for the left perturbation T <- exp(xi) T in the submap's local frame.
 * Inputs (HOST): R0 f64[n,9] row-major, T0 f64[n,3], finite.  Outputs (HOST), per frame, as tslam_tsdf_register's per
 * pair: R_out f64[n,9], T_out f64[n,3], H_out f64[n,36], b_out f64[n,6], cost2 f64[n,2] (initial, final cost), info5
 * int64[n,5] (points selected, valid at the final pose, evaluations after the first, converged, status: 0 ok, 1 fewer
 * than min_points valid points at T0 - not a call error, the normal answer for the first frame of an empty submap).
 * A frame's result does not depend on the other frames of the call; two identical calls give the same bits, and host and
 * device input give the same bits.
 * Refused (TSLAM_E_INVALID) before the handle is looked at: n outside [1, TSLAM_REG_MAX_PAIRS] (n_points < 0), step < 1,
 * height or width not positive, huber not finite or not > 0, max_iters < 0 or min_points < 0, mem not a TSLAM_MEM_*;
 * then a NULL handle or array, a submap out of range, a non-finite initial pose.
 * Flushes the queued frames and pending commits first, synchronises once per iteration, and writes no map word, flag,
 * ESDF, mesh state or statistic other than the kernel-launch counter.  Scratch in the handle (shared with
 * tslam_tsdf_register, grown geometrically, freed by tslam_tsdf_destroy): 16 B per candidate chunk of 1024, the input
 * when it is in host memory, 16 B per kept point, 232 B per 1024-point chunk of every frame, ~300 B per frame. */
int tslam_tsdf_track_depth(tslam_tsdf_t* m, const uint16_t* depth, int mem, int32_t n, int32_t height, int32_t width,
                           const int32_t* submaps, const double* R0, const double* T0, int32_t step, float huber, int32_t max_iters,
                           int32_t min_points, double* R_out, double* T_out, double* H_out, double* b_out, double* cost2, int64_t* info5,
                           void* stream);
int tslam_tsdf_track_points(tslam_tsdf_t* m, const float* xyz, int mem, int32_t n_points, int32_t submap, const double* R0,
                            const double* T0, float huber, int32_t max_iters, int32_t min_points, double* R_out, double* T_out,
                            double* H_out, double* b_out, double* cost2, int64_t* info5, void* stream);

/* ----------------------------------------------------------------------------
 * Place recognition between TSDF submaps (DESIGN.md section 7, "Loop detection"): a descriptor per submap that ignores
 * yaw, and a batched search that shortlists, per query, database entries with a coarse 4-DoF pose (Scan Context, Kim &
 * Kim 2018, adapted to TSDF submaps).  The caller verifies a candidate with tslam_tsdf_register started from that pose.
 *   frames     M9 (HOST f32 [n,9] row-major, finite) is the levelled rotation M_s = L R_s of entry s, rounded to f32 once
 *              by the caller: R_s the submap's f64 base rotation (identity for a global map), L the minimal f64 rotation
 *              taking the world unit vector `up` to +z.  A point is x = M_s p_v in f32, pose_apply's operation order with
 *              a zero translation (((M0 px + M1 py) + M2 pz) + 0 per row); horizontal (x0, x1), height x2.
 *   points     the registration points of tslam_tsdf_register: voxels of non-ghost blocks with obs = 1, W > 0,
 *              W >= min_weight, |TSDF| <= band; p_v = (f32(i) vs, f32(j) vs, f32(k) vs).
 *   rings      rho2 = x0 x0 + x1 x1 (f32); ring = the first i with rho2 < B_i, B_i = f32((f64(r_max) (i + 1) / 20)^2);
 *              points with rho2 >= B_19 are left out of the polar grid.
 *   sectors    f_k = c_k x1 - s_k x0 (f32, in that order), (c_k, s_k) = f32(cos, sin(2 pi k / 60)), k mod 60; the
 *              sector is the first k in [0, 60) with f_k >= 0 and f_{k+1} < 0, or 0 when there is none (rho2 = 0).
 *   sc         f32 [n, 20 x 60] (DEVICE), row = ring: zmax - zmin (f32) of the bin's heights, 0 for an empty bin.
 *   ring       f32 [n, 20] (DEVICE): f32(non-empty bins of ring i) / 60.
 *   bev        u32 [n, 512] (DEVICE): the 128 x 128 bird's-eye bitmap, cell size c = f32(r_max) / 64, u = floor(x0 / c) +
 *              64, v = floor(x1 / c) + 64 (f32 division; points outside [0, 128) left out); bit v % 32 of word 4 u + v / 32
 *              is set iff the cell's zmax - zmin >= h_min (vertical structure, not floor).
 *   n_points   int64 [n] (HOST): the entry's registration points.
 * Every output is an exact function of the points (min and max commute): the same bits whatever the atomics' order.
 * Refused (TSLAM_E_INVALID, nothing written) before the handle is looked at: n outside [1, 1024], a NULL array or
 * params, r_max, h_min or band not finite or not > 0, min_weight not finite, a non-finite M9; then a NULL handle or a
 * submap out of range.  A submap may appear twice.  Flushes the queued frames first, synchronises once, and writes no map
 * word, flag, ESDF, mesh state or statistic other than the kernel-launch counter.  Scratch: tslam_tsdf_register's. */
typedef struct {
  float r_max;       /* radius of the polar grid, half the bitmap's side (m) */
  float h_min;       /* least height span of a set bitmap cell (m) */
  float band;        /* registration points: |TSDF| <= band */
  float min_weight;  /* registration points: W >= min_weight */
} tslam_place_params_t;
int tslam_tsdf_place_describe(tslam_tsdf_t* m, int32_t n, const int32_t* submaps, const float* M9, const tslam_place_params_t* params,
                              float* sc, float* ring, uint32_t* bev, int64_t* n_points, void* stream);

/* Matching of queries against a database of n_db descriptors (DEVICE sc, ring, bev as above; n_points, ids int64 [n_db]
 * DEVICE).  No handle: descriptors can be kept across calls.  queries (HOST int32 [n_q]) are database indices.
 *   eligible   d != q, |ids[q] - ids[d]| >= min_gap, n_points of both >= min_points.
 *   shortlist  ring distance sum_i (k_qi - k_di)^2 in f32, i ascending; the top_k eligible entries by (distance, index).
 *   yaw        for m in [0, 60): columns j where |sc_q[:, j]| and |sc_d[:, (j + m) % 60]| are both non-zero (norm sqrtf of
 *              the f32 sum of squares in ring order); cos_j = dot / (|a| |b|) (dot in ring order); D(m) = 1 - (sum_j
 *              cos_j, j ascending) / f32(n_j), 1 when n_j = 0; m* = argmin, ties to the smaller m.  x_d ~ Rz(6 m* deg) x_q.
 *   offset     yaws psi_y = (2 m* + y - 1) x 3 deg, y = 0, 1, 2 (f32 cos, sin of 2 pi h / 120).  q's bitmap is rotated by
 *              inverse mapping: cell (u, v) takes (a, b) = (f32(u - 64) + 0.5, f32(v - 64) + 0.5), (a', b') = (c a + s b,
 *              c b - s a) in f32, source cell (floor(a') + 64, floor(b') + 64), 0 outside.  score(dx, dy) = popc of rot
 *              q shifted by (dx, dy) cells AND d, dx, dy in [-32, 32].  Best: the largest score, ties to the smaller |dx| +
 *              |dy|, then the smaller y, then dy, then dx.  overlap = f32(score) / f32(min(popc(rot q), popc(d))), 0 when
 *              that is 0.  Then x_d ~ Rz(psi) x_q + (dx c, dy c).
 * Outputs (DEVICE), row qi top_k + slot: info6 int32 [.,6] (match index or -1 past the eligible entries, m*, y, dx, dy,
 * score), dist3 f32 [.,3] (ring distance, D(m*), overlap); an unmatched row is (-1, 0, 0, 0, 0, 0), (0, 1, 0).  A query's
 * rows do not depend on the other queries.  Refused (TSLAM_E_INVALID, nothing written): n_db or n_q outside [1, 1024],
 * top_k outside [1, TSLAM_PLACE_MAX_TOP_K], min_gap < 0, a NULL array, a query outside [0, n_db).  Runs asynchronously on
 * `stream` (stream-ordered scratch of about 40 B per row). */
#define TSLAM_PLACE_MAX_TOP_K 32
int tslam_place_match(int32_t n_db, const float* sc, const float* ring, const uint32_t* bev, const int64_t* n_points, const int64_t* ids,
                      int32_t n_q, const int32_t* queries, int32_t top_k, int64_t min_gap, int64_t min_points, int32_t* info6,
                      float* dist3, void* stream);

/* ----------------------------------------------------------------------------
 * Rendering of the TSDF's zero level (DESIGN.md section 7, "Rendering"): depth, normal and colour images of n pinhole
 * cameras, ray-cast to the surface that registration and frame tracking align to (KinectFusion's model image).
 *   cameras    1 <= n <= TSLAM_RENDER_MAX_CAMERAS, one pinhole K4 = (fx, fy, cx, cy) (HOST f64, rounded to f32 once) and
 *              one image size height x width for all.  Camera c has pose (R_c, T_c) (HOST f64 [n,9] row-major and [n,3],
 *              rounded to f32 once), which maps camera points into the local frame of submap submaps[c] (HOST int32 [n],
 *              or NULL for all zero): the (R, T) tslam_tsdf_integrate_depth and tslam_tsdf_track_depth take.
 *   ray        pixel (i, j) (column i, row j, no half-pixel offset): camera-frame direction r = ((f32(i) - cx) / fx,
 *              (f32(j) - cy) / fy, 1), each operation correctly rounded, turned into the local frame in pose_apply's
 *              order ((R0 rx + R1 ry) + R2 1) + 0 per row, giving dir.  The ray parameter is the camera-frame depth z.
 *   samples    K = floor((z_max - z_min) / step) + 1 (host, f64 of the f32 parameters); for k = 0 .. K-1:
 *              z_k = z_min + f32(k) step, x_k = T + z_k dir per axis, each operation one correctly rounded f32 operation.
 *   value      D_k = the trilinear interpolant of the committed TSDF of the camera's submap at x_k (u = x / vs,
 *              c0 = floor(u), fractions u - c0, lerp along x, then y, then z: the ESDF query's arithmetic).  Valid iff all
 *              8 corners lie in the volume, in present non-ghost blocks, and each has obs != 0 and W > 0: the corner rule
 *              of tslam_tsdf_register, with no other threshold.
 *   hit        the first k with samples k and k+1 both valid, D_k > 0 and D_{k+1} <= 0 (free space into the surface;
 *              back faces and crossings across an invalid sample are not hits).  a = D_k - D_{k+1}, f = D_k / a,
 *              z* = z_k + step f, x* = T + z* dir, each f32 in that order.
 * Outputs (DEVICE, row-major):
 *   depth      f32 [n,h,w]: z*, or 0 where there is no hit (the depth-image convention, which integrate drops).
 *   status     u8 [n,h,w]: 0 no hit; 1 hit with normal (and colour); 2 hit, but a corner of x*'s cell is not valid or
 *              |g| = 0.
 *   normal     f32 [n,h,w,3] (may be NULL): g / |g| in the submap's local frame, g the interpolant's gradient at x*
 *              (the ESDF query's), |g| = sqrtf((gx gx + gy gy) + gz gz).  NaN unless status is 1.
 *   color      f32 [n,h,w,3] (may be NULL; textured maps only): each channel of the committed colour interpolated at x*
 *              over the same 8 corners in the same lerp order.  NaN unless status is 1.
 * Every pixel is independent: batches, repeated calls and single-camera calls give the same bits.
 * Refused (TSLAM_E_INVALID) before the handle is looked at: n outside [1, TSLAM_RENDER_MAX_CAMERAS]; height or width < 1
 * or n h w >= 2^31; f32(fx), f32(fy) not finite or not > 0, f32(cx), f32(cy) not finite; z_min not finite or not > 0;
 * z_max not finite or not > z_min; step not finite or not > 0; K > TSLAM_RENDER_MAX_SAMPLES; K4, depth or status NULL.
 * Then: a NULL handle or pose array, a submap out of range, a pose not finite (in f64 or after rounding to f32), color
 * requested on a map without texture.
 * Flushes the queued frames and pending commits first; writes no map word, flag, ESDF, mesh state or statistic other
 * than the kernel-launch counter.  Asynchronous on `stream` apart from the upload of the per-camera jobs (52 B per
 * camera, in a scratch buffer of the handle grown geometrically and freed by tslam_tsdf_destroy). */
#define TSLAM_RENDER_MAX_CAMERAS 1024
#define TSLAM_RENDER_MAX_SAMPLES 65536
int tslam_tsdf_render(tslam_tsdf_t* m, int32_t n, int32_t height, int32_t width, const double* K4, const int32_t* submaps,
                      const double* R, const double* T, float z_min, float z_max, float step, float* depth, float* normal,
                      float* color, uint8_t* status, void* stream);

/* ----------------------------------------------------------------------------
 * Trajectories against an ESDF (DESIGN.md section 7, "Trajectories"; tslam_traj.cuh states every operation)
 *
 * T uniform cubic B-splines, trajectory t with N_t = n_ctrl[t] control points Q_0 .. Q_{N-1} (f64, the submap-local map
 * frame tslam_esdf_query takes) and knot span dt, optimised against the ESDF of `submap` as of its last update.  The
 * first three and the last three control points are fixed (start and end position, velocity and acceleration); the
 * free variables are Q_3 .. Q_{N-4}.  Span j = 0 .. N-4 uses Q_j .. Q_{j+3}; collision samples sit at u = k/K,
 * k = 0 .. K-1, on every span plus u = 1 on the last ((N-3) K + 1 samples); a sample's position is
 * ((b0 Q_j + b1 Q_{j+1}) + b2 Q_{j+2}) + b3 Q_{j+3} in f64, rounded to f32 once, and its distance d and gradient g are
 * exactly what the ESDF query returns at that f32 point, with its validity rule.  Cost, f64:
 *   J_s = sum |Q_{i+3} - 3 Q_{i+2} + 3 Q_{i+1} - Q_i|^2                        (smoothness)
 *   J_c = sum over valid samples with d < c of (c - d)^2                        (collision, c = clearance)
 *   J_u = number of invalid samples, no gradient                                (unknown or absent space)
 *   J_f = sum max(0, |V_i|^2 - v^2)^2 + sum max(0, |A_i|^2 - a^2)^2,  V_i = (Q_{i+1} - Q_i)/dt,
 *         A_i = (Q_{i+2} - 2 Q_{i+1} + Q_i)/dt^2                                (feasibility)
 *   J   = w_s J_s + w_c J_c + w_f J_f + w_u J_u
 * Solver: L-BFGS on the device in f64, memory M; the first direction is -g scaled to one voxel in its largest
 * component, and a direction that does not descend resets the history; Armijo backtracking from alpha = 1 (c1 = 1e-4,
 * halving, at most 30 trials); a pair is kept when s'y > 1e-10 y'y.  Status: 1 |g|inf <= g_tol, 2 line search
 * exhausted, 0 max_iters steps taken, 3 N < 7 (nothing to optimise: evaluated only).  max_iters = 0 evaluates the input
 * (a batched safety check of committed trajectories).  Then a dense check of the result at C samples per span, placed
 * the same way.  Every sum runs in a fixed order (tslam_traj.cuh), so one trajectory's result depends on nothing else
 * in the call, and repeated calls give the same bits.
 *
 * Arrays (HOST): n_ctrl i32[T]; ctrl_in, ctrl_out f64[sum N, 3] (trajectories back to back); cost f64[T, 6]: J_s, J_c,
 * J_f, J_u at the result, J at the input, the least d over the valid check samples (+inf when none); info i32[T, 7]:
 * iterations, evaluations, status, invalid check samples, valid check samples with d < c, and the span and k of the
 * least d (lowest (span, k) on ties; -1 when no sample is valid).
 * Refused (TSLAM_E_INVALID) before the handle is looked at: a NULL array or params; T outside [1, 1024]; an N outside
 * [4, 1024]; sum N > 2^20; samples (K) outside [1, 16], check_samples (C) outside [1, 64], memory (M) outside [1, 16];
 * dt, v_max, a_max not finite and > 0; a weight, the clearance or g_tol not finite and >= 0; max_iters < 0; a
 * non-finite control point.  Then: a NULL handle; the field not readable (tslam_esdf_query's rules for the TSDF;
 * tslam_octo_esdf_query's for the Octomap, which refuse a hit-count map); a clearance above the field's far value (the
 * TSDF's max_ray_length; the max_dist of the Octomap's last ESDF update).
 * Writes no map word, ESDF, frontier, travel or mesh state and no statistic other than the kernel-launch counter.  One
 * launch; synchronises on `stream`.  Device scratch of (18 + 6 M) 8 sum N bytes plus the inputs and outputs, grown
 * geometrically and freed by destroy; an allocation failure is TSLAM_E_CUDA with the byte count in tslam_last_error. */
typedef struct tslam_traj_params {
  double dt;                  /* knot span (s) */
  double v_max, a_max;        /* velocity and acceleration limits */
  double w_smooth, w_collision, w_feasibility, w_unknown;
  double clearance;           /* c (m) */
  double g_tol;               /* stop when |g|inf <= g_tol */
  int32_t max_iters;          /* L-BFGS steps at most (0: evaluate and check only) */
  int32_t memory;             /* M, L-BFGS pairs kept */
  int32_t samples;            /* K, collision samples per span */
  int32_t check_samples;      /* C, check samples per span */
} tslam_traj_params_t;
#define TSLAM_TRAJ_MAX 1024
#define TSLAM_TRAJ_MAX_CTRL 1024
int tslam_esdf_trajectory(tslam_tsdf_t* m, int32_t submap, int32_t T, const int32_t* n_ctrl, const double* ctrl_in,
                          const tslam_traj_params_t* params, double* ctrl_out, double* cost, int32_t* info, void* stream);
int tslam_octo_esdf_trajectory(tslam_octo_t* m, int32_t submap, int32_t T, const int32_t* n_ctrl, const double* ctrl_in,
                               const tslam_traj_params_t* params, double* ctrl_out, double* cost, int32_t* info, void* stream);

/* ----------------------------------------------------------------------------
 * Submap pose-graph optimisation (DESIGN.md section 7, "Pose-graph optimisation"; tests/pose_graph_reference.py states
 * the same contract in numpy).  Stateless: no handle.  All arithmetic is f64.
 *   nodes      X_i = (R_i, t_i), i < N, maps submap-local coordinates to world coordinates.  fixed[i] != 0 marks a node
 *              that never moves (the gauge); it is returned bit-identical to its input.
 *   edges      edge k = (i, j, Z_k, Omega_k, c_k), i != j.  Z_k = (R, t) maps i-local to j-local: tslam_tsdf_register's
 *              T with i = reference and j = reading submap, detect_loops' with i = query and j = match.  Omega_k is 6x6 in
 *              xi = (rho, phi) order; only its upper triangle is read, and it may be rank-deficient (registration on one
 *              plane gives rank 3).  c_k >= 0 is the Cauchy scale, 0 for plain least squares.
 *   residual   e_k = Log(X_j^-1 X_i Z_k^-1), Log the exact inverse of registration's exponential R' = Exp(phi) R,
 *              t' = Exp(phi) t + V(phi) rho: theta = atan2(|w| / 2, (tr R - 1) / 2), w = vee(R - R^T); phi = theta w /
 *              (2 sin theta) when cos theta >= 0, else theta times the unit axis u of the symmetric part
 *              (R + R^T) / 2 - cos theta I = (1 - cos theta) u u^T (largest diagonal first), signed so that u . w >= 0;
 *              rho = V(phi)^-1 t.  Every angle coefficient (sin th / th, (1 - cos th) / th^2, (th - sin th) / th^3,
 *              (1 - (th / 2) cot(th / 2)) / th^2 and Barfoot's two Q coefficients) is its series through th^4 below
 *              theta = 1e-2.  If the measurement were exp(xi) Z for the true relative pose, e = xi exactly, so
 *              registration's H (for the left perturbation T <- exp(xi) T) is the information of e as it stands.
 *   cost       s_k = e_k^T Omega_k e_k; rho_k(s) = s when c_k = 0, else c_k^2 log1p(s / c_k^2); F = 1/2 sum rho_k(s_k),
 *              summed in edge order within chunks of 256 edges and then over the chunk sums in chunk order.  IRLS weight
 *              w_k = rho_k'(s_k) = 1 / (1 + s_k / c_k^2) (1 when c_k = 0).
 *   update     left perturbation in the world frame X_i <- exp(delta_i) X_i for free nodes.  J_i = de/ddelta_i =
 *              Jl^-1(e) Ad(X_j^-1) (Jl^-1 the closed-form inverse left Jacobian of SE(3)), J_j = -J_i, both exact.
 *              A = sum w J^T Omega J over free nodes, g = sum w J^T Omega e.
 *   solver     Levenberg-Marquardt with registration's schedule: (A + lam diag(max(A_ii, 1e-9 max_j A_jj))) delta = -g,
 *              lam from 1e-4; a step is accepted when F decreases (lam / 10), else rejected (poses kept, lam * 10).
 *              Converged when an accepted step has max |rho| < eps_t and max |phi| < eps_r.  Also stops after max_iters
 *              evaluations, when lam > 1e16 (no progress), or when a damped 6x6 diagonal block is not positive definite.
 *              max_iters = 0 evaluates F, s_k and w_k at the input and moves nothing.
 *   linear     preconditioned conjugate gradients (6x6 block-Jacobi preconditioner, Cholesky of the damped diagonal
 *              blocks) from x0 = 0, stopped when |r|_2 <= cg_tol |g|_2 or after max_cg iterations (or when p^T A p <= 0).
 *              A step from a CG run that hit max_cg is still tried: LM's acceptance test guards it.  One cooperative
 *              launch runs every CG iteration; its dot products sum fixed chunks of 32 free nodes in chunk order.
 * Determinism: two identical calls give the same bits, whatever the grid size (pcg_grid) or the SM count.
 * Inputs (HOST): R f64[N,9] row-major, T f64[N,3], fixed u8[N], ij int32[E,2], ZR f64[E,9], ZT f64[E,3], omega f64[E,36]
 * row-major, cauchy f64[E].  Outputs (HOST): R_out f64[N,9], T_out f64[N,3] (final poses), chi2 f64[E] (s_k) and weight
 * f64[E] (w_k) at the final poses, f3 f64[3] (F initial, F final, the largest final relative CG residual |r| / |g|),
 * info5 int64[5] (LM evaluations, accepted steps, CG iterations in all, converged, status: 0 converged, 1 max_iters
 * evaluations, 2 no progress, 3 damped block not positive definite).
 * Refused (TSLAM_E_INVALID, nothing written), in this order, before any device work: N outside [2, 4096] or E outside
 * [1, 65536]; a NULL array or params; eps_t or eps_r not finite or < 0, cg_tol not finite or outside [0, 1), max_iters
 * outside [0, TSLAM_PG_MAX_ITERS], max_cg outside [1, TSLAM_PG_MAX_ITERS], pcg_grid < 0; then per node in order a
 * non-finite pose, a rotation with max |R^T R - I| > 1e-6; then per edge in order an endpoint out of range or i == j, a
 * non-finite measurement, upper-triangle Omega entry or c_k, c_k < 0, a measured rotation with max |R^T R - I| > 1e-6, a
 * negative diagonal entry of Omega; then a connected component with no fixed node (union-find on the host: without one
 * the damped system has no gauge).
 * Uploads the graph once into stream-ordered scratch (about 600 B per edge, 700 B per free node, 200 B per node) and
 * synchronises `stream` once per LM evaluation. */
typedef struct {
  double eps_t;       /* convergence: max |rho| of an accepted step below this (m) */
  double eps_r;       /* convergence: max |phi| of an accepted step below this (rad) */
  double cg_tol;      /* CG stops at |r|_2 <= cg_tol |g|_2 */
  int32_t max_iters;  /* LM evaluations at most (0: evaluate the input only) */
  int32_t max_cg;     /* CG iterations per step at most */
  int32_t pcg_grid;   /* CTAs of the CG launch: 0 sizes it from the graph, clamped to the co-resident maximum */
} tslam_pg_params_t;
#define TSLAM_PG_MAX_ITERS 100000
int tslam_pose_graph_solve(int32_t n_nodes, const double* R, const double* T, const uint8_t* fixed, int32_t n_edges,
                           const int32_t* ij, const double* ZR, const double* ZT, const double* omega, const double* cauchy,
                           const tslam_pg_params_t* params, double* R_out, double* T_out, double* chi2, double* weight,
                           double* f3, int64_t* info5, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TSLAM_H */
