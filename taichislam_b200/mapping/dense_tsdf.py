"""DenseTSDF - the reference's class surface (taichi_slam/mapping/dense_tsdf.py) on libtslam.so.

Same constructor kwargs, attributes and methods as the reference class (SURVEY.md section 8b);
every method that launched a Taichi kernel now enqueues hand-written sm_90a kernels through
the C ABI (include/tslam.h).  Like Taichi, calls are asynchronous: `recast_depth_to_map`
hands the frame and its pose to the library's queue (pageable arrays are copied at once, page-locked
ones are fetched by the GPU itself a few calls later) and the queue integrates every 32 frames with
one launch triple; any reader (`count_active`, `to_numpy`, `cvt_*`, field reads, the mesher, the
planner queries) flushes the queue first, so results are indistinguishable from per-frame execution
(up to the commit-granularity note in DESIGN.md for voxels saturated at Wmax).
"""
import collections
import math
import time

import numpy as np

from .. import _capi as capi
from ..tsdf_handle import TsdfHandle
from .field import Field
from .mapping_common import BaseMap

Wmax = 1000  # dense_tsdf.py:8


class DenseTSDF(BaseMap):
    def __init__(self, map_scale=[10, 10], voxel_scale=0.05, texture_enabled=False,
                 max_disp_particles=1024 * 1024, num_voxel_per_blk_axis=16, max_ray_length=10, min_ray_length=0.3,
                 internal_voxels=10, max_submap_num=1024, is_global_map=False,
                 disp_ceiling=1.8, disp_floor=-0.3, recast_step=2, color_same_proj=True,
                 max_blocks=0, max_image_pixels=640 * 480):
        super(DenseTSDF, self).__init__(voxel_scale)
        import torch
        self._torch = torch
        # derived sizes exactly as dense_tsdf.py:18-31
        self.num_voxel_per_blk_axis = num_voxel_per_blk_axis
        self.voxel_scale = voxel_scale
        self.N = math.ceil(map_scale[0] / voxel_scale / num_voxel_per_blk_axis) * num_voxel_per_blk_axis
        self.Nz = math.ceil(map_scale[1] / voxel_scale / num_voxel_per_blk_axis) * num_voxel_per_blk_axis
        self.block_num_xy = math.ceil(map_scale[0] / voxel_scale / num_voxel_per_blk_axis)
        self.block_num_z = math.ceil(map_scale[1] / voxel_scale / num_voxel_per_blk_axis)
        self.map_size_xy = voxel_scale * self.N
        self.map_size_z = voxel_scale * self.Nz
        self.max_disp_particles = max_disp_particles
        self.enable_texture = texture_enabled
        self.max_ray_length = max_ray_length
        self.min_ray_length = min_ray_length
        self.tsdf_surface_thres = self.voxel_scale * 1.8  # :39
        self.internal_voxels = internal_voxels
        self.max_submap_num = max_submap_num
        self.is_global_map = is_global_map
        self.disp_ceiling = disp_ceiling
        self.disp_floor = disp_floor
        self.recast_step = recast_step
        self.color_same_proj = color_same_proj
        self.clear_last_TSDF_exporting = False  # assigned by SubmapMapping (submap_mapping.py:134)
        self.color = None  # the colour plane lives inside the library handle (dense_tsdf.py:48-50); read it with to_numpy

        self._h = TsdfHandle(self.N, self.Nz, voxel_scale=voxel_scale, max_ray_length=max_ray_length,
                             min_ray_length=min_ray_length, internal_voxels=internal_voxels, recast_step=recast_step,
                             K=None, is_global_map=is_global_map, disp_floor=disp_floor, disp_ceiling=disp_ceiling,
                             max_submaps=min(max_submap_num, 1024), max_blocks=max_blocks,
                             max_image_pixels=max_image_pixels, texture_enabled=texture_enabled)
        self.initialize_submap_fields(self.max_submap_num)
        self._init_export_fields()
        self._queue = self._h.L.tslam_tsdf_queue_depth
        self._queue_tex = self._h.L.tslam_tsdf_queue_depth_tex
        self._queue_begin = self._h.L.tslam_tsdf_queue_depth_begin
        self._queue_end = self._h.L.tslam_tsdf_queue_depth_end
        # page-locked frames are read by the GPU straight from host memory a few calls later (include/tslam.h): keep
        # the arrays alive for as long as the library may still read them (it never runs more than 2 batches ahead)
        self._frame_refs = collections.deque(maxlen=6 * capi.MAX_BATCH)  # depth + colour image per frame
        self._raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
        self._dev_index = torch.cuda.current_device()
        if texture_enabled:
            self._h.set_color_intrinsics([1, 0, 0, 0, 1, 0, 0, 0, 1], color_same_proj)
        self._pR, self._pT = self.input_R_np.ctypes.data, self.input_T_np.ctypes.data  # persistent pose buffers (BaseMap.set_pose)
        print(f"TSDF map initialized blocks {self.block_num_xy}x{self.block_num_xy}x{self.block_num_z}")

    # ------------------------------------------------------------------ fields (dense_tsdf.py:52-60, :129-134)
    def _init_export_fields(self):
        torch = self._torch
        dev = torch.device("cuda", torch.cuda.current_device())
        n = self.max_disp_particles
        fl = self._flush
        self.num_export_particles = Field(torch.zeros(1, dtype=torch.int32, device=dev), fl)
        self.num_TSDF_particles = Field(torch.zeros(1, dtype=torch.int32, device=dev), fl)
        self.num_export_ESDF_particles = Field(torch.zeros(1, dtype=torch.int32, device=dev), fl)
        self.export_x = Field(torch.full((n, 3), -100000.0, dtype=torch.float32, device=dev), fl)
        self.export_color = Field(torch.full((n, 3), 0.5, dtype=torch.float32, device=dev), fl)
        self.export_TSDF = Field(torch.zeros(n, dtype=torch.float32, device=dev), fl)
        self.export_TSDF_xyz = Field(torch.full((n, 3), -100000.0, dtype=torch.float32, device=dev), fl)
        self.export_ESDF = Field(torch.zeros(n, dtype=torch.float32, device=dev), fl)  # dense_esdf.py ESDF slice export
        self.export_ESDF_xyz = Field(torch.full((n, 3), -100000.0, dtype=torch.float32, device=dev), fl)

    def _on_intrinsics(self):
        self._flush()
        self._h.set_intrinsics(self.K_cam_dep)

    def set_color_camera_intrinsic(self, K):
        super(DenseTSDF, self).set_color_camera_intrinsic(K)
        self._flush()
        self._h.set_color_intrinsics(self.K_cam_color, self.color_same_proj)

    def _upload_submap_pose(self, submap_id, R, T):
        self._h.set_submap_pose(submap_id, R, T)

    # ------------------------------------------------------------------ integrate (dense_tsdf.py:157-165)
    def recast_depth_to_map(self, R, T, depthmap, texture):
        """Queue one depth frame (uint16 mm [h,w]); the library integrates queued frames in batches (:162-165).
        The frame is copied to the device right away (asynchronously when `depthmap` is pinned host memory)."""
        if self.K_cam_dep is None:
            raise RuntimeError("set_dep_camera_intrinsic() must be called before recast_depth_to_map")
        if depthmap.dtype != np.uint16 or not depthmap.flags.c_contiguous:
            depthmap = np.ascontiguousarray(depthmap, dtype=np.uint16)
        h, w = depthmap.shape
        sid = 0 if self.is_global_map else self.active_submap_id.v
        self._frame_refs.append(depthmap)
        if self.enable_texture and texture is not None and getattr(texture, "size", 0) > 0:
            # ti.static(self.enable_texture) (:205): the colour image rides along (uint8 [th,tw,3]); a caller that has no
            # image for this frame (empty array) integrates geometry only
            self.set_pose(R, T)
            if not self.color_same_proj and self.K_cam_color is None:
                raise RuntimeError("set_color_camera_intrinsic() must be called before recast_depth_to_map (color_same_proj=False)")
            if texture.dtype != np.uint8 or not texture.flags.c_contiguous:
                texture = np.ascontiguousarray(texture, dtype=np.uint8)
            th, tw = texture.shape[0], texture.shape[1]
            self._frame_refs.append(texture)
            if self.color_same_proj and (th < h or tw < w):
                raise ValueError("color_same_proj=True needs a colour image at least as large as the depth image")
            rc = self._queue_tex(self._h.h, depthmap.__array_interface__["data"][0], texture.__array_interface__["data"][0], h, w,
                                 th, tw, self._pR, self._pT, sid, self._stream_ptr())
        else:
            # the frame's copy is started first, the pose arithmetic (set_pose: convert_by_base in f64) runs while the
            # DMA is in flight, then the copy is awaited: the array has been consumed when this method returns
            st = self._stream_ptr()
            rc = self._queue_begin(self._h.h, depthmap.__array_interface__["data"][0], h, w, st)
            if rc:
                capi.check(rc)
            self.set_pose(R, T)
            rc = self._queue_end(self._h.h, self._pR, self._pT, sid, st)
        if rc:
            capi.check(rc)

    def set_frame_borrowing(self, on=True):
        """Opt in to zero-copy hand-over of PAGE-LOCKED depth frames: they are not copied, the GPU reads their sampled rows
        from host memory a few calls later, so the caller must leave them untouched until the next reader / flush.
        Default (off): recast_depth_to_map has consumed the array when it returns, like the reference."""
        self._flush()
        capi.check(self._h.L.tslam_tsdf_set_frame_mode(self._h.h, int(bool(on))))

    def set_commit_granularity(self, frames):
        """Frames per internal launch + commit (default 32).  1 = one commit per recast_depth_to_map call: the clamp at
        Wmax (dense_tsdf.py:267) then sees the same granule as a frame-by-frame run of the reference kernels."""
        self._flush()
        capi.check(self._h.L.tslam_tsdf_set_queue_launch(self._h.h, int(frames), int(frames)))

    def _stream_ptr(self):
        # raw handle of torch's current stream; the private accessor skips building a Stream object (once per frame)
        if self._raw_stream is not None:
            return self._raw_stream(self._dev_index)
        return self._torch.cuda.current_stream().cuda_stream

    def _flush(self):
        capi.check(self._h.L.tslam_tsdf_flush(self._h.h, self._stream_ptr()))

    def recast_pcl_to_map(self, R, T, xyz_array, rgb_array):
        """:157-160.  xyz_array [n,3] (any float dtype; computed in f32 like the kernel's ti.f32 cast, :171-174)."""
        self._flush()
        self.set_pose(R, T)
        xyz = np.ascontiguousarray(np.asarray(xyz_array, dtype=np.float32).reshape(-1, 3))
        s = 0 if self.is_global_map else self.active_submap_id[None]
        rgb = None
        if self.enable_texture and rgb_array is not None and np.size(rgb_array) > 0:  # :179-183
            rgb = np.ascontiguousarray(np.asarray(rgb_array, dtype=np.uint8).reshape(-1, 3))
        self._h.integrate_points(xyz, self.input_R_np, self.input_T_np, submap=s, commit=True, rgb=rgb)
        self._torch.cuda.current_stream().synchronize()  # pageable source

    # ------------------------------------------------------------------ submaps / fusion (:272-318)
    def reset(self):
        self._h.reset()

    def fuse_submaps(self, submaps):
        submaps._flush()
        t = time.time()
        self._h.fuse_from(submaps._h)
        print(f"[DenseTSDF] Fuse submaps {(time.time() - t) * 1000:.1f}ms, active local: {submaps.active_submap_id[None]} "
              f"remote: {submaps.remote_submap_num[None]}")

    def update_fused_submaps(self, submaps, include=None, tolerance=0.0, full=False):
        """Keep this global map equal to the fusion of `submaps` (a DenseTSDF collection) with exact integer sums,
        re-splatting only the submaps that were added, moved or removed since the last call (TsdfHandle.fuse_update).
        Queued frames of `submaps` are integrated first.  -> dict of the call's statistics."""
        submaps._flush()
        return self._h.fuse_update(submaps._h, include=include, tolerance=tolerance, full=full)

    def reclaim(self, submaps=None, all_blocks=False, empty=False, center=None, radius=None):
        """Give pool blocks back (TsdfHandle.reclaim): the blocks of `submaps` (None: all) that all_blocks, empty (no
        observed voxel) or the sphere (center, radius) select are dropped and the pool is compacted.  `center` is in
        the frame this map stores its submaps in (the map frame of a global map, a submap's own frame before its base
        pose).  Queued frames are integrated first.  -> dict of the call's statistics."""
        self._flush()
        return self._h.reclaim(submaps=submaps, all_blocks=all_blocks, empty=empty, center=center, radius=radius)

    # ------------------------------------------------------------------ exporters (:320-389)
    def _active(self):
        return 0 if self.is_global_map else self.active_submap_id[None]

    def cvt_occupy_to_voxels(self):
        self.cvt_TSDF_surface_to_voxels()

    def cvt_TSDF_surface_to_voxels(self):
        self._flush()
        self.num_TSDF_particles.t.zero_()  # add_to_cur=False (:342-343)
        self._h.extract_surface(self._active(), self.export_TSDF_xyz.t, self.export_color.t, self.num_TSDF_particles.t)

    def cvt_TSDF_surface_to_voxels_to(self, num_TSDF_particles, max_disp_particles, export_TSDF_xyz, export_color):
        self._flush()
        xyz = export_TSDF_xyz.t[:max_disp_particles]
        rgb = export_color.t[:max_disp_particles]
        self._h.extract_surface(self._active(), xyz, rgb, num_TSDF_particles.t)

    def cvt_TSDF_to_voxels_slice(self, z, dz=0.5, clear_last=True):
        self._flush()
        if clear_last:
            self.num_TSDF_particles.t.zero_()
        self._h.extract_slice(self._active(), z, dz, self.export_TSDF_xyz.t, self.export_TSDF.t, self.export_color.t,
                              self.num_TSDF_particles.t)

    def get_voxels_TSDF_surface(self):
        self.cvt_TSDF_surface_to_voxels()
        return self.export_TSDF_xyz.to_numpy(), self.export_TSDF.to_numpy(), None

    def get_voxels_TSDF_slice(self, z):
        self.cvt_TSDF_to_voxels_slice(z)
        return self.export_TSDF_xyz.to_numpy(), self.export_TSDF.to_numpy()

    def get_voxels_occupy(self):
        self.cvt_occupy_to_voxels()
        return self.export_TSDF_xyz.to_numpy(), self.export_color.to_numpy()

    def finalization_current_submap(self):
        self._flush()

    # ------------------------------------------------------------------ I/O (:412-515)
    def count_active(self):
        self._flush()
        return self._h.count_active(self._active())

    def to_numpy(self, data_indices, data_tsdf, data_wtsdf, data_occ, data_color):
        """Fill caller arrays (dtypes of export_submap, :459-462) with the observed voxels of the active submap."""
        self._flush()
        if self.enable_texture:
            idx, t, w, occ, col = self._h.gather(self._active(), color=True)
        else:
            idx, t, w, occ = self._h.gather(self._active())
        n = idx.shape[0]
        data_indices[:n] = idx
        data_tsdf[:n] = t
        data_wtsdf[:n] = w
        data_occ[:n] = occ
        if self.enable_texture:  # :437-440
            data_color[:n] = col

    def load_numpy(self, submap_id, data_indices, data_tsdf, data_wtsdf, data_occ, data_color):
        self._flush()
        occ = np.clip(np.asarray(data_occ).astype(np.int64), -128, 127).astype(np.int8)
        col = None
        if self.enable_texture:  # :450-453
            col = np.asarray(data_color, dtype=np.float32).reshape(-1, 3)
        self._h.scatter(submap_id, np.asarray(data_indices).astype(np.int32), np.asarray(data_tsdf, dtype=np.float32),
                        np.asarray(data_wtsdf, dtype=np.float32), occ, color=col)

    def export_submap(self):
        s = time.time()
        num = self.count_active()
        indices = np.zeros((num, 3), np.int16)
        tsdf = np.zeros((num), np.float16)
        w_tsdf = np.zeros((num), np.float16)
        occupy = np.zeros((num), np.int8)
        color = np.zeros((num, 3), np.float16) if self.enable_texture else np.array([])  # :463-466
        self.to_numpy(indices, tsdf, w_tsdf, occupy, color)
        obj = {
            'indices': indices,
            'TSDF': tsdf,
            'W_TSDF': w_tsdf,
            'color': color,
            'occupy': occupy,
            "map_scale": [self.map_size_xy, self.map_size_z],
            "voxel_scale": self.voxel_scale,
            "texture_enabled": self.enable_texture,
            "num_voxel_per_blk_axis": self.num_voxel_per_blk_axis,
        }
        print(f"Export submap {self.active_submap_id[None]} to numpy, voxels {num / 1024:.1f}k, time: {1000 * (time.time() - s):.1f}ms")
        return obj

    def saveMap(self, filename):
        np.save(filename, self.export_submap())

    @staticmethod
    def loadMap(filename):
        obj = np.load(filename, allow_pickle=True).item()
        vs = obj['voxel_scale'] if 'voxel_scale' in obj else obj['voxel_size']  # shipped fixtures carry the legacy key
        mapping = DenseTSDF(map_scale=obj['map_scale'], voxel_scale=float(vs), texture_enabled=obj['texture_enabled'],
                            num_voxel_per_blk_axis=obj['num_voxel_per_blk_axis'], is_global_map=True)
        mapping.load_numpy(0, obj['indices'], obj['TSDF'], obj['W_TSDF'], obj['occupy'], obj['color'])
        print(f"[SubmapMapping] Loaded {obj['TSDF'].shape[0]} voxels from {filename}")
        return mapping

    def input_remote_submap(self, submap):
        # remote submaps fill the table from the top (:500-515)
        self.remote_submap_num[None] = self.remote_submap_num[None] + 1
        idx = self.max_submap_num - self.remote_submap_num[None]
        R, T = submap['pose']
        color = submap['color'] if self.enable_texture else np.array([])  # :509-512
        self.load_numpy(idx, submap['indices'], submap['TSDF'], submap['W_TSDF'], submap['occupy'], color)
        self.set_base_pose_submap(idx, R, T)
        return idx

    # ------------------------------------------------------------------ planner queries (mapping_common.py:165-204)
    def _query_raycast(self, pos, dir, max_dist):
        self._flush()
        return self._h.raycast(pos, dir, max_dist, submap=self._active())

    def _query_points(self, xyz):
        self._flush()
        return self._h.query_points(xyz, submap=self._active())   # (is_occupy, is_unobserved), dense_tsdf.py:148-155

    def _query_near(self, xyz, voxel):
        self._flush()
        return self._h.query_near_occupy(xyz, voxel, submap=self._active())

    def init_sphere(self):
        """dense_tsdf.py:136-146 as intended by tests/marching_cube_test.py:20-21: an analytic sphere SDF of radius
        3 voxels in a 30^3 region (the reference indexes its 4-D fields with three indices there and uses uncentred
        coordinates, so the kernel does not run at HEAD; this is the centred, working form: TSDF = |p| - radius)."""
        r = np.arange(-15, 15)
        I, J, K = np.meshgrid(r, r, r, indexing="ij")
        idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
        p = idx.astype(np.float32) * np.float32(self.voxel_scale)
        t = np.sqrt((p * p).sum(1)).astype(np.float32) - np.float32(self.voxel_scale * 3)
        self.load_numpy(self._active(), idx, t, np.ones_like(t), np.zeros(len(t), np.int8),
                        np.full((len(t), 3), 0.5, np.float32) if self.enable_texture else np.array([]))

    # ------------------------------------------------------------------ extras (not in the reference)
    def frame_counters(self):
        """Flush, commit and read the integrate counters back (bench.py end-to-end arm)."""
        self._flush()
        st = self._h.stats()
        st["d2h_bytes"] = 8 * 8 + 5 * 8 + 4 * 4
        return st

    def esdf_update(self):
        """Converged ESDF of the active submap (DenseSDF.propogate_esdf semantics, dense_esdf.py:302-333)."""
        self._flush()
        return self._h.esdf_update(self._active())

    def get_voxels_ESDF(self):
        return self._h.esdf_gather(self._active())

    def esdf_query(self, xyz, update=True):
        """Interpolated ESDF and its gradient at points [n,3] of the active submap's map frame (what Voxblox, which
        dense_esdf.py:1 implements, answers for planners): (dist, grad, valid), torch CUDA tensors for a torch tensor,
        numpy arrays for a numpy array.  update=True first brings the field up to date (incremental esdf_update);
        update=False answers from the field as of the last update."""
        self._flush()
        if update:
            self._h.esdf_update(self._active())
        return self._h.esdf_query(xyz, submap=self._active())

    def optimize_trajectories(self, paths_or_ctrl, clearance, spacing=None, ctrl=False, update=True, **settings):
        """Smooth collision-free trajectories along paths or control points of the active submap's map frame: each
        entry of paths_or_ctrl is a path f[n,3] (e.g. plan_exploration()["path"] or a travel_path result), made into
        control points by trajectory.control_points(path, spacing) (spacing defaults to two voxels), or, with
        ctrl=True, control points themselves.  The free control points are optimised on the GPU against the ESDF
        (L-BFGS, include/tslam.h tslam_esdf_trajectory) and the result checked densely.  update=True first brings the
        field up to date, as esdf_query(update=True) does.  -> a list of dicts, one per trajectory: ctrl f64[N,3], the
        cost terms, iterations, evaluations, status and the check (min_dist, min_at, invalid, close, ok).  settings:
        trajectory.DEFAULTS (dt, v_max, a_max, weights, g_tol, max_iters, memory, samples, check_samples)."""
        from ..trajectory import control_points
        self._flush()
        if update:
            self._h.esdf_update(self._active())
        sp = 2.0 * self.voxel_scale if spacing is None else float(spacing)
        qs = [np.asarray(q, np.float64) if ctrl else control_points(q, sp) for q in paths_or_ctrl]
        return self._h.trajectory(qs, clearance, submap=self._active(), **settings)

    def cvt_ESDF_to_voxels_slice(self, z):
        """dense_esdf.py:498-509, after bringing the field up to date: the ESDF voxels of the slice at height z into
        export_ESDF / export_ESDF_xyz, their number into num_export_ESDF_particles.  Only voxels observed at the update
        are exported (the reference's struct-for also visits unobserved cells of active blocks, ESDF 0)."""
        self._flush()
        s = self._active()
        self._h.esdf_update(s)
        self.num_export_ESDF_particles.t.zero_()
        self._h.esdf_extract_slice(s, z, self.export_ESDF_xyz.t, self.export_ESDF.t, self.num_export_ESDF_particles.t)

    def get_voxels_ESDF_slice(self, z):
        """dense_esdf.py:569-571."""
        self.cvt_ESDF_to_voxels_slice(z)
        return self.export_ESDF_xyz.to_numpy(), self.export_ESDF.to_numpy()

    def base_pose(self, submap_id):
        """f64 (R, T) of a submap's local frame in the world frame: the stored base pose, the identity for a global map."""
        if self.is_global_map:
            return np.eye(3), np.zeros(3)
        return np.array(self.submaps_base_R_np[submap_id], dtype=np.float64), np.array(self.submaps_base_T_np[submap_id], dtype=np.float64)

    def register_submaps(self, ref_submaps, reading_submaps, reading=None, poses=None, band=None, min_weight=0.0, huber=None,
                         max_iters=20, min_points=100):
        """SDF-to-SDF registration of submap pairs on the GPU (tslam_tsdf_register, DESIGN.md section 7): pair p aligns
        the near-surface voxels (|TSDF| <= band, W >= min_weight) of submap ref_submaps[p] of this map with the TSDF of
        submap reading_submaps[p] of `reading` (default: this map) and returns the pose T_p = (R, T) that maps points of
        the reference submap's local frame into the reading submap's local frame.  poses: initial (R [P,3,3], T [P,3]);
        default base_b^-1 * base_a from the stored base poses in f64.  band defaults to 4 voxels (the weight ramp
        theta, :219), huber to one voxel.  Flushes both maps.  -> one dict per pair: R, T, H (6x6 information at the
        final pose, xi = (rho, phi) of the left perturbation), b, cost_init, cost, n_points, n_valid, iterations,
        converged, status (1: fewer than min_points valid points at the initial pose)."""
        reading = self if reading is None else reading
        a = [int(s) for s in np.asarray(ref_submaps).reshape(-1)]
        r = [int(s) for s in np.asarray(reading_submaps).reshape(-1)]
        assert len(a) == len(r), "one reading submap per reference submap"
        if poses is None:
            R0, T0 = np.zeros((len(a), 3, 3)), np.zeros((len(a), 3))
            for p, (sa, sb) in enumerate(zip(a, r)):
                Ra, Ta = self.base_pose(sa)
                Rb, Tb = reading.base_pose(sb)
                R0[p], T0[p] = Rb.T @ Ra, Rb.T @ (Ta - Tb)
        else:
            R0, T0 = poses
        self._flush()
        reading._flush()
        band = 4.0 * self.voxel_scale if band is None else band
        out = self._h.register(reading._h, a, r, R0, T0, band, min_weight, huber, max_iters, min_points)
        keys = ("R", "T", "H", "b", "cost_init", "cost", "n_points", "n_valid", "iterations", "converged", "status")
        return [{k: (out[k][p].copy() if out[k].ndim > 1 else out[k][p].item()) for k in keys} for p in range(len(a))]

    # ------------------------------------------------------------------ loop detection (DESIGN.md section 7)
    LOOP_DEFAULTS = dict(r_max=8.0, h_min=0.3, band=None, min_weight=0.0, top_k=8, min_gap=1, min_points=200, max_sc_dist=0.35,
                         min_overlap=0.3, min_inlier_ratio=0.5, max_cost=None, huber=None, max_iters=100)

    def describe_places(self, submaps, up=None, r_max=8.0, h_min=0.3, band=None, min_weight=0.0, base_poses=None):
        """Place descriptors of `submaps` on the GPU (tslam_tsdf_place_describe): each submap's registration points,
        levelled by M_s = L R_s (L takes `up`, default +z, to +z; R_s the f64 base rotation), binned into a 20 x 60
        polar grid of height spans, a ring key and a 128 x 128 bird's-eye bitmap of cells whose span is >= h_min.
        band defaults to 4 voxels.  base_poses: submap -> world (R, T) to use instead of the stored base poses (a
        collection whose poses are kept elsewhere).  Flushes the queued frames.  -> dict: sc, ring, bev (torch CUDA
        tensors), n_points (numpy), M (f64 [n,3,3], the levelled rotations)."""
        from .. import place
        sm = [int(s) for s in np.asarray(submaps).reshape(-1)]
        L = place.level((0.0, 0.0, 1.0) if up is None else up)
        pose = self.base_pose if base_poses is None else (lambda s: base_poses[s])
        M = np.stack([L @ np.asarray(pose(s)[0], np.float64) for s in sm]) if sm else np.zeros((0, 3, 3))
        self._flush()
        band = 4.0 * self.voxel_scale if band is None else band
        out = self._h.place_describe(sm, M, r_max, h_min, band, min_weight)
        out["M"] = M
        return out

    def detect_loops(self, query_submaps, database_submaps=None, up=None, base_poses=None, **opts):
        """Find loop closures between the query submaps and the database on the GPU: describe every submap
        (describe_places), shortlist and coarsely align each query against the database (place.match: ring keys, the
        best yaw of the polar descriptor, the bird's-eye offset), then verify each candidate with D <= max_sc_dist and
        overlap >= min_overlap by registering it from the coarse pose (register_submaps, query = reference).  The
        database defaults to every submap up to the active one, queries included (a query never matches itself;
        entries need min_points points and submap ids at least min_gap apart).  opts: LOOP_DEFAULTS; max_cost defaults
        to (0.5 voxel)^2 / 2, the mean Huber cost of a half-voxel residual, huber and band to register_submaps'.
        base_poses: as describe_places.
        Returns one dict per verified candidate: query, match (submap ids), R, T (query local -> match local), H, b,
        sc_distance, yaw_deg, dx, dy, overlap, n_points, n_valid, cost (final, summed), converged, accepted (status 0,
        converged, n_valid >= min_points, n_valid / n_points >= min_inlier_ratio, cost / n_valid <= max_cost).  Moves
        nothing: the constraints are for the caller's pose graph."""
        from .. import place
        o = dict(self.LOOP_DEFAULTS)
        unknown = set(opts) - set(o)
        if unknown:
            raise TypeError(f"detect_loops: unknown options {sorted(unknown)}")
        o.update(opts)
        vs = self.voxel_scale
        max_cost = 0.5 * (0.5 * vs) ** 2 if o["max_cost"] is None else o["max_cost"]
        queries = [int(s) for s in np.asarray(query_submaps).reshape(-1)]
        if database_submaps is None:
            last = 0 if self.is_global_map else int(self.active_submap_id[None])
            database_submaps = range(0, max([last] + queries) + 1)
        entries = sorted(set(int(s) for s in database_submaps) | set(queries))
        at = {s: i for i, s in enumerate(entries)}
        desc = self.describe_places(entries, up=up, r_max=o["r_max"], h_min=o["h_min"], band=o["band"], min_weight=o["min_weight"],
                                    base_poses=base_poses)
        mt = place.match(desc["sc"], desc["ring"], desc["bev"], desc["n_points"], np.array(entries, np.int64), [at[q] for q in queries],
                         top_k=o["top_k"], min_gap=o["min_gap"], min_points=o["min_points"])
        cand = []
        for qi, q in enumerate(queries):
            if desc["n_points"][at[q]] < o["min_points"]:
                continue
            for k in range(o["top_k"]):
                d = int(mt["match"][qi, k])
                if d < 0 or not (mt["sc_dist"][qi, k] <= o["max_sc_dist"] and mt["overlap"][qi, k] >= o["min_overlap"]):
                    continue
                R0, T0 = place.coarse_pose(desc["M"][at[q]], desc["M"][d], mt["yaw_deg"][qi, k], mt["dx"][qi, k], mt["dy"][qi, k],
                                           o["r_max"])
                cand.append((q, entries[d], qi, k, R0, T0))
        out = []
        for c0 in range(0, len(cand), 1024):
            batch = cand[c0:c0 + 1024]
            res = self.register_submaps([c[0] for c in batch], [c[1] for c in batch],
                                        poses=(np.stack([c[4] for c in batch]), np.stack([c[5] for c in batch])), band=o["band"],
                                        min_weight=o["min_weight"], huber=o["huber"], max_iters=o["max_iters"],
                                        min_points=o["min_points"])
            for (q, d, qi, k, _, _), r in zip(batch, res):
                nv, npt = int(r["n_valid"]), int(r["n_points"])
                ok = (r["status"] == 0 and bool(r["converged"]) and nv >= o["min_points"] and npt > 0 and nv / npt >= o["min_inlier_ratio"]
                      and r["cost"] / max(nv, 1) <= max_cost)
                out.append(dict(query=q, match=d, R=r["R"], T=r["T"], H=r["H"], b=r["b"], sc_distance=float(mt["sc_dist"][qi, k]),
                                yaw_deg=float(mt["yaw_deg"][qi, k]), dx=int(mt["dx"][qi, k]), dy=int(mt["dy"][qi, k]),
                                overlap=float(mt["overlap"][qi, k]), n_points=npt, n_valid=nv, cost=float(r["cost"]),
                                converged=bool(r["converged"]), accepted=bool(ok)))
        return out

    def track_depth(self, R, T, depthmap, step=None, huber=None, max_iters=20, min_points=100):
        """Track one depth frame (uint16 mm [h,w]) against the TSDF of the active submap (submap 0 of a global map) on the
        GPU (tslam_tsdf_track_depth, DESIGN.md section 7, "Frame tracking"), before it is integrated: the pose at which
        the frame's points lie on the map's zero level.  R, T: the initial pose in the frame recast_depth_to_map takes.
        step defaults to recast_step, huber to one voxel.  Flushes the queued frames first.  -> dict: R, T (the tracked
        pose in the caller's frame, to hand to recast_depth_to_map; the input R, T unchanged, bit for bit, when status
        is 1 or no step was accepted), R_local, T_local (in the submap's local frame), H, b (information at the tracked
        pose, xi = (rho, phi) of the left perturbation in the local frame), cost_init, cost, n_points, n_valid,
        iterations, converged, status (1: fewer than min_points valid points at the initial pose)."""
        if self.K_cam_dep is None:
            raise RuntimeError("set_dep_camera_intrinsic() must be called before track_depth")
        depth = np.ascontiguousarray(depthmap, dtype=np.uint16)
        return self._track(R, T, lambda R0, T0, s: self._h.track_depth(depth, R0[None], T0[None], submaps=[s], step=step, huber=huber,
                                                                      max_iters=max_iters, min_points=min_points))

    def track_pcl(self, R, T, xyz_array, huber=None, max_iters=20, min_points=100):
        """track_depth for a point cloud xyz_array [n,3] in the sensor frame (recast_pcl_to_map's input): points that are
        not finite or whose range lies outside [min_ray_length, max_ray_length) are dropped.  -> the same dict."""
        xyz = np.ascontiguousarray(np.asarray(xyz_array, dtype=np.float32).reshape(-1, 3))
        return self._track(R, T, lambda R0, T0, s: self._h.track_points(xyz, R0, T0, submap=s, huber=huber, max_iters=max_iters,
                                                                       min_points=min_points))

    def _track(self, R, T, call):
        R_in, T_in = np.array(R, dtype=np.float64), np.array(T, dtype=np.float64).reshape(3)
        R0, T0 = self.convert_by_base(R_in, T_in)
        if self.submap_enabled:  # the base pose convert_by_base used
            b = self.active_submap_id[None]
            Rb, Tb = self.submaps_base_R_np[b], self.submaps_base_T_np[b]
        else:
            Rb, Tb = self.base_R_np, self.base_T_np
        out = call(R0, T0, self._active())
        res = {k: (v[0].copy() if v.ndim > 1 else v[0].item()) for k, v in out.items()}
        res["R_local"], res["T_local"] = res.pop("R"), res.pop("T")
        moved = not (np.array_equal(res["R_local"], R0) and np.array_equal(res["T_local"], T0))
        if res["status"] == 0 and moved:
            res["R"], res["T"] = Rb @ res["R_local"], Rb @ res["T_local"] + Tb
        else:
            res["R"], res["T"] = R_in, T_in
        return res

    def render(self, R, T, height, width, K=None, submap=None, z_min=None, z_max=None, step=None, color=False):
        """Depth, normal (and colour) images of the TSDF's zero level seen from a pinhole camera at pose R, T, in the frame
        recast_depth_to_map takes (tslam_tsdf_render, DESIGN.md section 7, "Rendering").  The pose is carried into the
        local frame of `submap` (default: the active submap, submap 0 of a global map) through that submap's base pose
        in f64.  K defaults to the depth intrinsics; z_min, z_max, step to min_ray_length, max_ray_length and the voxel
        scale.  Flushes the queued frames first.  -> dict of numpy arrays: depth f32 [h,w] (0: no hit), status u8 [h,w]
        (0 no hit, 1 hit, 2 hit without normal), normal f32 [h,w,3] in the caller's frame (NaN unless status is 1), and
        color f32 [h,w,3] when asked (textured maps)."""
        K = self.K_cam_dep if K is None else [float(k) for k in np.asarray(K).reshape(-1)]
        if K is None:
            raise RuntimeError("set_dep_camera_intrinsic() must be called before render, or K given")
        s = self._active() if submap is None else int(submap)
        if self.submap_enabled:
            Rb, Tb = self.submaps_base_R_np[s], self.submaps_base_T_np[s]
        else:
            Rb, Tb = self.base_R_np, self.base_T_np
        R, T = np.asarray(R, dtype=np.float64), np.asarray(T, dtype=np.float64).reshape(3)
        Rl, Tl = Rb.T @ R, Rb.T @ (T - Tb)  # convert_by_base, for submap s
        depth, status, nrm, col = self._h.render(Rl[None], Tl[None], height, width, K, submaps=[s], z_min=z_min, z_max=z_max,
                                                 step=step, color=color)
        out = dict(depth=depth[0].cpu().numpy(), status=status[0].cpu().numpy())
        out["normal"] = (nrm[0].cpu().numpy().astype(np.float64) @ np.asarray(Rb, np.float64).T).astype(np.float32)
        if color:
            out["color"] = col[0].cpu().numpy()
        return out
