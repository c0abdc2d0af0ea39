"""ctypes binding of libtslam.so (include/tslam.h) + thin device-buffer helpers: the ABI's protocols (host-or-device
inputs, count-then-fill readers, counted exports, packing by destination rank, the submap table size), written once
for the TSDF, Octomap and mesh handles and the tiled global map.  Every tslam_* call stays at its call site.

There is NO CPU fallback: importing this module never touches the oracle, and every
compute entry point raises when the library or a CUDA device is missing.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtslam.so")

TSLAM_OK = 0
E_INVALID, E_CUDA, E_POOL_FULL, E_CAPACITY, E_NOGPU = -1, -2, -3, -4, -5
MEM_DEVICE, MEM_HOST = 0, 1
F_COMMIT = 1
MAX_BATCH = 64
REG_MAX_PAIRS = 1024
RENDER_MAX_CAMERAS = 1024
RENDER_MAX_SAMPLES = 65536
ABI_VERSION = 6
FUSE_REASONS = ("incremental", "first call", "full requested", "other source", "destination written", "content changed",
                "cheaper than subtract and re-add")
RECLAIM_ALL, RECLAIM_EMPTY, RECLAIM_OUTSIDE = 1, 2, 4
TILED_FUSE_REASONS = FUSE_REASONS + ("tile cuts changed", "sums not valid")  # tslam_tsdf_fuse_update_tiled_*


class TslamError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libtslam error {code}: {msg}")
        self.code = code


class TrajParams(C.Structure):
    """tslam_traj_params_t"""
    _fields_ = [("dt", C.c_double), ("v_max", C.c_double), ("a_max", C.c_double), ("w_smooth", C.c_double),
                ("w_collision", C.c_double), ("w_feasibility", C.c_double), ("w_unknown", C.c_double),
                ("clearance", C.c_double), ("g_tol", C.c_double), ("max_iters", C.c_int32), ("memory", C.c_int32),
                ("samples", C.c_int32), ("check_samples", C.c_int32)]


class TsdfConfig(C.Structure):
    _fields_ = [("voxel_scale", C.c_double), ("N", C.c_int32), ("Nz", C.c_int32),
                ("max_ray_length", C.c_double), ("min_ray_length", C.c_double),
                ("internal_voxels", C.c_int32), ("recast_step", C.c_int32),
                ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("is_global_map", C.c_int32),
                ("disp_floor", C.c_double), ("disp_ceiling", C.c_double),
                ("max_submaps", C.c_int32), ("max_blocks", C.c_int32),
                ("max_image_pixels", C.c_int32), ("max_points", C.c_int32), ("texture_enabled", C.c_int32)]


class OctoLogodds(C.Structure):
    _fields_ = [("l_hit", C.c_int32), ("l_miss", C.c_int32), ("l_min", C.c_int32), ("l_max", C.c_int32), ("l_occ", C.c_int32)]


class OctoConfig(C.Structure):
    _fields_ = [("voxel_scale", C.c_double), ("N", C.c_int32), ("Nz", C.c_int32), ("K", C.c_int32),
                ("max_ray_length", C.c_double), ("min_ray_length", C.c_double),
                ("recast_step", C.c_int32),
                ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("min_occupy_thres", C.c_int32), ("max_submaps", C.c_int32), ("max_blocks", C.c_int32),
                ("max_image_pixels", C.c_int32), ("max_points", C.c_int32), ("texture_enabled", C.c_int32)]


class ViewCamera(C.Structure):
    """tslam_view_camera_t: the simulated depth camera of the viewpoint-gain calls."""
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("width", C.c_int32),
                ("height", C.c_int32), ("step", C.c_int32), ("max_range", C.c_float)]


class PgParams(C.Structure):
    """tslam_pg_params_t"""
    _fields_ = [("eps_t", C.c_double), ("eps_r", C.c_double), ("cg_tol", C.c_double), ("max_iters", C.c_int32),
                ("max_cg", C.c_int32), ("pcg_grid", C.c_int32)]


_vp, _i32, _i64, _f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float

# name -> (restype, argtypes).  Every symbol declared in include/tslam.h appears here
# (tests/test_abi.py cross-checks this table against the header and the .so).
SIGNATURES = {
    "tslam_last_error": (C.c_char_p, []),
    "tslam_device_count": (C.c_int, []),
    "tslam_abi_version": (C.c_int, []),
    "tslam_tsdf_create": (C.c_int, [C.POINTER(TsdfConfig), C.POINTER(_vp)]),
    "tslam_tsdf_destroy": (C.c_int, [_vp]),
    "tslam_tsdf_reset": (C.c_int, [_vp, _vp]),
    "tslam_tsdf_set_intrinsics": (C.c_int, [_vp, C.c_double, C.c_double, C.c_double, C.c_double]),
    "tslam_tsdf_set_submap_pose": (C.c_int, [_vp, _i32, _vp, _vp]),
    "tslam_tsdf_integrate_depth": (C.c_int, [_vp, _vp, C.c_int, _i32, _i32, _i32, _vp, _vp, _vp, C.c_int, _vp]),
    "tslam_tsdf_queue_depth": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _i32, _vp]),
    "tslam_tsdf_flush": (C.c_int, [_vp, _vp]),
    "tslam_tsdf_set_frame_mode": (C.c_int, [_vp, C.c_int]),
    "tslam_tsdf_queue_depth_begin": (C.c_int, [_vp, _vp, _i32, _i32, _vp]),
    "tslam_tsdf_queue_depth_end": (C.c_int, [_vp, _vp, _vp, _i32, _vp]),
    "tslam_tsdf_set_queue_launch": (C.c_int, [_vp, _i32, _i32]),
    "tslam_tsdf_set_color_intrinsics": (C.c_int, [_vp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int]),
    "tslam_tsdf_integrate_depth_tex": (C.c_int, [_vp, _vp, _vp, C.c_int, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, C.c_int, _vp]),
    "tslam_tsdf_queue_depth_tex": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _vp]),
    "tslam_tsdf_integrate_points_rgb": (C.c_int, [_vp, _vp, _vp, C.c_int, _i32, _vp, _vp, _i32, C.c_int, _vp]),
    "tslam_tsdf_gather2": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_tsdf_scatter2": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tslam_mc_generate2": (C.c_int, [_vp, _i32, _f32, _i64, _vp, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_tsdf_integrate_points": (C.c_int, [_vp, _vp, C.c_int, _i32, _vp, _vp, _i32, C.c_int, _vp]),
    "tslam_tsdf_commit": (C.c_int, [_vp, _vp]),
    "tslam_tsdf_count_active": (C.c_int, [_vp, _i32, C.POINTER(_i64)]),
    "tslam_tsdf_gather": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_tsdf_scatter": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_fuse": (C.c_int, [_vp, _vp, _vp]),
    "tslam_tsdf_extract_surface": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_extract_slice": (C.c_int, [_vp, _i32, _f32, _f32, _i64, _vp, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_get_stats": (C.c_int, [_vp, _vp, C.c_int]),
    "tslam_tsdf_sync": (C.c_int, [_vp, _vp]),
    "tslam_tsdf_launch_count": (_i64, [_vp]),
    "tslam_tsdf_set_profiling": (C.c_int, [_vp, C.c_int]),
    "tslam_tsdf_kernel_ms": (C.c_int, [_vp, _i32, _vp, C.POINTER(_i32)]),
    "tslam_tsdf_kernel_ms2": (C.c_int, [_vp, _i32, _vp, C.POINTER(_i32)]),
    "tslam_tsdf_get_march_stats": (C.c_int, [_vp, _vp]),
    "tslam_tsdf_get_march_stats2": (C.c_int, [_vp, _vp]),
    "tslam_tsdf_query_points": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp]),
    "tslam_tsdf_query_near_occupy": (C.c_int, [_vp, _i32, _i64, _vp, _i32, _vp, _vp]),
    "tslam_tsdf_raycast": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _f32, _vp, _vp, _vp, _vp]),
    "tslam_octo_query_points": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp]),
    "tslam_octo_raycast": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _f32, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_fuse_pending": (C.c_int, [_vp, _vp, _vp]),
    "tslam_tsdf_commit_fused": (C.c_int, [_vp, _vp]),
    "tslam_tiling_owner": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, C.POINTER(_i32)]),
    "tslam_tiling_set_cuts": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_dirty_hist": (C.c_int, [_vp, _vp, _vp]),
    "tslam_tsdf_foreign_count": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp]),
    "tslam_tsdf_foreign_pack": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_unpack_add": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_halo_count": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp]),
    "tslam_tsdf_halo_pack": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _i64, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_ghost_unpack": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_foreign_pack2": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_unpack_add2": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_halo_pack2": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_ghost_unpack2": (C.c_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "tslam_tiling_owner_points": (C.c_int, [_vp, _vp, _i32, _i64, _vp, _vp, _vp]),
    "tslam_tiling_owner_cells": (C.c_int, [_vp, _vp, _i32, _i64, _vp, _vp, _vp]),
    "tslam_tsdf_raycast_tiled": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_query_near_occupy_tiled": (C.c_int, [_vp, _i32, _i64, _vp, _i32, _vp, _vp]),
    "tslam_esdf_tiled_begin": (C.c_int, [_vp, _i32, C.POINTER(_i32), _vp]),
    "tslam_esdf_halo_count": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _vp]),
    "tslam_esdf_halo_pack": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _i64, _vp, _vp, _vp]),
    "tslam_esdf_ghost_unpack": (C.c_int, [_vp, _i64, _vp, _vp, _vp]),
    "tslam_esdf_tiled_relax": (C.c_int, [_vp, C.POINTER(_i32), _vp]),
    "tslam_esdf_tiled_end": (C.c_int, [_vp]),
    "tslam_mc_generate": (C.c_int, [_vp, _i32, _f32, _i64, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_mesh_create": (C.c_int, [_vp, C.POINTER(_vp)]),
    "tslam_mesh_destroy": (C.c_int, [_vp]),
    "tslam_mesh_update": (C.c_int, [_vp, _f32, _i64, _vp, _vp, _vp, C.POINTER(_i64), _vp, _vp]),
    "tslam_mesh_updated_blocks": (C.c_int, [_vp, _i64, _vp, _vp, _vp, C.POINTER(_i64), C.POINTER(_i32), _vp]),
    "tslam_esdf_update": (C.c_int, [_vp, _i32, C.POINTER(_i32), _vp]),
    "tslam_esdf_update2": (C.c_int, [_vp, _i32, _i32, _vp, _vp]),
    "tslam_esdf_gather": (C.c_int, [_vp, _i32, _i64, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_esdf_query": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp, _vp, _vp]),
    "tslam_esdf_extract_slice": (C.c_int, [_vp, _i32, _f32, _i64, _vp, _vp, _vp, _vp]),
    "tslam_octo_create": (C.c_int, [C.POINTER(OctoConfig), C.POINTER(_vp)]),
    "tslam_octo_destroy": (C.c_int, [_vp]),
    "tslam_octo_reset": (C.c_int, [_vp, _vp]),
    "tslam_octo_set_submap_pose": (C.c_int, [_vp, _i32, _vp, _vp]),
    "tslam_octo_set_intrinsics": (C.c_int, [_vp, C.c_double, C.c_double, C.c_double, C.c_double]),
    "tslam_octo_integrate_points": (C.c_int, [_vp, _vp, C.c_int, _i32, _vp, _vp, _i32, _vp]),
    "tslam_octo_integrate_depth": (C.c_int, [_vp, _vp, C.c_int, _i32, _i32, _vp, _vp, _i32, _vp]),
    "tslam_octo_gather": (C.c_int, [_vp, _i32, _i64, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_octo_extract": (C.c_int, [_vp, _i32, _i32, _i64, _vp, _vp, _vp]),
    "tslam_octo_fuse": (C.c_int, [_vp, _vp, _vp]),
    "tslam_octo_fuse_update": (C.c_int, [_vp, _vp, _vp, _f32, _i32, _vp, _vp]),
    "tslam_octo_set_color_intrinsics": (C.c_int, [_vp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int]),
    "tslam_octo_integrate_points_rgb": (C.c_int, [_vp, _vp, _vp, C.c_int, _i32, _vp, _vp, _i32, _vp]),
    "tslam_octo_integrate_depth_tex": (C.c_int, [_vp, _vp, _vp, C.c_int, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _vp]),
    "tslam_octo_gather2": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_octo_extract2": (C.c_int, [_vp, _i32, _i32, _i64, _vp, _vp, _vp, _vp]),
    "tslam_octo_sync": (C.c_int, [_vp, _vp]),
    "tslam_octo_launch_count": (_i64, [_vp]),
    "tslam_octo_create_logodds": (C.c_int, [C.POINTER(OctoConfig), C.POINTER(OctoLogodds), C.POINTER(_vp)]),
    "tslam_octo_query_near_occupy": (C.c_int, [_vp, _i32, _i64, _vp, _i32, _vp, _vp]),
    "tslam_octo_gather_logodds": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_octo_get_stats": (C.c_int, [_vp, _vp, C.c_int]),
    "tslam_octo_esdf_update": (C.c_int, [_vp, _i32, _f32, _i32, _vp, _vp]),
    "tslam_octo_esdf_gather": (C.c_int, [_vp, _i32, _i64, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_octo_esdf_query": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp, _vp, _vp]),
    "tslam_octo_frontier_update": (C.c_int, [_vp, _i32, _i32, _vp, _vp]),
    "tslam_octo_frontier_gather": (C.c_int, [_vp, _i32, _i64, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_octo_frontier_clusters": (C.c_int, [_vp, _i32, _i64, _vp, C.POINTER(_i64), _vp]),
    "tslam_octo_view_gain_unknown": (C.c_int, [_vp, _i32, _i64, _vp, _vp, C.POINTER(ViewCamera), _vp, _vp, _vp]),
    "tslam_octo_view_gain_frontier": (C.c_int, [_vp, _i32, _i64, _vp, _vp, C.POINTER(ViewCamera), _i64, _vp, _vp, _vp, _vp]),
    "tslam_octo_frontier_viewpoints": (C.c_int, [_vp, _i32, C.POINTER(ViewCamera), _i32, _vp, _f32, _i32, _i32, _i64, _vp, _vp, _vp,
                                                 _vp, _vp, _vp]),
    "tslam_octo_travel_update": (C.c_int, [_vp, _i32, _vp, _f32, _f32, _vp, _vp]),
    "tslam_octo_travel_gather": (C.c_int, [_vp, _i32, _i64, _vp, _vp, C.POINTER(_i64), _vp]),
    "tslam_octo_travel_query": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp]),
    "tslam_octo_travel_path": (C.c_int, [_vp, _i32, _i64, _vp, _i32, _vp, _vp, _vp]),
    "tslam_octo_travel_multi_update": (C.c_int, [_vp, _i32, _i32, _vp, _f32, _f32, _vp, _vp, _vp, _vp]),
    "tslam_octo_travel_multi_query": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _vp]),
    "tslam_octo_travel_multi_path": (C.c_int, [_vp, _i32, _i64, _vp, _vp, _i32, _vp, _vp, _vp]),
    "tslam_tour_open": (C.c_int, [_i32, _vp, _i32, C.c_uint64, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tslam_tsdf_register": (C.c_int, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _i32, _i32, _vp, _vp, _vp, _vp, _vp,
                                      _vp, _vp]),
    "tslam_tsdf_track_depth": (C.c_int, [_vp, _vp, C.c_int, _i32, _i32, _i32, _vp, _vp, _vp, _i32, _f32, _i32, _i32, _vp, _vp, _vp, _vp,
                                         _vp, _vp, _vp]),
    "tslam_tsdf_track_points": (C.c_int, [_vp, _vp, C.c_int, _i32, _i32, _vp, _vp, _f32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                          _vp]),
    "tslam_tsdf_place_describe": (C.c_int, [_vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tslam_place_match": (C.c_int, [_i32, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _i32, _i64, _i64, _vp, _vp, _vp]),
    "tslam_tsdf_fuse_update": (C.c_int, [_vp, _vp, _vp, _f32, _i32, _vp, _vp]),
    "tslam_tsdf_reclaim": (C.c_int, [_vp, _i32, _vp, _vp, C.c_double, _vp, _vp]),
    "tslam_tsdf_block_keys": (C.c_int, [_vp, _i64, _vp, C.POINTER(_i64), _vp]),
    "tslam_tsdf_fuse_update_tiled_plan": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _vp, _f32, _i32, _vp, _vp, _vp]),
    "tslam_tsdf_fuse_update_tiled_splat": (C.c_int, [_vp, _vp, _i32, _vp]),
    "tslam_tsdf_fuse_update_tiled_pack": (C.c_int, [_vp, _vp, _i32, _i32, _vp, _i64, _vp, _vp]),
    "tslam_tsdf_fuse_update_tiled_unpack": (C.c_int, [_vp, _i64, _vp, _vp]),
    "tslam_tsdf_fuse_update_tiled_finish": (C.c_int, [_vp, _vp, _i32, _vp, _vp]),
    "tslam_tsdf_render": (C.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _vp, _vp, _vp, _vp, _vp]),
    "tslam_esdf_trajectory": (C.c_int, [_vp, _i32, _i32, _vp, _vp, C.POINTER(TrajParams), _vp, _vp, _vp, _vp]),
    "tslam_octo_esdf_trajectory": (C.c_int, [_vp, _i32, _i32, _vp, _vp, C.POINTER(TrajParams), _vp, _vp, _vp, _vp]),
    "tslam_pose_graph_solve": (C.c_int, [_i32, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, C.POINTER(PgParams), _vp, _vp, _vp,
                                         _vp, _vp, _vp, _vp]),
}

class PlaceParams(C.Structure):
    """tslam_place_params_t"""
    _fields_ = [("r_max", _f32), ("h_min", _f32), ("band", _f32), ("min_weight", _f32)]


_lib = None


def load():
    """Load libtslam.so (built in-tree by taichislam_b200.build).  Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing - run `python -m taichislam_b200.build` (nvcc, sm_90a). "
            "taichislam_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(L, name)  # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    if L.tslam_abi_version() != ABI_VERSION:
        raise ImportError("libtslam.so ABI version mismatch - rebuild it")
    _lib = L
    return L


def check(rc):
    if rc != TSLAM_OK:
        raise TslamError(rc, load().tslam_last_error().decode())


def require_gpu():
    if load().tslam_device_count() <= 0:
        raise TslamError(E_NOGPU, "no CUDA device visible - taichislam_b200 has no CPU fallback")


def np_ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def f32c(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64).astype(np.float32))


def stream_ptr():
    """The current torch CUDA stream as a void* for the ABI."""
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def tptr(t):
    """Device pointer of a torch CUDA tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def device():
    """The current CUDA device as a torch.device."""
    import torch
    return torch.device("cuda", torch.cuda.current_device())


def to_device(a, shape, dtype="float32"):
    """a as a contiguous CUDA tensor of `dtype` and `shape`: a torch tensor is converted on the device (no host
    synchronisation), anything else through numpy"""
    import torch
    dev = device()
    if isinstance(a, torch.Tensor):
        return a.to(device=dev, dtype=getattr(torch, dtype)).reshape(shape).contiguous()
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype).reshape(shape))).to(dev)


def results(as_torch, *tensors):
    """torch in -> the CUDA tensors, numpy in -> numpy arrays (one value for one tensor, else a tuple)"""
    r = tensors if as_torch else tuple(t.cpu().numpy() for t in tensors)
    return r if len(r) > 1 else r[0]


# -- inputs the C side reads from host or device memory (mem = MEM_HOST / MEM_DEVICE) -------------------------------
def source(a, np_dtype, torch_dtypes, shape=None):
    """A depth frame or point cloud -> (a, mem, ptr, shape): a torch CUDA tensor (contiguous, dtype in torch_dtypes) is
    read on the device; anything else becomes a contiguous numpy array of np_dtype (reshaped to `shape` when given),
    returned as `a` so that it outlives the call."""
    import torch
    if isinstance(a, torch.Tensor):
        assert a.is_cuda and a.dtype in torch_dtypes and a.is_contiguous()
        return a, MEM_DEVICE, tptr(a), tuple(a.shape)
    a = np.asarray(a, dtype=np_dtype)
    a = np.ascontiguousarray(a if shape is None else a.reshape(shape))
    return a, MEM_HOST, np_ptr(a), a.shape


def companion(c, mem):
    """The uint8 colour (texture or rgb) of a source in memory space mem -> (c, ptr), (None, None) for none: a
    contiguous torch CUDA tensor with a device source, else a contiguous numpy array, returned as `c` so that it
    outlives the call.  The caller checks its shape."""
    import torch
    if c is None:
        return None, None
    if isinstance(c, torch.Tensor):
        assert mem == MEM_DEVICE and c.is_cuda and c.dtype == torch.uint8 and c.is_contiguous()
        return c, tptr(c)
    assert mem == MEM_HOST
    c = np.ascontiguousarray(c, dtype=np.uint8)
    return c, np_ptr(c)


# -- readers -----------------------------------------------------------------------------------------------------------
def count_fill(call, *alloc, cap=None):
    """The two-call protocol of a count-then-fill reader.  call(cap, n_ref, *ptrs) makes the C call; a probe with
    cap 0 and NULL buffers gives the count n (unless cap is given).  Without alloc that count is the result; else
    each (trailing shape, torch dtype) of alloc becomes a device tensor [max(n, 1), *shape], the second call fills
    them, and they come back sliced to the rows written."""
    import torch
    n = C.c_int64(0)
    if cap is None:
        rc = call(0, C.byref(n), *(None for _ in alloc))
        if rc not in (TSLAM_OK, E_CAPACITY):
            check(rc)
        cap = int(n.value)
        if not alloc:
            return cap
    dev = device()
    out = [torch.empty((max(cap, 1),) + tuple(shape), dtype=dt, device=dev) for shape, dt in alloc]
    check(call(cap, C.byref(n), *(tptr(t) for t in out)))
    k = int(n.value)
    return tuple(t[:k] for t in out)


def extract(call, cap, *alloc):
    """The device-counter protocol of an export.  Each (trailing shape, torch dtype[, zeroed]) of alloc becomes a device
    tensor of cap rows (zero-filled when zeroed: rows the call may leave unwritten; cap 0 still gets a valid buffer, so
    it asks for the count alone); call(count, *tensors) appends to them and adds the rows it wanted to count (int32[1]
    on the device).  -> (wanted, *the rows written as numpy arrays)."""
    import torch
    dev = device()
    out = [(torch.zeros if any(zeroed) else torch.empty)((max(cap, 1),) + tuple(shape), dtype=dt, device=dev)
           for shape, dt, *zeroed in alloc]
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    call(cnt, *(t[:cap] for t in out))
    n = int(cnt.item())
    k = min(n, cap)
    return (n,) + tuple(t[:k].cpu().numpy() for t in out)


def pack(count, fill, world, *alloc):
    """Rows grouped by destination rank: count(counts) writes the rows per rank into counts (host int32[world]); each
    (trailing shape, torch dtype) of alloc becomes a device tensor of max(n, 1) rows, n the total; fill(counts, n,
    *ptrs) packs them.  -> (counts, the tensors sliced to n rows)."""
    import torch
    send = np.zeros(int(world), np.int32)
    check(count(np_ptr(send)))
    n = int(send.sum())
    dev = device()
    out = [torch.empty((max(n, 1),) + tuple(shape), dtype=dt, device=dev) for shape, dt in alloc]
    check(fill(np_ptr(send), n, *(tptr(t) for t in out)))
    return send, tuple(t[:n] for t in out)


def owner_ranks(fn, h, tiles_c, world, rank, xyz):
    """Points f32[n,3] on the device and the rank that answers each: fn (tslam_tiling_owner_points or _cells) names
    the owning tile; owner < 0 (no tile holds the point) means this rank."""
    import torch
    x = to_device(xyz, (-1, 3))
    owner = torch.empty(x.shape[0], dtype=torch.int32, device=x.device)
    check(fn(h, tiles_c, world, x.shape[0], tptr(x), tptr(owner), stream_ptr()))
    return x, torch.where(owner < 0, torch.full_like(owner, rank), owner).long()


# -- planner queries shared by the TSDF and Octomap handles: fn is the map's tslam_* entry -----------------------------
def query_flags(fn, h, xyz, submap):
    """uint8 flags per point of a *_query_points entry, numpy."""
    import torch
    x = to_device(xyz, (-1, 3))
    f = torch.empty(x.shape[0], dtype=torch.uint8, device=x.device)
    check(fn(h, int(submap), x.shape[0], tptr(x), tptr(f), stream_ptr()))
    return f.cpu().numpy()


def near_occupy(fn, h, xyz, voxel, submap):
    """is_near_pos_occupy per point of a *_query_near_occupy entry, numpy bool."""
    import torch
    x = to_device(xyz, (-1, 3))
    f = torch.empty(x.shape[0], dtype=torch.uint8, device=x.device)
    check(fn(h, int(submap), x.shape[0], tptr(x), int(voxel), tptr(f), stream_ptr()))
    return f.cpu().numpy().astype(bool)


def raycast(fn, h, pos, direction, max_dist, submap):
    """(hit bool, last position f32[n,3], length f32) per ray of a *_raycast entry, numpy."""
    import torch
    p, d = to_device(pos, (-1, 3)), to_device(direction, (-1, 3))
    n = p.shape[0]
    hit = torch.empty(n, dtype=torch.uint8, device=p.device)
    xyz = torch.empty((n, 3), dtype=torch.float32, device=p.device)
    ln = torch.empty(n, dtype=torch.float32, device=p.device)
    check(fn(h, int(submap), n, tptr(p), tptr(d), float(max_dist), tptr(hit), tptr(xyz), tptr(ln), stream_ptr()))
    return hit.cpu().numpy().astype(bool), xyz.cpu().numpy(), ln.cpu().numpy()


def esdf_query(fn, h, xyz, submap):
    """(dist f32[n], grad f32[n,3], valid bool[n]) of an *esdf_query entry: torch in -> torch out without a host
    synchronisation, numpy in -> numpy out."""
    import torch
    x = to_device(xyz, (-1, 3))
    n = x.shape[0]
    dist = torch.empty(n, dtype=torch.float32, device=x.device)
    grad = torch.empty((n, 3), dtype=torch.float32, device=x.device)
    valid = torch.empty(n, dtype=torch.uint8, device=x.device)
    check(fn(h, int(submap), n, tptr(x), tptr(dist), tptr(grad), tptr(valid), stream_ptr()))
    return results(isinstance(xyz, torch.Tensor), dist, grad, valid.view(torch.bool))  # the kernel writes 0 / 1


# -- incremental fusion ------------------------------------------------------------------------------------------------
def submap_table(n):
    """The submap table size of a map created with max_submaps = n: tslam_tsdf_create and tslam_octo_create
    (csrc/tslam_tsdf.cu, csrc/tslam_octo.cu) replace a value outside (0, 1024] by 1024."""
    n = int(n)
    return n if 0 < n <= 1024 else 1024


def include_u8(include, n):
    """include of the fusion updates (None or bools / 0-1 per submap) -> None or u8[n], n the submap table size."""
    if include is None:
        return None
    a = np.asarray(include).reshape(-1).astype(bool)
    assert a.shape[0] <= n, "include has more entries than max_submaps"
    inc = np.zeros(n, np.uint8)
    inc[:a.shape[0]] = a
    return inc


def fuse_stats(st, reasons):
    return dict(full=bool(st[0] != 0), reason=reasons[int(st[0])], added=int(st[1]), moved=int(st[2]), removed=int(st[3]),
                within_tolerance=int(st[4]), voxels_splatted=int(st[5]), voxels_skipped=int(st[6]), blocks_committed=int(st[7]))


def fuse_update(fn, dst, src, include, tolerance, full):
    """The body of the handles' fuse_update: fn is tslam_tsdf_fuse_update or tslam_octo_fuse_update."""
    inc = include_u8(include, submap_table(dst.cfg.max_submaps))
    st = np.zeros(8, np.int64)
    check(fn(dst.h, src.h, np_ptr(inc) if inc is not None else None, float(tolerance), int(bool(full)), np_ptr(st),
             stream_ptr()))
    return fuse_stats(st, FUSE_REASONS)
