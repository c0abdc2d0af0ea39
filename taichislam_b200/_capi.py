"""ctypes binding of libtslam.so (include/tslam.h) + thin device-buffer helpers.

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
