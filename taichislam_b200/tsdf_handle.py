"""TsdfHandle - the thinnest Python face of the TSDF part of the C ABI.

Used by the reference-surface classes in taichislam_b200.mapping, by bench.py and by
the parity tests (which therefore exercise the C ABI, not private Python helpers).
"""
import ctypes as C

import numpy as np

from . import _capi as capi


class TsdfHandle:
    def __init__(self, N, Nz, voxel_scale=0.05, max_ray_length=10.0, min_ray_length=0.3, internal_voxels=10,
                 recast_step=2, K=None, is_global_map=False, disp_floor=-0.3, disp_ceiling=1.8, max_submaps=1024,
                 max_blocks=0, max_image_pixels=0, max_points=0, texture_enabled=False):
        capi.require_gpu()
        import torch  # device buffers / streams only
        self.torch = torch
        L = capi.load()
        K = K if K is not None else [1, 0, 0, 0, 1, 0, 0, 0, 1]
        self.cfg = capi.TsdfConfig(voxel_scale, N, Nz, max_ray_length, min_ray_length, internal_voxels, recast_step,
                                   K[0], K[4], K[2], K[5], int(is_global_map), disp_floor, disp_ceiling,
                                   max_submaps, max_blocks, max_image_pixels, max_points, int(bool(texture_enabled)))
        self.texture_enabled = bool(texture_enabled)
        h = C.c_void_p()
        torch.cuda.init()
        torch.cuda.current_stream()  # make sure the primary context exists and is current
        capi.check(L.tslam_tsdf_create(C.byref(self.cfg), C.byref(h)))
        self.h = h
        self.L = L
        self.N, self.Nz = N, Nz

    def close(self):
        if getattr(self, "h", None):
            self.L.tslam_tsdf_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- state ---------------------------------------------------------------------------
    def reset(self):
        capi.check(self.L.tslam_tsdf_reset(self.h, capi.stream_ptr()))

    def set_intrinsics(self, K9):
        capi.check(self.L.tslam_tsdf_set_intrinsics(self.h, K9[0], K9[4], K9[2], K9[5]))

    def set_color_intrinsics(self, K9, color_same_proj=False):
        """set_color_camera_intrinsic (mapping_common.py:28-29) + color_same_proj (dense_tsdf.py:16)."""
        capi.check(self.L.tslam_tsdf_set_color_intrinsics(self.h, K9[0], K9[4], K9[2], K9[5], int(bool(color_same_proj))))

    def set_submap_pose(self, s, R, T):
        R, T = capi.f32c(R).reshape(9), capi.f32c(T).reshape(3)
        capi.check(self.L.tslam_tsdf_set_submap_pose(self.h, int(s), capi.np_ptr(R), capi.np_ptr(T)))

    # -- integrate ------------------------------------------------------------------------
    def integrate_depth(self, depth, Rs, Ts, submaps=None, commit=True, texture=None):
        """depth: uint16 [n,h,w] (or [h,w]) numpy (host) or torch CUDA tensor; Rs [n,3,3]; Ts [n,3];
        texture: uint8 [n,th,tw,3] in the same memory space as depth (textured maps)."""
        depth, mem, ptr, shape = capi.source(depth, np.uint16, (self.torch.uint16, self.torch.int16))
        if len(shape) == 2:
            shape = (1,) + tuple(shape)
        n, h, w = shape
        Rs = capi.f32c(Rs).reshape(n, 9)
        Ts = capi.f32c(Ts).reshape(n, 3)
        sm = None
        if submaps is not None:
            sm = np.ascontiguousarray(np.broadcast_to(np.asarray(submaps, dtype=np.int32), (n,)))
        texture, tptr = capi.companion(texture, mem)
        tshape = (0, 0, 0, 3)
        if texture is not None:
            tshape = tuple(texture.shape)
            if len(tshape) == 3:
                tshape = (1,) + tshape
            assert tshape[0] == n and tshape[3] == 3
        capi.check(self.L.tslam_tsdf_integrate_depth_tex(self.h, ptr, tptr, mem, n, h, w, tshape[1], tshape[2], capi.np_ptr(Rs),
                                                         capi.np_ptr(Ts), capi.np_ptr(sm) if sm is not None else None,
                                                         capi.F_COMMIT if commit else 0, capi.stream_ptr()))

    def integrate_points(self, xyz, R, T, submap=0, commit=True, rgb=None):
        xyz, mem, ptr, shape = capi.source(xyz, np.float32, (self.torch.float32,), (-1, 3))
        n = shape[0]
        R, T = capi.f32c(R).reshape(9), capi.f32c(T).reshape(3)
        rgb, cptr = capi.companion(rgb, mem)
        if rgb is not None:
            assert tuple(rgb.shape) == (n, 3)
        capi.check(self.L.tslam_tsdf_integrate_points_rgb(self.h, ptr, cptr, mem, n, capi.np_ptr(R), capi.np_ptr(T), int(submap),
                                                          capi.F_COMMIT if commit else 0, capi.stream_ptr()))

    def commit(self):
        capi.check(self.L.tslam_tsdf_commit(self.h, capi.stream_ptr()))

    def sync(self):
        capi.check(self.L.tslam_tsdf_sync(self.h, capi.stream_ptr()))

    # -- readers --------------------------------------------------------------------------
    def count_active(self, submap=0):
        self.torch.cuda.current_stream().synchronize()
        n = C.c_int64(0)
        capi.check(self.L.tslam_tsdf_count_active(self.h, int(submap), C.byref(n)))
        return int(n.value)

    def gather_device(self, submap=0, cap=None, color=False):
        """Observed voxels of `submap` as torch CUDA tensors (idx int32[n,3], tsdf, w f32[n], occ int8[n]
        [, color f32[n,3]])."""
        torch = self.torch
        if cap is None:
            cap = self.count_active(submap)
        alloc = [((3,), torch.int32), ((), torch.float32), ((), torch.float32), ((), torch.int8)] + ([((3,), torch.float32)] if color else [])
        return capi.count_fill(lambda cap, n, idx, t, w, occ, col=None: self.L.tslam_tsdf_gather2(
            self.h, int(submap), cap, idx, t, w, occ, col, n, capi.stream_ptr()), *alloc, cap=cap)

    def gather(self, submap=0, color=False):
        return tuple(a.cpu().numpy() for a in self.gather_device(submap, color=color))

    def scatter(self, submap, idx, tsdf, w, occ, color=None):
        idx = capi.to_device(idx, (-1, 3), "int32")
        n = idx.shape[0]
        tsdf, w = capi.to_device(tsdf, (-1,)), capi.to_device(w, (-1,))
        occ = capi.to_device(occ, (-1,), "int8")
        if color is not None:
            color = capi.to_device(color, (n, 3))
        capi.check(self.L.tslam_tsdf_scatter2(self.h, int(submap), n, capi.tptr(idx), capi.tptr(tsdf), capi.tptr(w), capi.tptr(occ),
                                              capi.tptr(color), capi.stream_ptr()))
        self.torch.cuda.current_stream().synchronize()  # the temporaries above must outlive the kernel

    def fuse_from(self, src):
        capi.check(self.L.tslam_tsdf_fuse(self.h, src.h, capi.stream_ptr()))

    def fuse_update(self, src, include=None, tolerance=0.0, full=False):
        """Incremental fusion of the submaps of `src` (a TsdfHandle) into this global map (tslam_tsdf_fuse_update):
        afterwards this map is the exact-sum fusion of the included submaps at their fused poses.  include: None (all) or
        bools / 0-1 per submap (up to max_submaps); tolerance: how far (metres, translation + angle x radius) a fused
        submap may move before it is re-splatted; full=True forces a rebuild.  -> dict of the call's statistics."""
        return capi.fuse_update(self.L.tslam_tsdf_fuse_update, self, src, include, tolerance, full)

    def reclaim(self, submaps=None, all_blocks=False, empty=False, center=None, radius=None):
        """Drop pool blocks and compact the pool in place (tslam_tsdf_reclaim).  Candidates are the blocks of `submaps`
        (None: every submap; else ids or bools / 0-1 per submap); a candidate is dropped when all_blocks, when empty and
        it holds no observed voxel, or when center / radius are given and it lies outside that sphere (metres, in the
        frame the map stores its submaps in).  -> dict of the call's statistics."""
        rules = (capi.RECLAIM_ALL if all_blocks else 0) | (capi.RECLAIM_EMPTY if empty else 0)
        c = None
        if center is not None or radius is not None:
            assert center is not None and radius is not None, "OUTSIDE needs both center and radius"
            rules |= capi.RECLAIM_OUTSIDE
            c = np.ascontiguousarray(np.asarray(center, np.float64).reshape(3))
        mask = self.submap_mask_u8(submaps)
        st = np.zeros(6, np.int64)
        capi.check(self.L.tslam_tsdf_reclaim(self.h, rules, capi.np_ptr(mask) if mask is not None else None,
                                             capi.np_ptr(c) if c is not None else None, float(radius) if c is not None else 0.0,
                                             capi.np_ptr(st), capi.stream_ptr()))
        return dict(blocks_before=int(st[0]), candidates=int(st[1]), dropped=int(st[2]), dropped_nonempty=int(st[3]),
                    moved=int(st[4]), blocks_after=int(st[5]))

    def submap_mask_u8(self, submaps):
        """None, submap ids, or bools / 0-1 per submap -> None or u8[submap table size]."""
        if submaps is None:
            return None
        a = np.asarray(submaps).reshape(-1)
        if a.dtype == bool:
            return self.include_u8(a)
        n = capi.submap_table(self.cfg.max_submaps)
        ids = a.astype(np.int64)
        assert np.all((ids >= 0) & (ids < n)), "submap id out of range"
        mask = np.zeros(n, np.uint8)
        mask[ids] = 1
        return mask

    def block_keys(self):
        """The pool in slot order: int32[n_blocks, 4] rows (submap, bx, by, bz)."""
        (keys,) = capi.count_fill(lambda cap, n, keys: self.L.tslam_tsdf_block_keys(self.h, cap, keys, n, capi.stream_ptr()),
                                  ((4,), self.torch.int32))
        return keys.cpu().numpy()

    def include_u8(self, include):
        """include of the fusion updates (None or bools / 0-1 per submap) -> None or u8[submap table size]."""
        return capi.include_u8(include, capi.submap_table(self.cfg.max_submaps))

    # -- incremental fusion of a tiled global map, phase by phase (tslam_tsdf_fuse_update_tiled_*) ------------------
    # distributed.TiledGlobalMap.update_fused_submaps drives these on every rank; each raises capi.TslamError.
    def fuse_update_tiled_plan(self, src, tiles, rank, world, include=None, tolerance=0.0, full=False):
        """-> (plan int64[3] = this rank's full-update reason, cost, cost_full; present bool[submap table size])."""
        inc = self.include_u8(include)
        plan = np.zeros(3, np.int64)
        present = np.zeros(capi.submap_table(self.cfg.max_submaps), np.uint8)
        t = (C.c_int32 * 3)(*tiles)
        capi.check(self.L.tslam_tsdf_fuse_update_tiled_plan(self.h, src.h, t, int(rank), int(world), capi.np_ptr(inc) if inc is not None else None,
                                                            float(tolerance), int(bool(full)), capi.np_ptr(plan), capi.np_ptr(present),
                                                            capi.stream_ptr()))
        return plan, present.astype(bool)

    def fuse_update_tiled_splat(self, src, reason):
        capi.check(self.L.tslam_tsdf_fuse_update_tiled_splat(self.h, src.h, int(reason), capi.stream_ptr()))

    def fuse_update_tiled_pack(self, tiles, rank, world):
        """-> (rows per destination rank int32[world], rows int64[n, 1 + planes * 4096] torch CUDA, grouped by destination)."""
        t = (C.c_int32 * 3)(*tiles)
        planes = 6 if self.texture_enabled else 3
        send, (rows,) = capi.pack(
            lambda send: self.L.tslam_tsdf_foreign_count(self.h, t, int(rank), int(world), send, capi.stream_ptr()),
            lambda send, n, rows: self.L.tslam_tsdf_fuse_update_tiled_pack(self.h, t, int(rank), int(world), send, n, rows,
                                                                          capi.stream_ptr()),
            world, ((1 + planes * 4096,), self.torch.int64))
        return send, rows

    def fuse_update_tiled_unpack(self, rows):
        rows = rows.contiguous()
        capi.check(self.L.tslam_tsdf_fuse_update_tiled_unpack(self.h, rows.shape[0], capi.tptr(rows), capi.stream_ptr()))

    def fuse_update_tiled_finish(self, src, ok):
        """-> this rank's statistics (as fuse_update's) when ok, else None."""
        st = np.zeros(8, np.int64)
        capi.check(self.L.tslam_tsdf_fuse_update_tiled_finish(self.h, src.h, int(bool(ok)), capi.np_ptr(st), capi.stream_ptr()))
        return capi.fuse_stats(st, capi.TILED_FUSE_REASONS) if ok else None

    def extract_surface(self, submap, xyz, rgb, count):
        """Append to torch CUDA buffers xyz/rgb f32[cap,3]; count: int32[1] device counter."""
        capi.check(self.L.tslam_tsdf_extract_surface(self.h, int(submap), xyz.shape[0], capi.tptr(xyz), capi.tptr(rgb),
                                                     capi.tptr(count), capi.stream_ptr()))

    def extract_slice(self, submap, z, dz, xyz, val, rgb, count):
        capi.check(self.L.tslam_tsdf_extract_slice(self.h, int(submap), float(z), float(dz), xyz.shape[0], capi.tptr(xyz),
                                                   capi.tptr(val), capi.tptr(rgb), capi.tptr(count), capi.stream_ptr()))

    def surface(self, submap=0, cap=1 << 22):
        f32 = self.torch.float32
        return capi.extract(lambda cnt, xyz, rgb: self.extract_surface(submap, xyz, rgb, cnt), cap, ((3,), f32), ((3,), f32))

    def slice(self, z, dz=0.5, submap=0, cap=1 << 22):
        f32 = self.torch.float32
        return capi.extract(lambda cnt, xyz, val: self.extract_slice(submap, z, dz, xyz, val, None, cnt), cap, ((3,), f32), ((), f32))

    def marching_cubes(self, step=1, thres=0.1, cap_tri=1 << 21, color=False):
        torch = self.torch
        dev = capi.device()
        v = torch.empty((3 * cap_tri, 3), dtype=torch.float32, device=dev)
        nrm = torch.empty((3 * cap_tri, 3), dtype=torch.float32, device=dev)
        col = torch.empty((3 * cap_tri, 3), dtype=torch.float32, device=dev) if color else None
        n = C.c_int64(0)
        rc = self.L.tslam_mc_generate2(self.h, int(step), float(thres), cap_tri, capi.tptr(v), capi.tptr(nrm), capi.tptr(col), C.byref(n),
                                       capi.stream_ptr())
        if rc != capi.E_CAPACITY:
            capi.check(rc)
        k = min(int(n.value), cap_tri)
        if color:
            return int(n.value), v[:3 * k].cpu().numpy(), nrm[:3 * k].cpu().numpy(), col[:3 * k].cpu().numpy()
        return int(n.value), v[:3 * k].cpu().numpy(), nrm[:3 * k].cpu().numpy()

    # -- planner queries (batched @ti.func helpers of BaseMap, mapping_common.py:165-204) ------------------
    def query_points(self, xyz, submap=0):
        """(is_pos_occupy, is_pos_unobserved) per point."""
        f = capi.query_flags(self.L.tslam_tsdf_query_points, self.h, xyz, submap)
        return (f & 1).astype(bool), (f & 2).astype(bool)

    def query_near_occupy(self, xyz, voxel, submap=0):
        return capi.near_occupy(self.L.tslam_tsdf_query_near_occupy, self.h, xyz, voxel, submap)

    def raycast(self, pos, direction, max_dist, submap=0):
        """BaseMap.raycast for a batch of rays: (hit, last position, length)."""
        return capi.raycast(self.L.tslam_tsdf_raycast, self.h, pos, direction, max_dist, submap)

    def esdf_update(self, submap=0):
        sw = C.c_int32(0)
        capi.check(self.L.tslam_esdf_update(self.h, int(submap), C.byref(sw), capi.stream_ptr()))
        return int(sw.value)

    def esdf_update2(self, submap=0, full=False):
        """-> dict(lower_sweeps, raise_sweeps (-1: full recompute), changed, suspect)."""
        st = np.zeros(4, np.int32)
        capi.check(self.L.tslam_esdf_update2(self.h, int(submap), 1 if full else 0, capi.np_ptr(st), capi.stream_ptr()))
        return dict(lower_sweeps=int(st[0]), raise_sweeps=int(st[1]), changed=int(st[2]), suspect=int(st[3]))

    # -- ESDF of a tiled global map (the exchange between the phases is taichislam_b200.distributed's) ----------
    def esdf_tiled_begin(self, submap=0):
        """Seed owned and ghost blocks, run the local wave with ghosts as read-only sources -> sweeps."""
        sw = C.c_int32(0)
        capi.check(self.L.tslam_esdf_tiled_begin(self.h, int(submap), C.byref(sw), capi.stream_ptr()))
        return int(sw.value)

    def esdf_ghost_unpack(self, keys, esdf):
        """Overwrite the ESDF of existing ghost blocks: keys int64[n], esdf f32[n,4096] torch CUDA tensors."""
        n = int(keys.shape[0])
        capi.check(self.L.tslam_esdf_ghost_unpack(self.h, n, capi.tptr(keys), capi.tptr(esdf), capi.stream_ptr()))

    def esdf_tiled_relax(self):
        """The wave from the ghosts unpacked since the last relax -> sweeps."""
        sw = C.c_int32(0)
        capi.check(self.L.tslam_esdf_tiled_relax(self.h, C.byref(sw), capi.stream_ptr()))
        return int(sw.value)

    def esdf_tiled_end(self):
        capi.check(self.L.tslam_esdf_tiled_end(self.h))

    def esdf_gather(self, submap=0):
        torch = self.torch
        cap = self.count_active(submap)
        idx, e = capi.count_fill(lambda cap, n, idx, e: self.L.tslam_esdf_gather(self.h, int(submap), cap, idx, e, n, capi.stream_ptr()),
                                 ((3,), torch.int32), ((), torch.float32), cap=cap)
        return idx.cpu().numpy(), e.cpu().numpy()

    def esdf_query(self, xyz, submap=0):
        """Trilinear ESDF and its exact gradient at points [n,3] of the submap's map frame, as of the last esdf_update of
        `submap`: (dist f32[n], grad f32[n,3], valid bool[n]); dist and grad are NaN where valid is False.
        A torch CUDA tensor in -> torch CUDA tensors out, enqueued on the current stream without a host synchronisation
        (a planner's torch loop can call it); a numpy array in -> numpy arrays out."""
        return capi.esdf_query(self.L.tslam_esdf_query, self.h, xyz, submap)

    def trajectory(self, ctrls, clearance, submap=0, **settings):
        """Optimise uniform cubic B-splines (control points f[N,3] each, the submap's map frame) against the ESDF of
        `submap` as of its last esdf_update (tslam_esdf_trajectory) -> a list of dicts (trajectory.solve).  settings:
        trajectory.DEFAULTS."""
        from . import trajectory
        return trajectory.solve(self.L.tslam_esdf_trajectory, self.h, submap, ctrls, clearance, **settings)

    def esdf_extract_slice(self, submap, z, xyz, val, count):
        """Append the ESDF slice at height z to torch CUDA buffers xyz f32[cap,3] / val f32[cap]; count: int32[1] device counter."""
        capi.check(self.L.tslam_esdf_extract_slice(self.h, int(submap), float(z), xyz.shape[0], capi.tptr(xyz), capi.tptr(val),
                                                   capi.tptr(count), capi.stream_ptr()))

    def esdf_slice(self, z, submap=0, cap=1 << 22):
        """cvt_ESDF_to_voxels_slice (dense_esdf.py:498-509) as of the last esdf_update: (demand, xyz, ESDF) numpy."""
        f32 = self.torch.float32
        return capi.extract(lambda cnt, xyz, val: self.esdf_extract_slice(submap, z, xyz, val, cnt), cap, ((3,), f32), ((), f32))

    # -- SDF-to-SDF registration of submap pairs (tslam_tsdf_register) -------------------------------------
    def register(self, reading, ref_submaps, read_submaps, R0, T0, band, min_weight=0.0, huber=None, max_iters=20,
                 min_points=100):
        """Register reference submaps of this map against reading submaps of `reading` (a TsdfHandle, may be self).
        R0 [P,3,3], T0 [P,3]: initial poses (reference local frame -> reading local frame), f64.  huber defaults to the
        voxel scale.  -> dict of numpy arrays: R [P,3,3], T [P,3], H [P,6,6], b [P,6], cost_init, cost [P], n_points,
        n_valid, iterations [P] int64, converged, status [P] int64 (1: fewer than min_points valid points at R0, T0)."""
        a = np.ascontiguousarray(np.asarray(ref_submaps, dtype=np.int32).reshape(-1))
        r = np.ascontiguousarray(np.asarray(read_submaps, dtype=np.int32).reshape(-1))
        P = a.shape[0]
        R0 = np.ascontiguousarray(np.asarray(R0, dtype=np.float64).reshape(P, 9))
        T0 = np.ascontiguousarray(np.asarray(T0, dtype=np.float64).reshape(P, 3))
        huber = float(self.cfg.voxel_scale) if huber is None else float(huber)
        R, T = np.zeros((P, 9)), np.zeros((P, 3))
        H, b, cost2 = np.zeros((P, 36)), np.zeros((P, 6)), np.zeros((P, 2))
        info = np.zeros((P, 5), np.int64)
        capi.check(self.L.tslam_tsdf_register(self.h, reading.h, P, capi.np_ptr(a), capi.np_ptr(r), capi.np_ptr(R0), capi.np_ptr(T0),
                                              float(band), float(min_weight), huber, int(max_iters), int(min_points), capi.np_ptr(R),
                                              capi.np_ptr(T), capi.np_ptr(H), capi.np_ptr(b), capi.np_ptr(cost2), capi.np_ptr(info),
                                              capi.stream_ptr()))
        return self._solver_out(P, R, T, H, b, cost2, info)

    # -- place descriptors for loop detection (tslam_tsdf_place_describe) --------------------------------------------
    def place_describe(self, submaps, M, r_max, h_min, band, min_weight=0.0):
        """Place descriptors of `submaps` (DESIGN.md section 7, "Loop detection"): M [n,3,3] the levelled rotations (f64,
        rounded to f32 here).  -> dict: sc f32 [n,20,60], ring f32 [n,20], bev int32 [n,512] (the uint32 words' bits)
        as torch CUDA tensors, n_points int64 [n] numpy."""
        torch = self.torch
        sm = np.ascontiguousarray(np.asarray(submaps, dtype=np.int32).reshape(-1))
        n = sm.shape[0]
        M9 = np.ascontiguousarray(np.asarray(M, dtype=np.float64).reshape(n, 9).astype(np.float32))
        params = capi.PlaceParams(float(r_max), float(h_min), float(band), float(min_weight))
        dev = capi.device()
        rows = max(n, 1)
        sc = torch.empty((rows, 20, 60), dtype=torch.float32, device=dev)
        ring = torch.empty((rows, 20), dtype=torch.float32, device=dev)
        bev = torch.empty((rows, 512), dtype=torch.int32, device=dev)
        npts = np.zeros(rows, np.int64)
        capi.check(self.L.tslam_tsdf_place_describe(self.h, n, capi.np_ptr(sm), capi.np_ptr(M9), C.byref(params), capi.tptr(sc),
                                                    capi.tptr(ring), capi.tptr(bev), capi.np_ptr(npts), capi.stream_ptr()))
        return dict(sc=sc[:n], ring=ring[:n], bev=bev[:n], n_points=npts[:n])

    @staticmethod
    def _solver_out(P, R, T, H, b, cost2, info):
        return dict(R=R.reshape(P, 3, 3), T=T, H=H.reshape(P, 6, 6), b=b, cost_init=cost2[:, 0], cost=cost2[:, 1],
                    n_points=info[:, 0], n_valid=info[:, 1], iterations=info[:, 2], converged=info[:, 3], status=info[:, 4])

    # -- frame tracking against the TSDF (tslam_tsdf_track_depth / _points) ----------------------------------------
    def _track(self, name, n, args, R0, T0, huber, max_iters, min_points):
        R0 = np.ascontiguousarray(np.asarray(R0, dtype=np.float64).reshape(n, 9))
        T0 = np.ascontiguousarray(np.asarray(T0, dtype=np.float64).reshape(n, 3))
        huber = float(self.cfg.voxel_scale) if huber is None else float(huber)
        R, T = np.zeros((n, 9)), np.zeros((n, 3))
        H, b, cost2 = np.zeros((n, 36)), np.zeros((n, 6)), np.zeros((n, 2))
        info = np.zeros((n, 5), np.int64)
        head, tail = args
        capi.check(getattr(self.L, name)(self.h, *head, capi.np_ptr(R0), capi.np_ptr(T0), *tail, huber, int(max_iters), int(min_points),
                                         capi.np_ptr(R), capi.np_ptr(T), capi.np_ptr(H), capi.np_ptr(b), capi.np_ptr(cost2),
                                         capi.np_ptr(info), capi.stream_ptr()))
        return self._solver_out(n, R, T, H, b, cost2, info)

    def track_depth(self, depth, Rs, Ts, submaps=None, step=None, huber=None, max_iters=20, min_points=100):
        """Track depth frames against the map's TSDF: the pose of each frame in its submap's local frame at which the
        frame's points lie on the zero level.  depth: uint16 [n,h,w] (or [h,w]) numpy (host) or torch CUDA tensor; Rs
        [n,3,3], Ts [n,3]: initial poses (f64, the frame of integrate_depth's Rs, Ts); submaps: per frame (default 0);
        step defaults to recast_step, huber to the voxel scale.  -> dict of numpy arrays keyed like register()."""
        depth, mem, ptr, shape = capi.source(depth, np.uint16, (self.torch.uint16, self.torch.int16))
        if len(shape) == 2:
            shape = (1,) + tuple(shape)
        n, h, w = shape
        sm = np.ascontiguousarray(np.broadcast_to(np.asarray(0 if submaps is None else submaps, dtype=np.int32), (n,)))
        step = int(self.cfg.recast_step) if step is None else int(step)
        return self._track("tslam_tsdf_track_depth", n, ((ptr, mem, n, h, w, capi.np_ptr(sm)), (step,)), Rs, Ts, huber, max_iters,
                           min_points)

    def track_points(self, xyz, R, T, submap=0, huber=None, max_iters=20, min_points=100):
        """Track one point cloud xyz [n,3] (sensor frame; numpy or torch CUDA f32) against submap `submap`: points that are
        not finite or whose range lies outside [min_ray_length, max_ray_length) are dropped.  R [3,3], T [3]: initial pose
        (f64).  -> dict of numpy arrays keyed like register(), one row."""
        xyz, mem, ptr, shape = capi.source(xyz, np.float32, (self.torch.float32,), (-1, 3))
        return self._track("tslam_tsdf_track_points", 1, ((ptr, mem, shape[0], int(submap)), ()), R, T, huber, max_iters, min_points)

    # -- rendering (tslam_tsdf_render) -----------------------------------------------------
    def render(self, Rs, Ts, height, width, K9, submaps=None, z_min=None, z_max=None, step=None, normals=True, color=False):
        """Ray-cast n cameras to the zero level of the committed TSDF: Rs [n,3,3], Ts [n,3] (f64) map camera points into
        the local frame of each camera's submap (the frame of integrate_depth's Rs, Ts); K9 the pinhole (fx, fy, cx, cy
        at 0, 4, 2, 5); submaps per camera (default 0); z_min, z_max, step default to min_ray_length, max_ray_length
        and the voxel scale.  -> torch CUDA tensors (depth f32 [n,h,w] (0: no hit), status u8 [n,h,w] (0 no hit, 1 hit,
        2 hit without normal), normal f32 [n,h,w,3] or None, colour f32 [n,h,w,3] or None), NaN where status is not 1."""
        torch = self.torch
        R = np.ascontiguousarray(np.asarray(Rs, dtype=np.float64).reshape(-1, 9))
        n = R.shape[0]
        T = np.ascontiguousarray(np.asarray(Ts, dtype=np.float64).reshape(n, 3))
        K4 = np.ascontiguousarray([K9[0], K9[4], K9[2], K9[5]], dtype=np.float64)
        sm = np.ascontiguousarray(np.broadcast_to(np.asarray(0 if submaps is None else submaps, dtype=np.int32), (n,)))
        z_min = float(self.cfg.min_ray_length) if z_min is None else float(z_min)
        z_max = float(self.cfg.max_ray_length) if z_max is None else float(z_max)
        step = float(self.cfg.voxel_scale) if step is None else float(step)
        dev = capi.device()
        h, w = int(height), int(width)
        depth = torch.empty((n, h, w), dtype=torch.float32, device=dev)
        status = torch.empty((n, h, w), dtype=torch.uint8, device=dev)
        nrm = torch.empty((n, h, w, 3), dtype=torch.float32, device=dev) if normals else None
        col = torch.empty((n, h, w, 3), dtype=torch.float32, device=dev) if color else None
        capi.check(self.L.tslam_tsdf_render(self.h, n, h, w, capi.np_ptr(K4), capi.np_ptr(sm), capi.np_ptr(R), capi.np_ptr(T), z_min,
                                            z_max, step, capi.tptr(depth), capi.tptr(nrm) if normals else None,
                                            capi.tptr(col) if color else None, capi.tptr(status), capi.stream_ptr()))
        return depth, status, nrm, col

    # -- introspection --------------------------------------------------------------------
    def stats(self, clear=False):
        o = np.zeros(8, np.int64)
        capi.check(self.L.tslam_tsdf_get_stats(self.h, capi.np_ptr(o), int(clear)))
        return dict(n_px=int(o[0]), n_valid=int(o[1]), n_rays=int(o[2]), n_updates=int(o[3]), n_oob=int(o[4]),
                    n_blocks=int(o[5]), err_flags=int(o[6]), launches=int(o[7]))

    def launch_count(self):
        return int(self.L.tslam_tsdf_launch_count(self.h))

    def set_profiling(self, on=True):
        capi.check(self.L.tslam_tsdf_set_profiling(self.h, int(on)))

    def kernel_ms(self, n=512):
        """[rows,3] ms of (bucket, ray-march, commit) for the most recent profiled integrate launches."""
        o = np.zeros((n, 3), np.float32)
        k = C.c_int32(0)
        capi.check(self.L.tslam_tsdf_kernel_ms(self.h, n, capi.np_ptr(o), C.byref(k)))
        return o[:k.value]

    def kernel_ms2(self, n=512):
        """[rows,7] ms: bucket, ray march (total), commit, 0, then ray set-up + counting walk + class + scan, scattering
        walk, block march - from the kernels' own timer stamps, each stage charged from the end of the one before it
        (DESIGN.md section 5)."""
        o = np.zeros((n, 7), np.float32)
        k = C.c_int32(0)
        capi.check(self.L.tslam_tsdf_kernel_ms2(self.h, n, capi.np_ptr(o), C.byref(k)))
        return o[:k.value]

    def march_stats(self):
        """Diagnostics of the block-binned ray march since the last stats(clear=True).  n_seg_guard counts segments the
        counting and the scattering walk disagreed about; it must stay 0."""
        o = np.zeros(7, np.int64)
        capi.check(self.L.tslam_tsdf_get_march_stats2(self.h, capi.np_ptr(o)))
        return dict(n_segs=int(o[0]), n_items=int(o[1]), n_slow=int(o[2]), n_fallback=int(o[3]), n_generic=int(o[4]),
                    n_verify_bad=int(o[5]), n_seg_guard=int(o[6]))
