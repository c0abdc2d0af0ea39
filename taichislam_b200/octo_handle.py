"""OctoHandle - thin Python face of the Octomap part of the C ABI (include/tslam.h)."""
import ctypes as C

import numpy as np

from . import _capi as capi


class OctoHandle:
    def __init__(self, N, Nz, K=2, voxel_scale=0.05, min_occupy_thres=3, min_ray_length=0.3, max_ray_length=3.0,
                 recast_step=2, Kcam=None, max_submaps=1024, max_blocks=0, max_image_pixels=0, max_points=0,
                 texture_enabled=False, logodds=None):
        """logodds: None (hit counter) or a dict l_hit, l_miss, l_min, l_max, l_occ of Q10 log-odds (log-odds occupancy,
        fixed for the map's life)."""
        capi.require_gpu()
        import torch
        self.torch = torch
        L = capi.load()
        Kc = Kcam if Kcam is not None else [1, 0, 0, 0, 1, 0, 0, 0, 1]
        self.cfg = capi.OctoConfig(voxel_scale, N, Nz, K, max_ray_length, min_ray_length, recast_step, Kc[0], Kc[4], Kc[2],
                                   Kc[5], min_occupy_thres, max_submaps, max_blocks, max_image_pixels, max_points,
                                   int(bool(texture_enabled)))
        self.texture_enabled = bool(texture_enabled)
        torch.cuda.init()
        torch.cuda.current_stream()
        h = C.c_void_p()
        self.logodds = dict(logodds) if logodds is not None else None
        if self.logodds is None:
            capi.check(L.tslam_octo_create(C.byref(self.cfg), C.byref(h)))
        else:
            lp = capi.OctoLogodds(*(int(self.logodds[k]) for k in ("l_hit", "l_miss", "l_min", "l_max", "l_occ")))
            capi.check(L.tslam_octo_create_logodds(C.byref(self.cfg), C.byref(lp), C.byref(h)))
        self.h, self.L = h, L
        self.N, self.Nz, self.K = N, Nz, K

    def close(self):
        if getattr(self, "h", None):
            self.L.tslam_octo_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        capi.check(self.L.tslam_octo_reset(self.h, capi.stream_ptr()))

    def set_submap_pose(self, s, R, T):
        R, T = capi.f32c(R).reshape(9), capi.f32c(T).reshape(3)
        capi.check(self.L.tslam_octo_set_submap_pose(self.h, int(s), capi.np_ptr(R), capi.np_ptr(T)))

    def set_intrinsics(self, K9):
        capi.check(self.L.tslam_octo_set_intrinsics(self.h, K9[0], K9[4], K9[2], K9[5]))

    def set_color_intrinsics(self, K9, color_same_proj=False):
        capi.check(self.L.tslam_octo_set_color_intrinsics(self.h, K9[0], K9[4], K9[2], K9[5], int(bool(color_same_proj))))

    def integrate_points(self, xyz, R, T, submap=0, rgb=None):
        xyz, mem, ptr, shape = capi.source(xyz, np.float32, (self.torch.float32,), (-1, 3))
        n = shape[0]
        R, T = capi.f32c(R).reshape(9), capi.f32c(T).reshape(3)
        rgb, cptr = capi.companion(rgb, mem)
        if rgb is not None:
            assert tuple(rgb.shape) == (n, 3)
        capi.check(self.L.tslam_octo_integrate_points_rgb(self.h, ptr, cptr, mem, n, capi.np_ptr(R), capi.np_ptr(T), int(submap),
                                                          capi.stream_ptr()))
        if mem == capi.MEM_HOST:
            self.torch.cuda.current_stream().synchronize()  # pageable host source must outlive the copy

    def integrate_depth(self, depth, R, T, submap=0, texture=None):
        depth, mem, ptr, (h, w) = capi.source(depth, np.uint16, (self.torch.uint16, self.torch.int16))
        R, T = capi.f32c(R).reshape(9), capi.f32c(T).reshape(3)
        texture, tptr = capi.companion(texture, mem)
        th, tw = (0, 0) if texture is None else (int(texture.shape[0]), int(texture.shape[1]))
        capi.check(self.L.tslam_octo_integrate_depth_tex(self.h, ptr, tptr, mem, h, w, th, tw, capi.np_ptr(R), capi.np_ptr(T),
                                                         int(submap), capi.stream_ptr()))
        if mem == capi.MEM_HOST:
            self.torch.cuda.current_stream().synchronize()

    def gather_device(self, submap=0, cap=None, color=False):
        torch = self.torch
        alloc = [((3,), torch.int32), ((), torch.int32)] + ([((3,), torch.float32)] if color else [])
        return capi.count_fill(lambda cap, n, idx, cnt, col=None: self.L.tslam_octo_gather2(
            self.h, int(submap), cap, idx, cnt, col, n, capi.stream_ptr()), *alloc, cap=cap)

    def gather_logodds_device(self, submap=0, color=False):
        """(idx int32[n,3], L int32[n][, color f32[n,3]]) of the known voxels of a log-odds map, on the device."""
        torch = self.torch
        alloc = [((3,), torch.int32), ((), torch.int32)] + ([((3,), torch.float32)] if color else [])
        return capi.count_fill(lambda cap, n, idx, lo, col=None: self.L.tslam_octo_gather_logodds(
            self.h, int(submap), cap, idx, lo, col, n, capi.stream_ptr()), *alloc)

    def gather(self, submap=0, color=False):
        """Hit counter: (idx, count uint32[, color]).  Log-odds map: (idx, L int32[, color]) of the known voxels."""
        if self.logodds is not None:
            r = self.gather_logodds_device(submap, color=color)
            return tuple(t.cpu().numpy() for t in r)
        r = self.gather_device(submap, color=color)
        out = (r[0].cpu().numpy(), r[1].cpu().numpy().view(np.uint32))
        return out + (r[2].cpu().numpy(),) if color else out

    def extract(self, submap, level, xyz, count, rgb=None):
        capi.check(self.L.tslam_octo_extract2(self.h, int(submap), int(level), xyz.shape[0], capi.tptr(xyz),
                                              capi.tptr(rgb) if rgb is not None else None, capi.tptr(count), capi.stream_ptr()))

    def export(self, level=1, submap=0, cap=1 << 22, color=False):
        f32 = self.torch.float32
        alloc = [((3,), f32)] + ([((3,), f32, True)] if color else [])  # rgb stays 0 where the map has no colour
        return capi.extract(lambda cnt, xyz, rgb=None: self.extract(submap, level, xyz, cnt, rgb), cap, *alloc)

    def query_flags(self, xyz, submap=0):
        """uint8 flags per point: bit0 occupied, bit1 unknown (log-odds maps; always 0 for a hit counter)."""
        return capi.query_flags(self.L.tslam_octo_query_points, self.h, xyz, submap)

    def query_points(self, xyz, submap=0):
        """occupied per point; a log-odds map returns (occupied, unknown)."""
        f = self.query_flags(xyz, submap)
        if self.logodds is not None:
            return (f & 1).astype(bool), (f & 2).astype(bool)
        return f.astype(bool)

    def query_near(self, xyz, voxel, submap=0):
        """is_near_pos_occupy: any occupied cell in [-voxel, voxel)^3 around each point's cell."""
        return capi.near_occupy(self.L.tslam_octo_query_near_occupy, self.h, xyz, voxel, submap)

    def stats(self, clear=False):
        """Log-odds counters since the last clear: rays cast, in-volume miss-cell visits, hit voxels, voxels updated."""
        out = (C.c_int64 * 4)()
        capi.check(self.L.tslam_octo_get_stats(self.h, out, int(bool(clear))))
        return dict(zip(("rays", "miss_visits", "hit_voxels", "updated_voxels"), (int(v) for v in out)))

    # -- occupancy ESDF of a log-odds map (tslam_octo_esdf_*, DESIGN.md section 7) ------------------------------------
    def esdf_update(self, submap=0, max_dist=1.0, full=False):
        """Bring the ESDF of `submap` up to date, truncated at max_dist (incremental unless full, the last update was for
        another submap or max_dist, or the map was reset or fused) -> dict(lower_sweeps, raise_sweeps (-1: full
        recompute), changed, suspect)."""
        st = np.zeros(4, np.int32)
        capi.check(self.L.tslam_octo_esdf_update(self.h, int(submap), float(max_dist), 1 if full else 0, capi.np_ptr(st),
                                                 capi.stream_ptr()))
        return dict(lower_sweeps=int(st[0]), raise_sweeps=int(st[1]), changed=int(st[2]), suspect=int(st[3]))

    def esdf_gather(self, submap=0, as_torch=False):
        """(idx int32[n,3], ESDF f32[n]) of the voxels known at the last esdf_update: numpy arrays, or torch CUDA tensors
        with as_torch."""
        torch = self.torch
        return capi.results(as_torch, *capi.count_fill(lambda cap, n, idx, e: self.L.tslam_octo_esdf_gather(
            self.h, int(submap), cap, idx, e, n, capi.stream_ptr()), ((3,), torch.int32), ((), torch.float32)))

    def esdf_query(self, xyz, submap=0):
        """Trilinear ESDF and its exact gradient at points [n,3] of the submap's map frame, as of the last esdf_update:
        (dist f32[n], grad f32[n,3], valid bool[n]); dist and grad are NaN where valid is False.  A torch CUDA tensor in
        -> torch CUDA tensors out, without a host synchronisation; a numpy array in -> numpy arrays out."""
        return capi.esdf_query(self.L.tslam_octo_esdf_query, self.h, xyz, submap)

    def esdf_trajectory(self, ctrls, clearance, submap=0, **settings):
        """Optimise uniform cubic B-splines (control points f[N,3] each, the submap's map frame) against the occupancy
        ESDF of `submap` as of its last esdf_update (tslam_octo_esdf_trajectory) -> a list of dicts (trajectory.solve).
        settings: trajectory.DEFAULTS."""
        from . import trajectory
        return trajectory.solve(self.L.tslam_octo_esdf_trajectory, self.h, submap, ctrls, clearance, **settings)

    # -- frontiers of a log-odds map (tslam_octo_frontier_*, DESIGN.md section 7) --------------------------------------
    def frontier_update(self, submap=0, full=False):
        """Bring the frontier set of `submap` up to date (incremental unless full, the last update was for another submap,
        or the map was reset or fused) -> dict(voxels, clusters, blocks (re-examined), full (bool))."""
        st = np.zeros(4, np.int32)
        capi.check(self.L.tslam_octo_frontier_update(self.h, int(submap), 1 if full else 0, capi.np_ptr(st), capi.stream_ptr()))
        return dict(voxels=int(st[0]), clusters=int(st[1]), blocks=int(st[2]), full=bool(st[3]))

    def frontier_gather(self, submap=0, as_torch=False):
        """(idx int32[n,3], cluster int32[n]) of the frontier voxels of the last frontier_update; cluster is the ordinal in
        frontier_clusters.  numpy arrays, or torch CUDA tensors with as_torch."""
        torch = self.torch
        return capi.results(as_torch, *capi.count_fill(lambda cap, n, idx, cl: self.L.tslam_octo_frontier_gather(
            self.h, int(submap), cap, idx, cl, n, capi.stream_ptr()), ((3,), torch.int32), ((), torch.int32)))

    def frontier_clusters(self, submap=0, as_torch=False):
        """int64[n,16] cluster records of the last frontier_update in label order (label, voxels, sum i / j / k, min i / j
        / k, max i / j / k, faces, sum of the unit offsets towards UNKNOWN x / y / z, 0)."""
        return capi.results(as_torch, *capi.count_fill(self._clusters_call(submap), ((16,), self.torch.int64)))

    def _clusters_call(self, submap):
        return lambda cap, n, rec=None: self.L.tslam_octo_frontier_clusters(self.h, int(submap), cap, rec, n, capi.stream_ptr())

    # -- viewpoint gain of a log-odds map (tslam_octo_view_gain_*, DESIGN.md section 7) ------------------------------
    @staticmethod
    def view_camera(cam):
        """tslam_view_camera_t from a mapping with fx, fy, cx, cy, width, height, step, max_range."""
        return capi.ViewCamera(float(cam["fx"]), float(cam["fy"]), float(cam["cx"]), float(cam["cy"]), int(cam["width"]),
                               int(cam["height"]), int(cam["step"]), float(cam["max_range"]))

    def _views(self, pos, R):
        """(as_torch, pos f32 [n,3], R f32 [n,9]) as contiguous CUDA tensors"""
        p, r = capi.to_device(pos, (-1, 3)), capi.to_device(R, (-1, 9))
        assert p.shape[0] == r.shape[0], "pos [n,3] and R [n,3,3] need the same n"
        return isinstance(pos, self.torch.Tensor), p, r

    def view_gain_unknown(self, pos, R, cam, submap=0):
        """Unknown gain of n views (positions pos [n,3], rotations R [n,3,3], camera `cam` as in view_camera) -> (valid
        bool[n], gain int64[n]): the distinct UNKNOWN voxels an all-far depth frame from each view would see up to the
        first occupied voxel of each ray.  Torch CUDA tensors in -> torch tensors out without a host synchronisation (a
        walk outside its view's window is then reported by the next sync()); numpy in -> numpy out."""
        torch = self.torch
        as_torch, p, r = self._views(pos, R)
        n = p.shape[0]
        valid = torch.empty(n, dtype=torch.uint8, device=p.device)
        gain = torch.empty(n, dtype=torch.int64, device=p.device)
        c = self.view_camera(cam)
        capi.check(self.L.tslam_octo_view_gain_unknown(self.h, int(submap), n, capi.tptr(p), capi.tptr(r), C.byref(c), capi.tptr(valid),
                                                       capi.tptr(gain), capi.stream_ptr()))
        if not as_torch:
            self.sync()
        return capi.results(as_torch, valid.view(torch.bool), gain)

    def view_gain_frontier(self, pos, R, cam, submap=0):
        """Frontier gain of n views against the frontier set of the last frontier_update -> (valid bool[n], total int32[n],
        per_cluster int32[n, clusters]): the frontier voxels in each view's frustum whose line of sight crosses FREE voxels
        only, per cluster ordinal (the rows of frontier_clusters).  Torch in -> torch out, numpy in -> numpy out."""
        torch = self.torch
        as_torch, p, r = self._views(pos, R)
        n = p.shape[0]
        nc = capi.count_fill(self._clusters_call(submap))
        valid = torch.empty(n, dtype=torch.uint8, device=p.device)
        total = torch.empty(n, dtype=torch.int32, device=p.device)
        per = torch.empty((n, nc), dtype=torch.int32, device=p.device)
        c = self.view_camera(cam)
        capi.check(self.L.tslam_octo_view_gain_frontier(self.h, int(submap), n, capi.tptr(p), capi.tptr(r), C.byref(c), nc,
                                                        capi.tptr(valid), capi.tptr(total), capi.tptr(per) if nc else None,
                                                        capi.stream_ptr()))
        return capi.results(as_torch, valid.view(torch.bool), total, per)

    def frontier_viewpoints(self, offsets, cam, clearance=0.0, min_visible=1, top_k=1, submap=0):
        """The best top_k candidate views per frontier cluster of the last frontier_update (DESIGN.md section 7, "Frontier
        viewpoints"): candidate s of cluster c sits at the cluster's f32 centroid plus offsets[s] (metres, [S,3],
        1 <= S <= 1024), level and facing the centroid; it is kept when its cell is traversable under travel_update's
        rule with `clearance` (> 0 reads the last esdf_update) and it sees at least min_visible of the cluster's frontier
        voxels -> (count int32[nc], sample int32[nc,top_k], visible int32[nc,top_k], pos f32[nc,top_k,3],
        R f32[nc,top_k,3,3]), rows in cluster ordinal order, slots at and beyond count[c] hold sample -1 and zeros.
        Torch in -> torch out without a host synchronisation; numpy in -> numpy out."""
        torch = self.torch
        off = capi.to_device(offsets, (-1, 3))
        S, k = off.shape[0], int(top_k)
        nc = capi.count_fill(self._clusters_call(submap))
        dev = off.device
        count = torch.empty(nc, dtype=torch.int32, device=dev)
        sample = torch.empty((nc, max(k, 0)), dtype=torch.int32, device=dev)
        visible = torch.empty((nc, max(k, 0)), dtype=torch.int32, device=dev)
        pos = torch.empty((nc, max(k, 0), 3), dtype=torch.float32, device=dev)
        R = torch.empty((nc, max(k, 0), 3, 3), dtype=torch.float32, device=dev)
        c = self.view_camera(cam)
        ptr = (lambda t: capi.tptr(t) if nc else None)
        capi.check(self.L.tslam_octo_frontier_viewpoints(self.h, int(submap), C.byref(c), S, capi.tptr(off), float(clearance),
                                                         int(min_visible), k, nc, ptr(count), ptr(sample), ptr(visible), ptr(pos),
                                                         ptr(R), capi.stream_ptr()))
        return capi.results(isinstance(offsets, torch.Tensor), count, sample, visible, pos, R)

    # -- travel cost on a log-odds map (tslam_octo_travel_*, DESIGN.md section 7) --------------------------------------
    def travel_limit(self):
        """The largest max_cost a travel update accepts: 2^22 * f32(voxel_scale)."""
        return float(np.ldexp(np.float32(self.cfg.voxel_scale), 22))

    def travel_update(self, submap, start, clearance=0.0, max_cost=None):
        """Travel-cost field of `submap` from `start` (metres, submap frame) through known free space, with `clearance`
        (> 0: cells whose occupancy ESDF at the last esdf_update is >= clearance) and max_cost (None: the limit
        2^22 * voxel_scale) -> dict(reachable, sweeps, traversable, start_ok (bool))."""
        p = capi.f32c(start).reshape(3)
        st = np.zeros(4, np.int32)
        mc = self.travel_limit() if max_cost is None else float(max_cost)
        capi.check(self.L.tslam_octo_travel_update(self.h, int(submap), capi.np_ptr(p), float(clearance), mc, capi.np_ptr(st),
                                                   capi.stream_ptr()))
        return dict(reachable=int(st[0]), sweeps=int(st[1]), traversable=int(st[2]), start_ok=bool(st[3]))

    def travel_gather(self, submap=0, as_torch=False):
        """(idx int32[n,3], cost f32[n]) of the cells reachable at the last travel_update: numpy arrays, or torch CUDA
        tensors with as_torch."""
        torch = self.torch
        return capi.results(as_torch, *capi.count_fill(lambda cap, n, idx, g: self.L.tslam_octo_travel_gather(
            self.h, int(submap), cap, idx, g, n, capi.stream_ptr()), ((3,), torch.int32), ((), torch.float32)))

    def travel_query(self, xyz, submap=0):
        """Travel cost f32[n] of the cells of points [n,3] as of the last travel_update (+inf where unreachable).  A torch
        CUDA tensor in -> a torch CUDA tensor out, without a host synchronisation; a numpy array in -> a numpy array out."""
        torch = self.torch
        x = capi.to_device(xyz, (-1, 3))
        n = x.shape[0]
        cost = torch.empty(n, dtype=torch.float32, device=x.device)
        capi.check(self.L.tslam_octo_travel_query(self.h, int(submap), n, capi.tptr(x), capi.tptr(cost), capi.stream_ptr()))
        return capi.results(isinstance(xyz, torch.Tensor), cost)

    def travel_path(self, xyz, submap=0, max_len=4096):
        """Paths from the cells of targets [n,3] back to the start of the last travel_update -> (cells int32[n,max_len,3]
        target -> start, len int32[n]: the full cell count, 0 when unreachable; rows beyond min(len, max_len) are
        undefined).  Torch in -> torch out without a host synchronisation; numpy in -> numpy out."""
        torch = self.torch
        as_torch, x = isinstance(xyz, torch.Tensor), capi.to_device(xyz, (-1, 3))
        n = x.shape[0]
        cells = torch.empty((n, int(max_len), 3), dtype=torch.int32, device=x.device)
        ln = torch.empty(n, dtype=torch.int32, device=x.device)
        capi.check(self.L.tslam_octo_travel_path(self.h, int(submap), n, capi.tptr(x), int(max_len), capi.tptr(cells), capi.tptr(ln),
                                                 capi.stream_ptr()))
        if not as_torch:
            self.sync()
        return capi.results(as_torch, cells, ln)

    def travel_multi_update(self, submap, starts, clearance=0.0, max_cost=None):
        """Travel-cost fields of `submap` from each of S starts [S,3] (metres, submap frame; 1 <= S <= 1024) in one update,
        row s exactly the field travel_update(starts[s]) would compute; clearance and max_cost as there -> dict(sweeps,
        traversable, reachable int32[S], start_ok bool[S])."""
        p = capi.f32c(starts).reshape(-1, 3)
        S = p.shape[0]
        st = np.zeros(2, np.int32)
        reach = np.zeros(max(S, 1), np.int32)
        ok = np.zeros(max(S, 1), np.uint8)
        mc = self.travel_limit() if max_cost is None else float(max_cost)
        capi.check(self.L.tslam_octo_travel_multi_update(self.h, int(submap), S, capi.np_ptr(p), float(clearance), mc, capi.np_ptr(st),
                                                         capi.np_ptr(reach), capi.np_ptr(ok), capi.stream_ptr()))
        self._travel_multi_S = S
        return dict(sweeps=int(st[0]), traversable=int(st[1]), reachable=reach[:S].copy(), start_ok=ok[:S].astype(bool))

    def travel_multi_query(self, xyz, submap=0):
        """Travel costs f32[S,n] of the cells of points [n,3] from each start of the last travel_multi_update (+inf where
        unreachable); the starts themselves give the S x S matrix.  Torch in -> torch out without a host
        synchronisation; numpy in -> numpy out."""
        torch = self.torch
        x = capi.to_device(xyz, (-1, 3))
        n = x.shape[0]
        cost = torch.empty((getattr(self, "_travel_multi_S", 0), n), dtype=torch.float32, device=x.device)
        capi.check(self.L.tslam_octo_travel_multi_query(self.h, int(submap), n, capi.tptr(x), capi.tptr(cost), capi.stream_ptr()))
        return capi.results(isinstance(xyz, torch.Tensor), cost)

    def travel_multi_path(self, source, xyz, submap=0, max_len=4096):
        """Paths of pairs (source[q], xyz[q]) from the cell of the target back to starts[source[q]] of the last
        travel_multi_update -> (cells int32[n,max_len,3], len int32[n]) as travel_path returns them.  A source outside
        [0, S) gets len 0 and the next sync() raises.  Torch in -> torch out without a host synchronisation; numpy in ->
        numpy out."""
        torch = self.torch
        x, src = capi.to_device(xyz, (-1, 3)), capi.to_device(source, (-1,), "int32")
        n = x.shape[0]
        assert src.shape[0] == n, "source [n] and xyz [n,3] need the same n"
        cells = torch.empty((n, int(max_len), 3), dtype=torch.int32, device=x.device)
        ln = torch.empty(n, dtype=torch.int32, device=x.device)
        capi.check(self.L.tslam_octo_travel_multi_path(self.h, int(submap), n, capi.tptr(src), capi.tptr(x), int(max_len), capi.tptr(cells),
                                                       capi.tptr(ln), capi.stream_ptr()))
        return capi.results(isinstance(xyz, torch.Tensor), cells, ln)

    def raycast(self, pos, direction, max_dist, submap=0):
        return capi.raycast(self.L.tslam_octo_raycast, self.h, pos, direction, max_dist, submap)

    def fuse_from(self, src):
        capi.check(self.L.tslam_octo_fuse(self.h, src.h, capi.stream_ptr()))

    def fuse_update(self, src, include=None, tolerance=0.0, full=False):
        """Incremental fusion of the submaps of `src` (an OctoHandle of the same occupancy model) into this global map
        (tslam_octo_fuse_update): afterwards this map is bit for bit fuse_from of the included submaps at their fused
        poses.  include: None (all) or bools / 0-1 per submap (up to max_submaps); tolerance: how far (metres,
        translation + angle x radius) a fused submap may move before it is placed again; full=True forces a rebuild.
        -> dict of the call's statistics (TsdfHandle.fuse_update's keys; voxels_skipped counts recoloured voxels)."""
        return capi.fuse_update(self.L.tslam_octo_fuse_update, self, src, include, tolerance, full)

    def sync(self):
        capi.check(self.L.tslam_octo_sync(self.h, capi.stream_ptr()))

    def launch_count(self):
        return int(self.L.tslam_octo_launch_count(self.h))
