"""Octomap - the reference's class surface (taichi_slam/mapping/taichi_octomap.py) on the hash grid of libtslam.so.

occupancy_model="hits" (default) is the reference's "Octomap": a per-voxel hit counter (occupy += 1 per point,
:116-119) with a threshold test (:86-88), no ray casting.  occupancy_model="logodds" is OctoMap's probabilistic model
(Hornung et al., 2013): each frame casts a ray from the sensor to every measured point, the end voxel gets a hit update
and every voxel the ray crosses a miss update, in clamped Q10 integer log-odds (DESIGN.md section 7)."""
import math
import time

import numpy as np

from ..octo_handle import OctoHandle
from .field import Field
from .mapping_common import BaseMap


def _q10(p):
    """Q10 log-odds of probability p: round_half_away(logit(p) * 1024), in f64."""
    v = math.log(p / (1.0 - p)) * 1024.0
    return int(math.copysign(math.floor(abs(v) + 0.5), v))


class Octomap(BaseMap):
    def __init__(self, map_scale=[10, 10], voxel_scale=0.05, min_occupy_thres=3, texture_enabled=False,
                 min_ray_length=0.3, max_ray_length=3.0, max_disp_particles=1000000, K=2,
                 max_submap_num=1024, disp_ceiling=10.0, disp_floor=-10.0,
                 is_global_map=False, recast_step=2, color_same_proj=True, max_blocks=0, occupancy_model="hits",
                 prob_hit=0.7, prob_miss=0.4, prob_min=0.1192, prob_max=0.971, prob_occupied=0.5):
        super(Octomap, self).__init__(voxel_scale)
        import torch
        self._torch = torch
        # :19-28
        self.Rxy = math.ceil(math.log2(map_scale[0] / voxel_scale) / math.log2(K))
        self.Rz = math.ceil(math.log2(map_scale[1] / voxel_scale) / math.log2(K))
        self.map_size_xy = map_scale[0]
        self.map_size_z = map_scale[1]
        self.K = K
        self.N = self.K ** self.Rxy
        self.Nz = self.K ** self.Rz
        ctor_voxel_scale = voxel_scale              # the kernels keep using the constructor's value (mapping_common.py:22-23)
        self.voxel_scale = self.map_size_xy / self.N  # :28
        self.max_disp_particles = max_disp_particles
        self.min_occupy_thres = min_occupy_thres
        self.max_ray_length = max_ray_length
        self.min_ray_length = min_ray_length
        self.enable_texture = texture_enabled
        self.max_submap_num = max_submap_num
        self.disp_ceiling = disp_ceiling
        self.disp_floor = disp_floor
        self.is_global_map = is_global_map
        self.recast_step = recast_step
        self.color_same_proj = color_same_proj
        self.color = None  # the colour plane lives inside the library handle (:77-79); read it with _h.gather(color=True)
        if occupancy_model not in ("hits", "logodds"):
            raise ValueError(f"occupancy_model must be 'hits' or 'logodds', not {occupancy_model!r}")
        self.occupancy_model = occupancy_model
        lo = None
        if occupancy_model == "logodds":
            self.prob_hit, self.prob_miss, self.prob_min, self.prob_max = prob_hit, prob_miss, prob_min, prob_max
            self.prob_occupied = prob_occupied
            self.l_hit, self.l_miss = _q10(prob_hit), _q10(prob_miss)
            self.l_min, self.l_max, self.l_occ = _q10(prob_min), _q10(prob_max), _q10(prob_occupied)
            lo = dict(l_hit=self.l_hit, l_miss=self.l_miss, l_min=self.l_min, l_max=self.l_max, l_occ=self.l_occ)
        self._h = OctoHandle(self.N, self.Nz, K=K, voxel_scale=ctor_voxel_scale, min_occupy_thres=min_occupy_thres,
                             min_ray_length=min_ray_length, max_ray_length=max_ray_length, recast_step=recast_step,
                             max_submaps=min(max_submap_num, 1024), max_blocks=max_blocks, texture_enabled=texture_enabled,
                             logodds=lo)
        if texture_enabled:
            self._h.set_color_intrinsics([1, 0, 0, 0, 1, 0, 0, 0, 1], color_same_proj)
        dev = torch.device("cuda", torch.cuda.current_device())
        n = max_disp_particles
        self.num_export_particles = Field(torch.zeros(1, dtype=torch.int32, device=dev))
        self.export_x = Field(torch.full((n, 3), -100000.0, dtype=torch.float32, device=dev))       # :56-60
        self.export_color = Field(torch.full((n, 3), 0.5, dtype=torch.float32, device=dev))
        self.initialize_submap_fields(self.max_submap_num)
        print(f'The map voxel is:[{self.max_submap_num}x{self.N}x{self.N}x{self.Nz}] voxel scale {self.voxel_scale:3.3f}^3 '
              f'map scale:[{self.map_size_xy}mx{self.map_size_xy}mx{self.map_size_z}m] tree depth [{self.Rxy}, {self.Rz}]')

    @property
    def occupy(self):
        """(idx int32[n,3], count uint32[n]) of the active submap - the leaf field of the reference's tree (:75-76).
        Log-odds maps: (idx, L / 1024 f32[n]) of the known voxels."""
        if self.occupancy_model == "logodds":
            idx, L = self._h.gather(self._active())
            return idx, (L.astype(np.float64) / 1024.0).astype(np.float32)
        return self._h.gather(self._active())

    def _flush(self):
        pass

    def _active(self):
        return self.active_submap_id[None]

    def _on_intrinsics(self):
        self._h.set_intrinsics(self.K_cam_dep)

    def set_color_camera_intrinsic(self, K):
        super(Octomap, self).set_color_camera_intrinsic(K)
        self._h.set_color_intrinsics(self.K_cam_color, self.color_same_proj)

    def _upload_submap_pose(self, submap_id, R, T):
        self._h.set_submap_pose(submap_id, R, T)

    # :126-132
    def recast_pcl_to_map(self, R, T, xyz_array, rgb_array, n=None):
        self.set_pose(R, T)
        xyz = np.ascontiguousarray(np.asarray(xyz_array, dtype=np.float32).reshape(-1, 3))
        rgb = None
        if self.enable_texture and rgb_array is not None and np.size(rgb_array) > 0:  # :142-143; BGR -> RGB inside (:120-124)
            rgb = np.ascontiguousarray(np.asarray(rgb_array, dtype=np.uint8).reshape(-1, 3))
        if n is not None:
            xyz = xyz[:n]
            rgb = rgb[:n] if rgb is not None else None
        self._h.integrate_points(xyz, self.input_R_np, self.input_T_np, submap=self._active(), rgb=rgb)

    def recast_depth_to_map(self, R, T, depthmap, texture):
        self.set_pose(R, T)
        tex = None
        if self.enable_texture and texture is not None and np.size(texture) > 0:  # :160-167
            tex = np.ascontiguousarray(texture, dtype=np.uint8)
        self._h.integrate_depth(np.asarray(depthmap), self.input_R_np, self.input_T_np, submap=self._active(), texture=tex)

    # :90-114
    @staticmethod
    def _lod(level):
        """`occupy.parent(level)` (:95): level 0 is the field's own node, level 1 the innermost pointer node - one cell per
        voxel either way (the node runs with disp_level = 0, taichislam_node.py:37); level L > 1 = K^(L-1)-voxel groups."""
        return max(int(level), 1)

    def cvt_occupy_to_voxels(self, level):
        level = self._lod(level)
        self.num_export_particles.t.zero_()
        self._h.extract(self._active(), level, self.export_x.t, self.num_export_particles.t,
                        self.export_color.t if self.enable_texture else None)  # :101-102

    def cvt_occupy_voxels_to(self, level, cur_num, max_disp_particles, x, color):
        level = self._lod(level)
        self._h.extract(self._active(), level, x.t[:max_disp_particles], cur_num.t,
                        color.t[:max_disp_particles] if self.enable_texture else None)  # :113-114

    def get_occupy_voxels(self, l):
        self.cvt_occupy_to_voxels(l)
        return self.export_x.to_numpy(), self.export_color.to_numpy()

    def fuse_submaps(self, submaps):  # :195-199
        t = time.time()
        self._h.fuse_from(submaps._h)
        print(f"[OctoMap] Fuse submaps {(time.time() - t) * 1000:.1f}ms, active local: {submaps.active_submap_id[None]} "
              f"remote: {submaps.remote_submap_num[None]}")

    def update_fused_submaps(self, submaps, include=None, tolerance=0.0, full=False):
        """Keep this global map equal to fuse_submaps of `submaps` (an Octomap collection of the same occupancy model),
        placing again only the submaps that were added, moved or removed since the last call (OctoHandle.fuse_update):
        bit for bit what fuse_submaps gives for the included submaps.  -> dict of the call's statistics."""
        return self._h.fuse_update(submaps._h, include=include, tolerance=tolerance, full=full)

    # planner queries (mapping_common.py:165-204; is_occupy :86-88; the reference's Octomap has no is_unobserved)
    def _query_raycast(self, pos, dir, max_dist):
        return self._h.raycast(pos, dir, max_dist, submap=self._active())

    def _query_points(self, xyz):
        f = self._h.query_flags(xyz, submap=self._active())
        # hit counter: BaseMap.is_unobserved prints "Not implemented" and returns False (:207-209), bit1 is always 0
        return (f & 1).astype(bool), (f & 2).astype(bool)

    def _query_near(self, xyz, voxel):
        if int(voxel) <= 0:  # range(-voxel, voxel) is empty (mapping_common.py:198): what TopoGraphGen asks for (:328)
            return np.zeros(len(xyz), bool)
        return self._h.query_near(xyz, int(voxel), submap=self._active())

    def _logodds_only(self, feature):
        if self.occupancy_model != "logodds":
            raise ValueError(f"{feature} needs Octomap(..., occupancy_model='logodds'): a hit counter cannot tell free space "
                             "from unknown space")

    # occupancy ESDF (log-odds maps only, DESIGN.md section 7): the interface of DenseTSDF's ESDF

    def esdf_update(self, max_dist=None):
        """Bring the ESDF of the active submap up to date (incremental when possible), truncated at max_dist (default
        max_ray_length, the TSDF ESDF's far value) -> dict(lower_sweeps, raise_sweeps (-1: full), changed, suspect)."""
        self._logodds_only("the occupancy ESDF")
        self.esdf_max_dist = float(self.max_ray_length if max_dist is None else max_dist)
        return self._h.esdf_update(self._active(), self.esdf_max_dist)

    def get_voxels_ESDF(self):
        """(idx int32[n,3], ESDF f32[n]) of the voxels known at the last esdf_update."""
        self._logodds_only("the occupancy ESDF")
        return self._h.esdf_gather(self._active())

    def esdf_query(self, xyz, update=True):
        """Interpolated ESDF and its gradient at points [n,3] of the active submap's map frame: (dist, grad, valid), torch
        CUDA tensors for a torch tensor, numpy arrays for a numpy array.  update=True first brings the field up to date
        (with the max_dist of the last esdf_update, else max_ray_length); update=False answers as of the last update."""
        self._logodds_only("the occupancy ESDF")
        if update:
            self.esdf_update(getattr(self, "esdf_max_dist", None))
        return self._h.esdf_query(xyz, submap=self._active())

    def optimize_trajectories(self, paths_or_ctrl, clearance, spacing=None, ctrl=False, update=True, **settings):
        """Smooth collision-free trajectories along paths or control points of the active submap's map frame: each
        entry of paths_or_ctrl is a path f[n,3] (e.g. plan_exploration()["path"] or a travel_path result), made into
        control points by trajectory.control_points(path, spacing) (spacing defaults to two voxels), or, with
        ctrl=True, control points themselves.  The free control points are optimised on the GPU against the ESDF
        (L-BFGS, include/tslam.h tslam_octo_esdf_trajectory) and the result checked densely.  update=True first brings the
        field up to date, as esdf_query(update=True) does.  -> a list of dicts, one per trajectory: ctrl f64[N,3], the
        cost terms, iterations, evaluations, status and the check (min_dist, min_at, invalid, close, ok).  settings:
        trajectory.DEFAULTS (dt, v_max, a_max, weights, g_tol, max_iters, memory, samples, check_samples)."""
        self._logodds_only("trajectory optimisation")
        from ..trajectory import control_points
        if update:
            self.esdf_update(getattr(self, "esdf_max_dist", None))
        sp = 2.0 * self.voxel_scale if spacing is None else float(spacing)
        qs = [np.asarray(q, np.float64) if ctrl else control_points(q, sp) for q in paths_or_ctrl]
        return self._h.esdf_trajectory(qs, clearance, submap=self._active(), **settings)

    # exploration frontiers (log-odds maps only, DESIGN.md section 7): FREE voxels next to in-volume UNKNOWN space
    def frontier_update(self, full=False):
        """Bring the frontier set of the active submap up to date (incremental when possible) -> dict(voxels, clusters,
        blocks (re-examined), full)."""
        self._logodds_only("the frontier tracker")
        return self._h.frontier_update(self._active(), full=full)

    def get_frontiers(self):
        """(idx int32[n,3], cluster int32[n]) of the frontier voxels at the last frontier_update; cluster indexes the
        arrays of get_frontier_clusters(min_voxels=1)."""
        self._logodds_only("the frontier tracker")
        return self._h.frontier_gather(self._active())

    def get_frontier_clusters(self, min_voxels=1):
        """The frontier clusters of the last frontier_update with at least min_voxels voxels, in label order, as numpy
        arrays: label, size, faces (voxel / UNKNOWN-neighbour pairs), centroid [n,3], bbox_min / bbox_max [n,3] (cell
        centres in metres of the submap frame, f64 of cell index * f32(constructor voxel_scale)) and direction [n,3]
        (the unit mean direction into unknown space, 0 where the offsets cancel)."""
        self._logodds_only("the frontier tracker")
        rec = self._h.frontier_clusters(self._active())
        rec = rec[rec[:, 1] >= int(min_voxels)]
        vs = float(np.float32(self._h.cfg.voxel_scale))
        size = rec[:, 1]
        d = rec[:, 12:15].astype(np.float64)
        norm = np.linalg.norm(d, axis=1, keepdims=True)
        return dict(label=rec[:, 0].copy(), size=size.copy(), faces=rec[:, 11].copy(),
                    centroid=rec[:, 2:5].astype(np.float64) / np.maximum(size, 1)[:, None] * vs,
                    bbox_min=rec[:, 5:8].astype(np.float64) * vs, bbox_max=rec[:, 8:11].astype(np.float64) * vs,
                    direction=np.divide(d, norm, out=np.zeros_like(d), where=norm > 0))

    def _camera(self, width, height, step, max_range):
        """the simulated depth camera of the view calls: the depth intrinsics with a width x height image; step and
        max_range default to recast_step and max_ray_length"""
        if self.K_cam_dep is None:
            raise ValueError("the view calls need the depth intrinsics: call set_dep_camera_intrinsic first")
        K = self.K_cam_dep
        return dict(fx=K[0], fy=K[4], cx=K[2], cy=K[5], width=int(width), height=int(height),
                    step=int(self.recast_step if step is None else step),
                    max_range=float(self.max_ray_length if max_range is None else max_range))

    def view_gain(self, pos, R, width, height, step=None, max_range=None, frontier=True, update=True):
        """What a depth camera would see from n candidate views of the active submap (positions pos [n,3], rotations R
        [n,3,3] in its map frame, integrate_depth's convention) -> dict(valid, unknown, frontier, frontier_per_cluster):
        the distinct UNKNOWN voxels an all-far frame would observe, and the frontier voxels in view with a FREE line of
        sight, in total and per cluster (frontier=False leaves both None).  The camera is the depth intrinsics with a
        width x height image; step and max_range default to recast_step and max_ray_length.  update=True first runs
        frontier_update(), so frontiers and classes agree.  Torch CUDA tensors in -> torch tensors out; numpy -> numpy."""
        self._logodds_only("a viewpoint gain")
        cam = self._camera(width, height, step, max_range)
        s = self._active()
        out = dict(frontier=None, frontier_per_cluster=None)
        if frontier and update:
            self.frontier_update()
        out["valid"], out["unknown"] = self._h.view_gain_unknown(pos, R, cam, submap=s)
        if frontier:
            _, out["frontier"], out["frontier_per_cluster"] = self._h.view_gain_frontier(pos, R, cam, submap=s)
        return out

    # travel cost through known free space (log-odds maps only, DESIGN.md section 7)
    def _travel_clearance(self, clearance):
        """a log-odds map, and with clearance > 0 the occupancy ESDF brought up to date for it"""
        self._logodds_only("a travel cost")
        if float(clearance) > 0.0:
            d = float(getattr(self, "esdf_max_dist", None) or self.max_ray_length)
            if np.float32(clearance) > np.float32(d):
                raise ValueError(f"clearance {clearance} exceeds the ESDF's max_dist {d}: call esdf_update(max_dist) with a "
                                 "larger max_dist first")
            self.esdf_update(d)

    def _travel_path(self, read, goal, max_len):
        """the path that read(targets [1,3], max_len) -> (cells, len) returns for `goal`, start to goal in metres, or None"""
        if isinstance(goal, self._torch.Tensor):
            goal = goal.detach().cpu().numpy()
        g = np.asarray(goal, np.float32).reshape(1, 3)
        cells, n = read(g, max_len)
        n = int(n[0])
        if n == 0:
            return None
        if n > max_len:   # the buffer was too small: once more with the reported length
            cells, n2 = read(g, n)
            assert int(n2[0]) == n
        vs = float(np.float32(self._h.cfg.voxel_scale))
        return cells[0, :n][::-1].astype(np.float64) * vs

    def travel_update(self, start, clearance=0.0, max_cost=None):
        """Travel-cost field of the active submap from `start` (metres, map frame) through known free space -> dict(
        reachable, sweeps, traversable, start_ok).  clearance > 0 keeps to cells at least that far from occupied space:
        it first runs esdf_update() with the max_dist of the last esdf_update (else max_ray_length) and raises
        ValueError when clearance exceeds it.  max_cost None: no bound below the limit 2^22 * voxel_scale."""
        self._travel_clearance(clearance)
        return self._h.travel_update(self._active(), start, clearance, max_cost)

    def travel_cost(self, xyz):
        """Travel cost of the cells of points [n,3] as of the last travel_update, +inf where unreachable: a torch CUDA
        tensor for a torch tensor, a numpy array for a numpy array."""
        self._logodds_only("a travel cost")
        return self._h.travel_query(xyz, submap=self._active())

    def travel_path(self, goal, max_len=4096):
        """The path of the last travel_update from its start to the cell of `goal` [3] as cell centres in metres (f64 of
        cell index * f32(constructor voxel_scale)), [n,3] ordered start to goal, or None when the goal is unreachable."""
        self._logodds_only("a travel cost")
        return self._travel_path(lambda g, m: self._h.travel_path(g, submap=self._active(), max_len=m), goal, max_len)

    def travel_update_multi(self, starts, clearance=0.0, max_cost=None):
        """Travel-cost fields of the active submap from each of S starts [S,3] (metres, map frame; 1 <= S <= 1024) in one
        update, row s exactly what travel_update(starts[s]) computes -> dict(sweeps, traversable, reachable int32[S],
        start_ok bool[S]).  clearance and max_cost as for travel_update (which also runs esdf_update() first)."""
        self._travel_clearance(clearance)
        return self._h.travel_multi_update(self._active(), starts, clearance, max_cost)

    def travel_cost_multi(self, xyz):
        """Travel costs [S,n] of the cells of points [n,3] from each start of the last travel_update_multi, +inf where
        unreachable; travel_cost_multi(starts) is the S x S matrix (not symmetrised: entry [s,t] and [t,s] may differ in
        the last bits).  A torch CUDA tensor for a torch tensor, a numpy array for a numpy array."""
        self._logodds_only("a travel cost")
        return self._h.travel_multi_query(xyz, submap=self._active())

    def travel_path_multi(self, source, goal, max_len=4096):
        """The path from start `source` of the last travel_update_multi to the cell of `goal` [3] as cell centres in
        metres, [n,3] ordered start to goal, or None when the goal is unreachable from that start."""
        self._logodds_only("a travel cost")
        S = getattr(self._h, "_travel_multi_S", 0)
        if not 0 <= int(source) < S:
            raise ValueError(f"source {source} is not a start of the last travel_update_multi ({S} starts)")
        src = np.array([int(source)], np.int32)
        return self._travel_path(lambda g, m: self._h.travel_multi_path(src, g, submap=self._active(), max_len=m), goal, max_len)

    def exploration_tour(self, position, goals, clearance=0.0, max_cost=None, restarts=64, seed=0):
        """The order in which to visit goals [k,3] (metres, map frame; k <= 1023) from `position` through known free
        space: travel_update_multi([position] + goals) with the clearance and max_cost of travel_update, the cost matrix
        travel_cost_multi of the same points (kept on the device), then solve_open_tour on it -> dict(
          order int64[m]: indices into goals in visiting order (the goals reachable from position);
          unreachable int64: the other goals' indices;  cost: the tour's travel cost in metres (the exact sum of its
          matrix entries, as f64);  leg_costs f32[m]: those entries;  inf_legs: legs between goals with no free path;
          converged: whether the best restart ended in a local optimum;
          path: travel_path_multi(0, goals[order[0]]), or None when no goal is reachable).
        The multi fields stay readable: travel_path_multi(s, ...) gives the path of any later leg (start s = goal s-1)."""
        self._logodds_only("an exploration tour")
        from ..tour import solve_open_tour
        torch = self._torch
        as_np = lambda a: a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
        g = np.asarray(as_np(goals), np.float32).reshape(-1, 3)
        if g.shape[0] > 1023:
            raise ValueError(f"exploration_tour takes at most 1023 goals (the start is the 1024th point), not {g.shape[0]}")
        pts = np.ascontiguousarray(np.concatenate([np.asarray(as_np(position), np.float32).reshape(1, 3), g]))
        self.travel_update_multi(pts, clearance, max_cost)
        C = self.travel_cost_multi(torch.from_numpy(pts).to(torch.device("cuda", torch.cuda.current_device())))
        r = solve_open_tour(C, restarts=restarts, seed=seed)
        tour = torch.from_numpy(np.concatenate([[0], r["order"]])).to(C.device)
        leg = C[tour[:-1], tour[1:]].cpu().numpy()
        order = r["order"] - 1
        path = self.travel_path_multi(0, g[order[0]]) if order.size else None
        return dict(order=order, unreachable=r["unreachable"] - 1, cost=r["cost"], leg_costs=leg, inf_legs=r["inf_legs"],
                    converged=bool(r["converged"][r["best"]]), path=path)

    @staticmethod
    def viewpoint_offsets(radii=(1.0, 1.5, 2.0), angles=16, heights=(0.0,)):
        """The cylinder of candidate offsets [S,3] f32 around a cluster centroid: heights outermost, then radii, then
        angles phi_j = 2 pi j / angles; each (r cos phi, r sin phi, h) computed in f64 and rounded to f32."""
        phi = 2.0 * np.pi * np.arange(int(angles), dtype=np.float64) / float(int(angles))
        rows = [(float(r) * np.cos(phi), float(r) * np.sin(phi), np.full(phi.shape, float(h))) for h in heights for r in radii]
        if not rows:
            return np.zeros((0, 3), np.float32)
        return np.concatenate([np.stack(t, 1) for t in rows]).astype(np.float32)

    def frontier_viewpoints(self, width, height, radii=(1.0, 1.5, 2.0), angles=16, heights=(0.0,), clearance=0.0, min_visible=1,
                            top_k=1, max_range=None, step=None, update=True):
        """Candidate sensor poses for every frontier cluster of the active submap (DESIGN.md section 7, "Frontier
        viewpoints"): around each cluster's centroid the offsets of viewpoint_offsets(radii, angles, heights), each a
        level camera facing the centroid, kept when its cell is traversable under travel_update's rule with `clearance`
        and it sees at least min_visible of the cluster's frontier voxels (view_gain's test, camera as there), the best
        top_k per cluster by that count (ties to the earlier sample).  update=True first runs frontier_update().  -> dict
        of numpy arrays, rows in the order of get_frontier_clusters(min_voxels=1): count int32[nc] (slots used), pos
        f32[nc,top_k,3], R f32[nc,top_k,3,3], yaw f64[nc,top_k] (atan2 of the viewing direction's y, x), visible
        int32[nc,top_k], sample int32[nc,top_k] (row of the offsets; -1 in unused slots, whose pose is zero)."""
        self._logodds_only("frontier viewpoints")
        cam = self._camera(width, height, step, max_range)
        self._travel_clearance(clearance)
        if update:
            self.frontier_update()
        off = self.viewpoint_offsets(radii, angles, heights)
        count, sample, visible, pos, R = self._h.frontier_viewpoints(off, cam, clearance, min_visible, top_k, submap=self._active())
        yaw = np.arctan2(R[..., 0, 0].astype(np.float64), R[..., 0, 2].astype(np.float64))
        return dict(count=count, pos=pos, R=R, yaw=yaw, visible=visible, sample=sample)

    def plan_exploration(self, position, width, height, radii=(1.0, 1.5, 2.0), angles=16, heights=(0.0,), clearance=0.0,
                         min_visible=1, top_k=1, max_range=None, step=None, max_cost=None, min_voxels=1, restarts=64, seed=0):
        """One exploration planning step of the active submap from `position` (metres, map frame), composed of public
        calls: frontier_viewpoints(...) (which runs frontier_update()), travel_update(position, clearance, max_cost) and
        travel_cost of every kept viewpoint; per cluster with at least min_voxels voxels, its best-ranked viewpoint with a
        finite travel cost; then exploration_tour(position, those viewpoints) -> dict(
          clusters int64[m]: cluster ordinals (rows of get_frontier_clusters(min_voxels=1)) in visiting order;
          pos f32[m,3], R f32[m,3,3], yaw f64[m], visible int32[m], sample int32[m]: their chosen viewpoints;
          unreachable int64: the qualifying clusters with no reachable kept viewpoint, ascending;
          cost, leg_costs, inf_legs, converged, path: as exploration_tour returns them).
        Raises ValueError when more than 1023 clusters have a reachable viewpoint."""
        self._logodds_only("an exploration plan")
        fv = self.frontier_viewpoints(width, height, radii, angles, heights, clearance, min_visible, top_k, max_range, step)
        size = self.get_frontier_clusters(min_voxels=1)["size"]
        self.travel_update(position, clearance, max_cost)
        nc, k = fv["sample"].shape
        kept = np.arange(k)[None, :] < fv["count"][:, None]
        cost = np.full((nc, k), np.inf, np.float32)
        if kept.any():
            cost[kept] = self.travel_cost(fv["pos"][kept])
        ok = kept & np.isfinite(cost)
        qual = size >= int(min_voxels)
        goals = np.nonzero(qual & ok.any(1))[0]
        if goals.size > 1023:
            raise ValueError(f"plan_exploration tours at most 1023 clusters, but {goals.size} have a reachable viewpoint: raise "
                             "min_voxels")
        j = np.argmax(ok, axis=1)[goals]
        tour = self.exploration_tour(position, fv["pos"][goals, j], clearance, max_cost, restarts, seed)
        c, jo = goals[tour["order"]], j[tour["order"]]
        unreachable = np.sort(np.concatenate([np.nonzero(qual & ~ok.any(1))[0], goals[tour["unreachable"]]])).astype(np.int64)
        return dict(clusters=c.astype(np.int64), pos=fv["pos"][c, jo], R=fv["R"][c, jo], yaw=fv["yaw"][c, jo],
                    visible=fv["visible"][c, jo], sample=fv["sample"][c, jo], unreachable=unreachable, cost=tour["cost"],
                    leg_costs=tour["leg_costs"], inf_legs=tour["inf_legs"], converged=tour["converged"], path=tour["path"])

    def saveMap(self, path):  # :201-202 (stub in the reference)
        pass

    def export_submap(self):  # :204-205
        return {}

    def finalization_current_submap(self):
        pass

    def reset(self):  # :210-211
        self._h.reset()
