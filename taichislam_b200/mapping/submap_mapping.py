"""SubmapMapping - keyframe -> submap policy, PGO pose correction and local -> global fusion on top of
the H100 map classes.

Host-side orchestration only (no kernels): it mirrors the public behaviour of the reference's
taichi_slam/mapping/submap_mapping.py (same constructor, attributes, method names and wire format) so
scripts/taichislam_node.py can drive it unchanged.  Differences, all fixes of reference quirks
(SURVEY.md Appendix B): no hard-coded save path (submap_mapping.py:144-145 writes to /home/xuhao/...),
`recast_depth_to_map(R, T, ...)` works (the reference calls need_create_new_submap with the wrong arity,
:195-196), send handles are optional.

global_fusion="incremental" keeps the global map with DenseTSDF.update_fused_submaps (TSDF submaps) or
Octomap.update_fused_submaps (Octomap submaps, either occupancy model) instead of rebuilding it at every submap switch:
only submaps that were added, moved or removed are placed again, so
set_frame_poses and input_remote_submap refresh the global map (its mesh and the callback) at once.  The active
submap is left out of the global map in that mode: the reference fuses at the switch, when the active submap is
empty, and its global-mode exporters add the active submap separately.  One deviation: when a remote submap arrives
in the middle of a submap, the reference's rebuild also fuses the local active submap; the incremental mode does not.
reclaim_empty=True (incremental mode with TSDF submaps only; the Octomap has no reclaim) gives the global map's blocks
that a move or removal left empty back to the pool after each such update, so loop closures do not grow the global map.
"""
import io
import time
import warnings
import zlib

import numpy as np

from .dense_tsdf import DenseTSDF
from .taichi_octomap import Octomap


def _merged(defaults, overrides):
    out = dict(defaults)
    out.update(overrides or {})
    return out


_COMMON = dict(voxel_scale=0.05, texture_enabled=False, min_ray_length=0.3, max_ray_length=3.0,
               max_disp_particles=1024 * 1024)


# optimize_poses defaults: odometry (sigma_t m, sigma_r degrees) and the Cauchy scale c of loop edges (sqrt(chi2) units).
# Registration's H sums tens of thousands of points, so a loop that is not applied has a chi2 of 1e7 or more, and its
# Cauchy cost c^2 log1p(chi2 / c^2) caps what it can buy in odometry chi2: about 1400 at c = 10.  The loop world of the
# tests needs about 200 to close its true loop; a loop 1 m and 20 degrees off is applied at c = 30 and rejected at c = 10.
# Picked there, not measured on real data.
ODOMETRY_SIGMA = (0.05, 1.0)
LOOP_ROBUST = 10.0


class SubmapMapping:
    def __init__(self, submap_type=DenseTSDF, keyframe_step=20, sub_opts={}, global_opts={}, autosave_path=None,
                 global_fusion="rebuild", fusion_tolerance=0.0, reclaim_empty=False):
        if global_fusion not in ("rebuild", "incremental"):
            raise ValueError(f"global_fusion must be 'rebuild' or 'incremental', not {global_fusion!r}")
        if global_fusion == "incremental" and submap_type not in (DenseTSDF, Octomap):
            raise ValueError("global_fusion='incremental' needs DenseTSDF or Octomap submaps")
        if reclaim_empty and global_fusion != "incremental":
            raise ValueError("reclaim_empty needs global_fusion='incremental' (a rebuild resets the global map anyway)")
        if reclaim_empty and submap_type is not DenseTSDF:
            raise ValueError("reclaim_empty needs TSDF submaps: the Octomap has no block reclaim")
        self.global_fusion = global_fusion
        self.fusion_tolerance = float(fusion_tolerance)
        self.reclaim_empty = bool(reclaim_empty)
        self.last_fusion_stats = None  # statistics of the last incremental update
        self.last_reclaim_stats = None  # statistics of the last reclaim of the global map (reclaim_empty)
        self.submap_type = submap_type
        self.keyframe_step = keyframe_step
        self.autosave_path = autosave_path
        kind = dict(num_voxel_per_blk_axis=10) if submap_type is DenseTSDF else dict(K=2)  # submap_mapping.py:14-34
        self.sub_opts = _merged(_merged(_COMMON, dict(map_scale=[10, 10], max_submap_num=1000, **kind)), sub_opts)
        self.submaps = {}            # frame_id -> submap id
        self.frame_count = 0
        self.exporting_global = False
        self.export_TSDF_xyz = self.export_color = self.export_x = None
        self.submap_collection = submap_type(**self.sub_opts)
        self.global_map = self.create_globalmap(global_opts)
        self.first_init = True
        self.set_exporting_global()
        self.ego_motion_poses = {}
        self.pgo_poses = {}
        self.submap_odometry = {}    # submap id -> the pose odometry reported at its creation frame (optimize_poses)
        self.last_frame_id = None
        self.active_submap_frame_id = 0
        self.enable_texture = self.global_map.enable_texture
        self.post_local_to_global_callback = None
        self.map_send_handle = None
        self.traj_send_handle = None

    def create_globalmap(self, global_opts={}):  # submap_mapping.py:58-84
        kind = dict(num_voxel_per_blk_axis=10, max_submap_num=1024) if self.submap_type is DenseTSDF else dict(K=2, max_submap_num=1000)
        opts = _merged(_merged(_COMMON, dict(map_scale=[100, 100], is_global_map=True, **kind)), global_opts)
        if getattr(self, "global_fusion", "rebuild") == "incremental" and "max_submap_num" not in (global_opts or {}):
            opts["max_submap_num"] = self.sub_opts["max_submap_num"]  # the incremental fusion pairs submap tables of one size
        return self.submap_type(**opts)

    # -- intrinsics ----------------------------------------------------------------------------
    def set_dep_camera_intrinsic(self, K):
        self.submap_collection.set_dep_camera_intrinsic(K)

    def set_color_camera_intrinsic(self, K):
        self.submap_collection.set_color_camera_intrinsic(K)

    # -- which map feeds the export buffers (:92-107) -------------------------------------------
    def set_exporting_global(self):
        self.exporting_global = True
        self.set_export_submap(self.global_map)

    def set_exporting_local(self):
        self.exporting_global = False
        self.set_export_submap(self.submap_collection)

    def set_export_submap(self, src):
        self.export_color = src.export_color
        if self.submap_type is DenseTSDF:
            self.export_TSDF_xyz = src.export_TSDF_xyz
            self.num_TSDF_particles = src.num_TSDF_particles
        else:
            self.export_x = src.export_x
            self.num_export_particles = src.num_export_particles

    # -- pose graph updates (:109-124) -----------------------------------------------------------
    def set_frame_poses(self, frame_poses, from_remote=False):
        self.pgo_poses.update(frame_poses)
        used = {}
        for fid, (R, T) in frame_poses.items():
            newer = self.last_frame_id is None or fid > self.last_frame_id
            if newer and fid in self.ego_motion_poses:
                self.last_frame_id = fid
            if fid in self.submaps:
                self.global_map.set_base_pose_submap(self.submaps[fid], R, T)
                used[fid] = (R, T)
        if used and self.global_fusion == "incremental":
            self.local_to_global()  # the correction reaches the global map now, not at the next submap switch
        if not from_remote:
            self.send_traj(used)

    def align_submap(self, frame_id, reference_frame_id=None, apply=False, **opts):
        """Register the submap created on `frame_id` against the submap of `reference_frame_id` (default: the submap
        created just before it) with DenseTSDF.register_submaps, starting from their current world poses (the global
        map's base poses).  Returns the registration result plus "world_R" / "world_T": the corrected world pose
        base_ref * T of the frame's submap.  apply=True hands that pose to set_frame_poses, which moves the submap in
        the global map.  opts: band, min_weight, huber, max_iters, min_points."""
        assert self.submap_type is DenseTSDF, "submap registration needs TSDF submaps"
        if reference_frame_id is None:
            older = [f for f in self.submaps if self.submaps[f] < self.submaps[frame_id]]
            if not older:
                raise ValueError(f"frame {frame_id} has no earlier submap to align against")
            reference_frame_id = max(older, key=lambda f: self.submaps[f])
        sa, sb = self.submaps[frame_id], self.submaps[reference_frame_id]
        g = self.global_map
        Ra, Ta = g.submaps_base_R_np[sa], g.submaps_base_T_np[sa]
        Rb, Tb = g.submaps_base_R_np[sb], g.submaps_base_T_np[sb]
        pose0 = ((Rb.T @ Ra)[None], (Rb.T @ (Ta - Tb))[None])
        res = self.submap_collection.register_submaps([sa], [sb], poses=pose0, **opts)[0]
        res["world_R"] = Rb @ res["R"]
        res["world_T"] = Rb @ res["T"] + Tb
        if apply and res["status"] == 0:
            self.set_frame_poses({frame_id: (res["world_R"], res["world_T"])})
        return res

    def detect_loops(self, frame_id=None, **opts):
        """Find loop closures for the submap created on `frame_id` (default: the newest submap) among the other submaps
        with DenseTSDF.detect_loops, describing every submap at its current world pose (the global map's base poses).
        Applies nothing: the caller's pose graph decides.  Returns the accepted constraints keyed by (frame_id,
        matched frame_id): the detect_loops dict (R, T: query-local -> match-local, H, b, ...) plus "world_R" /
        "world_T", the query submap's world pose that the constraint implies (base_match * T).  opts: up and
        DenseTSDF.LOOP_DEFAULTS."""
        assert self.submap_type is DenseTSDF, "loop detection needs TSDF submaps"
        if not self.submaps:
            return {}
        frame_of = {s: f for f, s in self.submaps.items()}
        if frame_id is None:
            frame_id = frame_of[max(frame_of)]
        g = self.global_map
        poses = {s: (g.submaps_base_R_np[s], g.submaps_base_T_np[s]) for s in frame_of}
        found = self.submap_collection.detect_loops([self.submaps[frame_id]], sorted(frame_of), base_poses=poses, **opts)
        out = {}
        for c in found:
            if not c["accepted"]:
                continue
            Rb, Tb = (np.asarray(a, np.float64) for a in poses[c["match"]])
            c["world_R"], c["world_T"] = Rb @ c["R"], Rb @ c["T"] + Tb
            out[(frame_id, frame_of[c["match"]])] = c
        return out

    def optimize_poses(self, loops, odometry_sigma=ODOMETRY_SIGMA, loop_sigma=None, loop_robust=LOOP_ROBUST, apply=True,
                       **solver):
        """Optimise the submap pose graph (pose_graph.optimize) and, with apply=True, move the submaps to the result.
        Nodes: the submaps at the global map's base poses; the lowest submap id is fixed, and submaps outside its
        connected component are left out (reported in "not_moved").  Edges: odometry between consecutive local submaps,
        from the odometry poses of their creation frames, information diag(sigma_t^-2 I, sigma_r^-2 I) (odometry_sigma =
        (sigma_t m, sigma_r degrees)), no robust kernel; and one loop per entry of `loops`, a dict keyed by (frame_id,
        matched frame_id) of detect_loops dicts (accumulated across calls by the caller), i = query, j = match, Z = (R,
        T), Omega = H / loop_sigma^2 (default half a voxel), Cauchy scale loop_robust.  When both (a, b) and (b, a) are
        given, only the first in key order is used: they come from the same pair of submaps.  The defaults were picked on the
        loop world of the tests, not measured on real data.  apply=True hands the moved submaps to set_frame_poses (which
        moves them in the global map) and carries the active submap's correction C = X_new X_old^-1 into its base poses
        and pgo_poses, so the next frames and submaps continue from the corrected pose.  solver: pose_graph.DEFAULTS.
        Returns dict(poses {frame_id: (R, T)}, edges [(kind, frame_i, frame_j)], chi2, weight, rejected (loop keys whose
        final weight is below 0.1), not_moved (frame ids), converged, info (the solver's result)).  A solve that does not
        converge warns (RuntimeWarning): its poses and weights are those of the last accepted step."""
        from .. import pose_graph
        g = self.global_map
        frame_of = {s: f for f, s in self.submaps.items()}
        sids = sorted(frame_of)
        if len(sids) < 2:
            return dict(poses={}, edges=[], chi2=np.zeros(0), weight=np.zeros(0), rejected=[], not_moved=list(self.submaps),
                        info=None)
        vs = float(g.voxel_scale)
        loop_sigma = 0.5 * vs if loop_sigma is None else float(loop_sigma)
        st, sr = float(odometry_sigma[0]), np.deg2rad(float(odometry_sigma[1]))
        O_odo = np.diag([st ** -2] * 3 + [sr ** -2] * 3)
        pairs, Zs, Os, cs, kinds = [], [], [], [], []
        local = [s for s in sids if s in self.submap_odometry]
        for a, b in zip(local[:-1], local[1:]):
            (Ra, Ta), (Rb, Tb) = self.submap_odometry[a], self.submap_odometry[b]
            pairs.append((a, b)), Zs.append((Rb.T @ Ra, Rb.T @ (Ta - Tb))), Os.append(O_odo), cs.append(0.0)
            kinds.append(("odometry", frame_of[a], frame_of[b]))
        seen = set()
        for (fq, fd), c in sorted(loops.items(), key=lambda kv: kv[0]):
            if frozenset((fq, fd)) in seen:  # (a, b) and (b, a) from the same registration data: count it once
                continue
            seen.add(frozenset((fq, fd)))
            pairs.append((self.submaps[fq], self.submaps[fd]))
            Zs.append((np.asarray(c["R"], np.float64), np.asarray(c["T"], np.float64)))
            Os.append(np.asarray(c["H"], np.float64).reshape(6, 6) / loop_sigma ** 2)
            cs.append(float(loop_robust))
            kinds.append(("loop", fq, fd))
        parent = {s: s for s in sids}

        def find(a):
            while parent[a] != a:
                a = parent[a]
            return a
        for a, b in pairs:
            parent[find(a)] = find(b)
        gauge = sids[0]
        nodes = [s for s in sids if find(s) == find(gauge)]
        keep = [k for k, (a, b) in enumerate(pairs) if find(a) == find(gauge)]
        if len(nodes) < 2 or not keep:
            return dict(poses={}, edges=[], chi2=np.zeros(0), weight=np.zeros(0), rejected=[], not_moved=list(self.submaps),
                        info=None)
        at = {s: n for n, s in enumerate(nodes)}
        R0 = np.stack([np.asarray(g.submaps_base_R_np[s], np.float64) for s in nodes])
        T0 = np.stack([np.asarray(g.submaps_base_T_np[s], np.float64) for s in nodes])
        edges = dict(ij=np.array([(at[pairs[k][0]], at[pairs[k][1]]) for k in keep]), R=np.stack([Zs[k][0] for k in keep]),
                     T=np.stack([Zs[k][1] for k in keep]), omega=np.stack([Os[k] for k in keep]),
                     cauchy=np.array([cs[k] for k in keep]))
        res = pose_graph.optimize(R0, T0, np.array([s == gauge for s in nodes]), edges, **solver)
        if not res["converged"]:
            warnings.warn(f"optimize_poses: the pose graph did not converge ({res['status_name']} after "
                          f"{res['evaluations']} evaluations, largest CG residual {res['cg_residual']:.2g})",
                          RuntimeWarning, stacklevel=2)
        kinds = [kinds[k] for k in keep]
        poses = {frame_of[s]: (res["R"][at[s]], res["T"][at[s]]) for s in nodes}
        out = dict(poses=poses, edges=kinds, chi2=res["chi2"], weight=res["weight"],
                   rejected=[(fi, fj) for (kd, fi, fj), w in zip(kinds, res["weight"]) if kd == "loop" and w < 0.1],
                   not_moved=[frame_of[s] for s in sids if s not in at], converged=res["converged"], info=res)
        if apply:
            act = self.submap_collection.get_active_submap_id()
            fa = frame_of.get(act)
            moved = {f: p for f, p in poses.items() if self.submaps[f] != act and self.submaps[f] != gauge}
            if moved:
                self.set_frame_poses(moved)
            if fa is not None and act in at and act != gauge:
                Rn, Tn = poses[fa]
                Ro, To = R0[at[act]], T0[at[act]]
                Rc = Rn @ Ro.T
                Tc = Tn - Rc @ To
                g.set_base_pose_submap(act, Rn, Tn)
                self.submap_collection.set_base_pose_submap(act, Rn, Tn)
                if self.last_frame_id is None or self.last_frame_id <= fa:
                    self.pgo_poses[fa] = (Rn, Tn)
                    if fa in self.ego_motion_poses:
                        self.last_frame_id = fa
                else:
                    Rl, Tl = self.pgo_poses[self.last_frame_id]
                    self.pgo_poses[self.last_frame_id] = (Rc @ Rl, Rc @ Tl + Tc)
                self.send_traj({fa: (Rn, Tn)})  # peers learn the active submap's pose as set_frame_poses tells them the others
        return out

    def convert_by_pgo(self, frame_id, R, T):  # :162-169
        self.ego_motion_poses[frame_id] = (R, T)
        if self.last_frame_id is None:
            return R, T
        ego_R, ego_T = self.ego_motion_poses[self.last_frame_id]
        pgo_R, pgo_T = self.pgo_poses[self.last_frame_id]
        dR = pgo_R @ ego_R.T
        return dR @ R, dR @ (T - ego_T) + pgo_T

    # -- submap life cycle (:126-160) ------------------------------------------------------------
    def need_create_new_submap(self, is_keyframe, R=None, T=None):
        if self.frame_count == 0:
            return True
        return bool(is_keyframe) and self.frame_count % self.keyframe_step == 0

    def create_new_submap(self, frame_id, R, T):
        print("[SubmapMapping] Create new submap ", frame_id)
        if self.first_init:
            self.first_init = False
        else:
            self.send_submap(self.submap_collection.export_submap())
            self.submap_collection.switch_to_next_submap()
            self.submap_collection.clear_last_TSDF_exporting = True
            self.local_to_global()
        sid = self.submap_collection.get_active_submap_id()
        self.global_map.set_base_pose_submap(sid, R, T)
        self.submap_collection.set_base_pose_submap(sid, R, T)
        self.submaps[frame_id] = sid
        self.pgo_poses[frame_id] = (R, T)
        # odometry edges come from these, not from the base poses, so that a second optimisation does not anchor the first
        odo = self.ego_motion_poses.get(frame_id, (R, T))
        self.submap_odometry[sid] = (np.array(odo[0], np.float64), np.array(odo[1], np.float64))
        self.active_submap_frame_id = frame_id
        print(f"[SubmapMapping] Created new submap on frame {frame_id}, now have {sid + 1} submaps")
        if self.autosave_path and sid % 2 == 0:
            self.saveMap(self.autosave_path)
        return self.submap_collection

    def local_to_global(self):
        if self.global_fusion == "incremental":
            sc = self.submap_collection
            include = np.ones(sc.max_submap_num, bool)
            include[sc.get_active_submap_id()] = False  # the growing submap is exported separately (see above)
            st = self.global_map.update_fused_submaps(sc, include=include, tolerance=self.fusion_tolerance)
            self.last_fusion_stats = st
            if self.reclaim_empty and (st["moved"] > 0 or st["removed"] > 0):
                # blocks the old poses covered are left empty by the subtraction: give them back to the pool
                self.last_reclaim_stats = self.global_map.reclaim(empty=True)
        else:
            self.global_map.fuse_submaps(self.submap_collection)
        if self.post_local_to_global_callback is not None:
            self.post_local_to_global_callback(self.global_map)

    # -- integrate (:171-200) --------------------------------------------------------------------
    def _enter_frame(self, frame_id, is_keyframe, pose, ext):
        R, T = self.convert_by_pgo(frame_id, pose[0], pose[1])
        if self.need_create_new_submap(is_keyframe, R, T):
            self.create_new_submap(frame_id, R, T)
        R_ext, T_ext = ext
        return R @ R_ext, T + R @ T_ext

    def recast_depth_to_map_by_frame(self, frame_id, is_keyframe, pose, ext, depthmap, texture):
        Rcam, Tcam = self._enter_frame(frame_id, is_keyframe, pose, ext)
        self.submap_collection.recast_depth_to_map(Rcam, Tcam, depthmap, texture)
        self.frame_count += 1

    def recast_pcl_to_map_by_frame(self, frame_id, is_keyframe, pose, ext, pcl, rgb_array):
        Rcam, Tcam = self._enter_frame(frame_id, is_keyframe, pose, ext)
        self.submap_collection.recast_pcl_to_map(Rcam, Tcam, pcl, rgb_array)
        self.frame_count += 1

    def recast_depth_to_map(self, R, T, depthmap, texture):
        if self.need_create_new_submap(True, R, T):
            self.create_new_submap(self.frame_count, R, T)
        self.submap_collection.recast_depth_to_map(R, T, depthmap, texture)
        self.frame_count += 1

    # -- exporters (:202-224) ----------------------------------------------------------------------
    def _export_src(self):
        return self.global_map if self.exporting_global else self.submap_collection

    def cvt_TSDF_to_voxels_slice(self, z):
        self._export_src().cvt_TSDF_to_voxels_slice(z)

    def cvt_TSDF_surface_to_voxels(self):
        if not self.submaps:
            return
        if self.exporting_global:
            g = self.global_map
            g.cvt_TSDF_surface_to_voxels()
            self.submap_collection.cvt_TSDF_surface_to_voxels_to(g.num_TSDF_particles, g.max_disp_particles,
                                                                 self.export_TSDF_xyz, self.export_color)
        else:
            self.submap_collection.cvt_TSDF_surface_to_voxels()

    def cvt_occupy_to_voxels(self, level):
        if self.exporting_global:
            g = self.global_map
            g.cvt_occupy_to_voxels(level)
            self.submap_collection.cvt_occupy_voxels_to(level, g.num_export_particles, g.max_disp_particles,
                                                        self.export_x, self.export_color)
        else:
            self.submap_collection.cvt_occupy_to_voxels(level)

    # -- wire format: zlib(level 1) of np.save(dict)  (:226-261) -----------------------------------
    @staticmethod
    def _pack(obj):
        f = io.BytesIO()
        np.save(f, obj)
        return f.getbuffer(), zlib.compress(f.getbuffer(), level=1)

    @staticmethod
    def _unpack(buf):
        return np.load(io.BytesIO(zlib.decompress(buf)), allow_pickle=True).item()

    def send_submap(self, submap):
        submap["frame_id"] = self.active_submap_frame_id
        submap["pose"] = self.pgo_poses[self.active_submap_frame_id]
        t0 = time.time()
        raw, packed = self._pack(submap)
        if self.map_send_handle is not None:
            self.map_send_handle(packed)
        print(f"[SubmapMapping] Send submap with {len(raw) / 1024.0:.1f} kB, compressed {len(packed) / 1024:.1f}kB "
              f"compress cost {(time.time() - t0) * 1000:.1f}ms")

    def send_traj(self, traj):
        raw, packed = self._pack(traj)
        if self.traj_send_handle is not None:
            self.traj_send_handle(packed)

    def input_remote_submap(self, buf):
        submap = self._unpack(buf)
        idx = self.submap_collection.input_remote_submap(submap)
        self.global_map.set_base_pose_submap(idx, submap["pose"][0], submap["pose"][1])
        self.local_to_global()
        self.submaps[submap["frame_id"]] = idx

    def input_remote_traj(self, buf):
        self.set_frame_poses(self._unpack(buf), True)

    def saveMap(self, filename):
        self.global_map.saveMap(filename)

    def export_submap(self):
        return self.submap_collection.export_submap()
