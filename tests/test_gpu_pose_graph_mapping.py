"""SubmapMapping.optimize_poses on the loop world (tests/loop_world.py): detect loops for every submap, optimise, and
check every room-A submap against the truth and the reference optimum of the same graph, a fabricated false loop,
the global map against a rebuild at the optimised poses, the carried correction and what peers are sent; and an
Octomap flow with a caller-given loop."""
import numpy as np
import pytest

import loop_world as lw
import pose_graph_reference as P
from submap_register_reference import pose_error
from taichislam_b200 import synthetic as syn
from util import as_dict_rows

pytestmark = pytest.mark.gpu
VS = 0.05


def run_loop_world():
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    sub = dict(map_scale=[12.8, 12.8], voxel_scale=VS, num_voxel_per_blk_axis=10, max_ray_length=6.0, max_submap_num=16,
               max_disp_particles=1 << 16)
    glo = dict(sub, map_scale=[25.6, 12.8])
    sm = SubmapMapping(DenseTSDF, sub_opts=sub, global_opts=glo, keyframe_step=lw.FRAMES, global_fusion="incremental")
    sm.set_dep_camera_intrinsic(syn.K_DEPTH)
    fid = 0
    for s in range(lw.N_LOOP):
        for f in range(lw.FRAMES):
            sm.recast_depth_to_map_by_frame(fid, True, lw.odometry_pose(s, f), (np.eye(3), np.zeros(3)), lw.render(s, f),
                                            np.array([]))
            fid += 1
    return sm, fid


def global_rows(g):
    return as_dict_rows(*g._h.gather(0))


def rebuild_rows(sm):
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    g = sm.global_map
    opts = dict(map_scale=[25.6, 12.8], voxel_scale=VS, num_voxel_per_blk_axis=10, max_ray_length=6.0, max_submap_num=16,
                max_disp_particles=1 << 16, is_global_map=True)
    reb = DenseTSDF(**opts)
    active = sm.submap_collection.get_active_submap_id()
    for s in range(16):
        T = g.submaps_base_T_np[s] + (np.array([1e4, 0.0, 0.0]) if s == active else 0.0)
        reb.set_base_pose_submap(s, g.submaps_base_R_np[s], T)
    reb.fuse_submaps(sm.submap_collection)
    return as_dict_rows(*reb._h.gather(0))


def assert_map_equal(sm):
    ni, nt, nw, _ = global_rows(sm.global_map)
    oi, ot, ow, _ = rebuild_rows(sm)
    assert np.array_equal(ni, oi)
    fin = np.isfinite(ot)
    heavy = fin & (ow >= 1e-3)
    assert heavy.mean() > 0.9 and np.abs(nt[heavy] - ot[heavy]).max() <= 1e-4
    assert np.all(np.abs(nw[fin] - ow[fin]) <= 1e-4 * np.maximum(1.0, ow[fin]))


def reference_graph(sm, loops, sigma_t=0.05, sigma_r_deg=1.0, robust=10.0):
    """The graph optimize_poses documents, built independently: nodes = the submaps at the global base poses (lowest id
    fixed), odometry edges between consecutive submaps from their creation-frame odometry, one loop edge per unordered
    pair (first key in order), Omega = H / (half a voxel)^2."""
    sids = sorted(sm.submaps.values())
    g = sm.global_map
    R0 = np.stack([g.submaps_base_R_np[s] for s in sids]).astype(np.float64)
    T0 = np.stack([g.submaps_base_T_np[s] for s in sids]).astype(np.float64)
    at = {s: n for n, s in enumerate(sids)}
    ij, ZR, ZT, om, c = [], [], [], [], []
    for a, b in zip(sids[:-1], sids[1:]):
        Ra, Ta = lw.odometry_pose(a, 0)
        Rb, Tb = lw.odometry_pose(b, 0)
        ij.append((at[a], at[b])), ZR.append(Rb.T @ Ra), ZT.append(Rb.T @ (Ta - Tb))
        om.append(P.information(sigma_t, np.deg2rad(sigma_r_deg))), c.append(0.0)
    seen = set()
    for (fq, fd), lp in sorted(loops.items(), key=lambda kv: kv[0]):
        if frozenset((fq, fd)) in seen:
            continue
        seen.add(frozenset((fq, fd)))
        ij.append((at[sm.submaps[fq]], at[sm.submaps[fd]])), ZR.append(lp["R"]), ZT.append(lp["T"])
        om.append(np.asarray(lp["H"]).reshape(6, 6) / (0.5 * VS) ** 2), c.append(robust)
    fixed = np.zeros(len(sids), bool)
    fixed[0] = True
    return R0, T0, fixed, dict(ij=np.array(ij), R=np.stack(ZR), T=np.stack(ZT), omega=np.stack(om), cauchy=np.array(c))


# The loop world's detections close one loop, between the first and the last submap (registration accepts no other
# pair: submaps across the odometry jump overlap too little).  One loop cannot tell which odometry edge holds the jump,
# so the optimum spreads the correction along the chain as the odometry information dictates: the closed submap ends at
# its true pose, the ones in between do not.  Their bounds below pin what that optimum is (measured 0.70 m / 11.8 deg
# at most), and the poses are checked against the reference optimum of the same graph.
INTERMEDIATE_BOUND = (0.75, 12.5)


@pytest.mark.parametrize("false_loop", [False, True])
def test_loop_world_optimise_and_move_the_global_map(false_loop):
    sm, next_fid = run_loop_world()
    loops = {}
    for f in sorted(sm.submaps):
        loops.update(sm.detect_loops(f, min_gap=2))
    assert sorted(loops) == [(0, lw.FRAMES * (lw.N_LOOP - 1)), (lw.FRAMES * (lw.N_LOOP - 1), 0)], sorted(loops)
    if false_loop:
        # submaps 1 and 4 do not overlap (registration finds no valid point between them), so the fabricated loop
        # carries the real H of the detected loop: registration-scale information, 1 m and 20 degrees off the truth
        Rt, Tt = lw.relative(1, 4)
        Rb, Tb = P.update(Rt, Tt, np.r_[1.0, 0.0, 0.0, 0.0, np.deg2rad(20.0), 0.0])
        loops[(lw.FRAMES, 4 * lw.FRAMES)] = dict(R=Rb, T=Tb, H=loops[(lw.FRAMES * (lw.N_LOOP - 1), 0)]["H"])
    act = sm.submap_collection.get_active_submap_id()
    fa = sm.active_submap_frame_id
    X_old = (sm.global_map.submaps_base_R_np[act].copy(), sm.global_map.submaps_base_T_np[act].copy())
    R0, T0, fixed, edges = reference_graph(sm, loops)
    ref = P.solve_edges(R0, T0, fixed, edges, eps_t=1e-8, eps_r=1e-10)
    # at these tolerances F may stop decreasing in f64 before a step is small enough (status "no progress"): both
    # solvers are then at the optimum to rounding, which is what is compared
    tight = sm.optimize_poses(loops, apply=False, eps_t=1e-8, eps_r=1e-10)
    assert tight["info"]["status_name"] in ("converged", "no progress")
    frames = sorted(tight["poses"], key=lambda f: sm.submaps[f])
    Rg = np.stack([tight["poses"][f][0] for f in frames])
    Tg = np.stack([tight["poses"][f][1] for f in frames])
    assert np.abs(Tg - ref["T"]).max() <= 1e-6 and np.abs(Rg - ref["R"]).max() <= 1e-7
    out = sm.optimize_poses(loops)  # the defaults, applied
    assert out["converged"] and out["info"]["F"] < out["info"]["F0"]
    assert len(out["edges"]) == len(edges["ij"])  # (a, b) and (b, a) counted once
    Tu = np.stack([out["poses"][f][1] for f in frames])
    assert np.abs(Tu - Tg).max() <= 1e-5
    err = np.array([pose_error(*out["poses"][f], *lw.true_pose(sm.submaps[f], 0)) for f in frames])
    print("errors", err.tolist(), "weights", out["weight"].tolist(), "rejected", out["rejected"])
    assert err[0, 0] <= 1e-9 and err[0, 1] <= 1e-5  # the gauge (drift-free) stays
    assert err[-1, 0] <= VS and err[-1, 1] <= 0.5
    assert err[1:-1, 0].max() <= INTERMEDIATE_BOUND[0] and err[1:-1, 1].max() <= INTERMEDIATE_BOUND[1]
    if false_loop:
        assert out["weight"][-1] < 0.1 and out["rejected"] == [(lw.FRAMES, 4 * lw.FRAMES)]
        assert out["weight"][:-1].min() > 0.5
    else:
        assert out["rejected"] == []
    assert_map_equal(sm)
    # the active submap's correction reaches its base poses and the next frame
    Rn, Tn = out["poses"][fa]
    assert np.allclose(sm.submap_collection.submaps_base_R_np[act], Rn) and np.allclose(sm.global_map.submaps_base_T_np[act], Tn)
    Rc = Rn @ X_old[0].T
    Tc = Tn - Rc @ X_old[1]
    Ro, To = lw.odometry_pose(lw.N_LOOP - 1, 1)
    R1, T1 = sm.convert_by_pgo(next_fid, Ro, To)
    assert np.allclose(R1, Rc @ Ro, atol=1e-12) and np.allclose(T1, Rc @ To + Tc, atol=1e-12)


def test_active_correction_is_sent_to_peers():
    sm, _ = run_loop_world()
    sent = []
    sm.traj_send_handle = lambda packed: sent.append(sm._unpack(packed))
    loops = sm.detect_loops(min_gap=2)
    out = sm.optimize_poses(loops)
    fa = sm.active_submap_frame_id
    got = {}
    for d in sent:
        got.update(d)
    assert set(got) == set(out["poses"]) - {0}
    assert np.array_equal(got[fa][0], out["poses"][fa][0]) and np.array_equal(got[fa][1], out["poses"][fa][1])


def test_octomap_flow_with_a_given_loop():
    from taichislam_b200.mapping.submap_mapping import SubmapMapping
    from taichislam_b200.mapping.taichi_octomap import Octomap
    from test_gpu_octo_fuse_update import KH, assert_same, rebuild
    from util import rot_xyz
    opts = dict(map_scale=[12.8, 12.8], voxel_scale=VS, max_ray_length=6.0, occupancy_model="logodds", min_occupy_thres=1)
    sm = SubmapMapping(Octomap, keyframe_step=2, sub_opts=dict(opts, max_submap_num=16), global_opts=dict(opts),
                       global_fusion="incremental")
    sm.set_dep_camera_intrinsic(KH)
    d = syn.scene_room(h=120, w=160)
    true = {}
    for q in range(8):
        R, T = rot_xyz(0.0, 0.0, 0.1 * q), np.array([0.05 * q, 0.0, 0.0])
        true[q] = (R, T)
        drift = P.exp([0.01 * q, 0.0, 0.0, 0.0, 0.0, 0.002 * q])
        sm.recast_depth_to_map_by_frame(q, True, (drift[0] @ R, drift[0] @ T + drift[1]), (np.eye(3), np.zeros(3)), d, None)
    fq, fd = 4, 0
    Z = P.relative(*true[fq], *true[fd])
    out = sm.optimize_poses({(fq, fd): dict(R=Z[0], T=Z[1], H=np.eye(6) * 1e4)})
    assert out["info"]["F"] < out["info"]["F0"]
    assert_same(sm.global_map._h, rebuild(sm, opts))
