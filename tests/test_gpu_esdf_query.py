"""GPU: batched ESDF distance / gradient queries and the ESDF slice export (tslam_esdf_query, tslam_esdf_extract_slice),
bit for bit against tests/esdf_query_reference.py on the map as of the last update."""
import numpy as np
import pytest

import esdf_query_reference as eqr
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu
F = np.float32
VS = 0.05


def state_of(g, submap=0, vs=VS):
    """The map as of now (call right after an update): observed rows with their TSDF and ESDF."""
    gi, gt, _, _ = as_dict_rows(*g.gather(submap))
    ei, ee = as_dict_rows(*g.esdf_gather(submap))
    assert np.array_equal(gi, ei)
    return eqr.EsdfState(gi, gt, ee, g.N, g.Nz, vs)


def assert_bit_equal(got, ref):
    (d, gr, v), (rd, rg, rv) = got, ref
    assert np.array_equal(v, rv), f"valid differs at {int((v != rv).sum())} points"
    assert np.array_equal(d[v].view(np.uint32), rd[v].view(np.uint32)), f"dist differs, max {np.abs(d[v] - rd[v]).max()}"
    assert np.array_equal(gr[v].view(np.uint32), rg[v].view(np.uint32)), f"grad differs, max {np.abs(gr[v] - rg[v]).max()}"
    assert np.isnan(d[~v]).all() and np.isnan(gr[~v]).all()


def special_points(st, rng, n_each=4000):
    """Exact voxel centres, corner cubes straddling 2 / 4 / 8 blocks, negative coordinates near 0, the volume's edges
    and beyond, non-finite and huge coordinates."""
    obs = st.idx[rng.integers(0, st.idx.shape[0], n_each)].astype(np.int64)
    pts = [obs.astype(F) * F(VS)]                                   # f = 0
    for axes in ((0,), (0, 1), (0, 1, 2), (1,), (2,), (1, 2)):      # 2, 4, 8 blocks
        i = obs.copy()
        for a in axes:
            i[:, a] = (i[:, a] & ~15) | 15
        f = rng.uniform(0.0, 1.0, size=i.shape)
        pts.append(((i + f) * VS).astype(F))
    pts.append(rng.uniform(-0.2, 0.0, size=(n_each, 3)).astype(F))    # negative, floor != trunc
    lo, hi, loz, hiz = -st.hN, st.N - st.hN - 1, -st.hNz, st.Nz - st.hNz - 1
    edge = []
    for u in (lo - 0.5, lo - 1e-3, lo, lo + 0.25, hi - 0.25, hi - 1e-3, hi, hi + 0.5):
        edge += [[u, 0, 1], [0, u, 1], [0, 1, u * (st.Nz / st.N)]]
    for u in (loz - 0.5, loz, hiz - 1e-3, hiz, hiz + 0.5):
        edge.append([1, 0, u])
    pts.append((np.array(edge) * VS).astype(F))
    pts.append(np.array([[np.nan, 0, 0], [0, np.nan, 0], [0, 0, np.nan], [np.inf, 0, 0], [0, -np.inf, 0], [0, 0, np.inf],
                         [1e30, 0, 0], [0, -1e30, 0], [0, 0, 1e30], [-1e30, 1e30, 0]], F))
    return np.concatenate(pts)


def room_map(**kw):
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True, max_ray_length=4.0, **kw)
    g.integrate_depth(syn.scene_room(), np.eye(3)[None], np.zeros((1, 3)))
    return g


def test_query_room_bit_exact_and_torch_path():
    import torch
    g = room_map()
    g.esdf_update()
    st = state_of(g)
    rng = np.random.default_rng(7)
    p = np.concatenate([rng.uniform([-3, -2, -0.5], [3, 2, 5.5], size=(1 << 20, 3)).astype(F), special_points(st, rng)])
    got = g.esdf_query(p)
    ref = eqr.query(st, p)
    assert_bit_equal(got, ref)
    v = ref[2]
    assert 0.05 < v[: 1 << 20].mean() < 0.95
    # every straddle group produced valid answers (the corner-block resolution is exercised, not skipped)
    assert v[(1 << 20) + 4000: (1 << 20) + 7 * 4000].reshape(6, 4000).any(1).all()
    # torch in -> torch CUDA tensors out, equal to the numpy path
    pt = torch.from_numpy(p).cuda()
    d, gr, vv = g.esdf_query(pt)
    assert d.is_cuda and gr.is_cuda and vv.is_cuda and vv.dtype == torch.bool and gr.shape == (p.shape[0], 3)
    assert_bit_equal((d.cpu().numpy(), gr.cpu().numpy(), vv.cpu().numpy()), got)
    # n == 0 is a no-op
    d0, g0, v0 = g.esdf_query(np.zeros((0, 3), F))
    assert d0.shape == (0,) and g0.shape == (0, 3) and v0.shape == (0,)


def test_query_volume_edges_with_known_corners():
    """A slab of known voxels along the +x, -x and +z faces of a 64^3 volume: the bounds test decides, not missing data.
    (vs = 1/16 m, so that u = p / vs is exactly the index coordinate the points were made from.)"""
    from taichislam_b200.tsdf_handle import TsdfHandle
    vs = 0.0625
    g = TsdfHandle(64, 64, voxel_scale=vs, is_global_map=True, max_ray_length=4.0)
    r = np.arange(-32, 32)
    I, J, K = np.meshgrid(r, r, r, indexing="ij")
    idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
    keep = (np.abs(idx[:, 0] + 0.5) > 28) | (idx[:, 2] > 28)
    idx = idx[keep]
    t = (0.3 + 0.01 * idx[:, 1]).astype(F)                                 # positive: relaxed values
    t[(idx[:, 1] % 7) == 0] = 0.01                                          # fixed-band seeds
    g.scatter(0, idx, t, np.ones(len(t), F), np.zeros(len(t), np.int8))
    g.esdf_update()
    st = state_of(g, vs=vs)
    rng = np.random.default_rng(11)
    u = []
    for x in (30.0, 30.999, 31.0, 31.5, -32.0, -31.5, -32.001):
        u += [[x, rng.uniform(-31, 30), rng.uniform(-31, 30)] for _ in range(50)]
    for z in (29.5, 30.999, 31.0):
        u += [[rng.uniform(-31, 30), rng.uniform(-31, 30), z] for _ in range(50)]
    p = (np.array(u) * vs).astype(F)
    got = g.esdf_query(p)
    assert_bit_equal(got, eqr.query(st, p))
    v = got[2].reshape(-1, 50)
    assert v[[0, 1, 4, 5, 7, 8]].all() and not v[[2, 3, 6, 9]].any()


def test_query_after_every_incremental_update_512():
    """The moving-sphere stream of test_esdf_incremental_equals_full_512: bit-exact after every incremental update."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True, max_ray_length=6.0)
    Rs, Ts = syn.stream_poses(20, start=40)
    rng = np.random.default_rng(5)
    n_upd = 0
    for q in range(20):
        g.integrate_depth(syn.scene_sphere(3.0 if q < 10 else 3.6), Rs[q][None], Ts[q][None])
        if q % 3 != 2 and q != 19:
            continue
        s = g.esdf_update2()
        assert q == 2 or s["raise_sweeps"] >= 1
        n_upd += 1
        st = state_of(g)
        p = np.concatenate([rng.uniform(-4.5, 4.5, size=(300000, 3)).astype(F), special_points(st, rng, 2000)])
        got = g.esdf_query(p)
        assert_bit_equal(got, eqr.query(st, p))
        assert got[2].sum() > 10000
    assert n_upd == 7


def test_answers_are_as_of_the_last_update():
    g = room_map()
    g.esdf_update()
    st = state_of(g)
    blocks0 = np.unique(st.idx >> 4, axis=0)
    rng = np.random.default_rng(9)
    p = np.concatenate([rng.uniform([-3, -2, -0.5], [3, 2, 5.5], size=(200000, 3)).astype(F), special_points(st, rng, 2000)])
    before = g.esdf_query(p)
    # more frames, no update: every answer is bit-identical, points in the newly allocated blocks are invalid
    for a in (0.4, -0.5, 0.9):
        g.integrate_depth(syn.scene_room(seed=4), rot_xyz(0.0, a, 0.2)[None], np.array([[0.3, -0.2, 0.1]]))
    after = g.esdf_query(p)
    assert_bit_equal(after, before)
    gi = g.gather()[0]
    new = ~(np.isin(np.ravel_multi_index(((gi >> 4) + 64).T, (128, 128, 128)),
                    np.ravel_multi_index((blocks0 + 64).T, (128, 128, 128))))
    assert new.sum() > 1000
    pn = np.concatenate([gi[new].astype(F) * F(VS), ((gi[new] + 0.5) * VS).astype(F)])
    dn, gn, vn = g.esdf_query(pn)
    assert not vn.any() and np.isnan(dn).all()
    # ... and the next update takes them in
    g.esdf_update()
    st2 = state_of(g)
    assert_bit_equal(g.esdf_query(p), eqr.query(st2, p))
    assert g.esdf_query(gi[new].astype(F) * F(VS))[2].mean() > 0.2


def test_reused_pool_slots_after_reset_answer_invalid():
    g = room_map()
    for a in (0.5, -0.5, 1.2):
        g.integrate_depth(syn.scene_room(seed=5), rot_xyz(0.0, a, 0.0)[None], np.zeros((1, 3)))
    g.esdf_update()
    n_first = g.stats()["n_blocks"]
    g.reset()
    g.integrate_depth(syn.scene_plane(2.0), np.eye(3)[None], np.zeros((1, 3)))    # fewer blocks than before the reset
    g.esdf_update()
    st = state_of(g)
    n_second = g.stats()["n_blocks"]
    assert n_second < n_first
    old_blocks = np.unique(st.idx >> 4, axis=0)
    g.integrate_depth(syn.scene_room(seed=5), rot_xyz(0.0, 1.2, 0.0)[None], np.zeros((1, 3)))   # into new blocks
    assert g.stats()["n_blocks"] > n_second
    gi = g.gather()[0]
    new = ~(np.isin(np.ravel_multi_index(((gi >> 4) + 64).T, (128, 128, 128)),
                    np.ravel_multi_index((old_blocks + 64).T, (128, 128, 128))))
    assert new.sum() > 1000
    pn = np.concatenate([gi[new].astype(F) * F(VS), ((gi[new] + 0.25) * VS).astype(F)])
    got = g.esdf_query(pn)
    assert not got[2].any()
    assert_bit_equal(got, eqr.query(st, pn))


def test_query_refuses_stale_or_foreign_state():
    from taichislam_b200 import _capi as capi
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=False, max_ray_length=4.0, max_submaps=4)
    p = np.zeros((4, 3), F)
    with pytest.raises(capi.TslamError, match="no ESDF has been computed"):
        g.esdf_query(p)
    g.integrate_depth(syn.scene_room(), np.eye(3)[None], np.zeros((1, 3)), submaps=1)
    g.esdf_update(submap=1)
    g.esdf_query(p, submap=1)
    with pytest.raises(capi.TslamError, match="submap 1, not 0"):
        g.esdf_query(p, submap=0)
    with pytest.raises(capi.TslamError, match="submap 1, not 2"):
        g.esdf_slice(1.0, submap=2)
    g.reset()
    with pytest.raises(capi.TslamError, match="reset"):
        g.esdf_query(p, submap=1)
    with pytest.raises(capi.TslamError, match="reset"):
        g.esdf_slice(1.0, submap=1)


def test_plane_known_answer():
    """S1 plane at z = 3 m, identity pose.  In the interior of the frustum between 1 m and 2.5 m the field is the
    distance to the plane: ESDF(v) = E(h) + path length from a fixed-band voxel h, and every fixed voxel carries its
    TSDF, which is the projective distance of its samples, not the Euclidean distance 3 - z of its centre.  With
    e = max |TSDF - (3 - z)| over the fixed voxels that can reach the query region (|x|, |y| <= 1.2 m; anything further
    out needs a path longer by > 0.2 m), a straight path down the z column gives ESDF <= (3 - z) + e, and any path is
    at least as long as the z distance, so ESDF >= (3 - z) - e.  The interpolant of a field within e of the linear
    3 - z is within e of it, and its differences over one voxel are within 2e: |dist - (3 - z)| <= e,
    |grad - (0, 0, -1)| <= 2e / vs (plus f32 rounding of the ~40 path additions)."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True)
    g.integrate_depth(syn.scene_plane(3.0), np.eye(3)[None], np.zeros((1, 3)))
    g.esdf_update()
    gi, gt, _, _ = g.gather()
    p_c = gi.astype(np.float64) * VS
    fixed = np.abs(gt) < F(VS)
    assert fixed.sum() > 1000 and p_c[fixed, 2].min() > 2.8       # the band is the plane, nowhere else
    near = fixed & (np.abs(p_c[:, 0]) <= 1.2) & (np.abs(p_c[:, 1]) <= 1.2)
    e = float(np.abs(gt[near] - (3.0 - p_c[near, 2])).max()) + 1e-4
    rng = np.random.default_rng(13)
    z = rng.uniform(1.0, 2.5, 200000)
    xy = rng.uniform(-0.25, 0.25, size=(200000, 2))
    p = np.concatenate([xy, z[:, None]], 1).astype(F)
    d, gr, v = g.esdf_query(p)
    assert v.mean() > 0.9
    zt = p[v, 2].astype(np.float64)
    print(f"plane: e = {e:.3g} m, max |dist - (3 - z)| = {np.abs(d[v] - (3.0 - zt)).max():.3g}, "
          f"max |grad - (0,0,-1)| = {np.abs(gr[v] - [0, 0, -1]).max():.3g}")
    assert np.abs(d[v] - (3.0 - zt)).max() <= e
    assert np.abs(gr[v] - np.array([0.0, 0.0, -1.0])).max() <= 2 * e / VS


def _multiset(xyz, val):
    a = np.concatenate([xyz.astype(F), val.astype(F)[:, None]], 1).view(np.uint32)
    return a[np.lexsort(a.T[::-1])]


def test_slice_equals_reference_selection():
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = room_map()
    g.esdf_update()
    st = state_of(g)
    total = 0
    for z in (0.3, 0.5, 1.0, 1.37, 2.5, 3.2):
        n, xyz, val = g.esdf_slice(z)
        rx, rv = eqr.slice_rows(st, z)
        assert n == rx.shape[0] > 0
        assert np.array_equal(_multiset(xyz, val), _multiset(rx, rv))
        total += n
    assert total > 2000
    # capacity: saturates, reports the true count, writes a subset of the rows
    n, xyz, val = g.esdf_slice(1.0)
    n2, xyz2, val2 = g.esdf_slice(1.0, cap=n // 3)
    assert n2 == n and xyz2.shape[0] == n // 3
    full = {r.tobytes() for r in _multiset(xyz, val)}
    assert all(r.tobytes() in full for r in _multiset(xyz2, val2))
    # a submap map: positions through the submap's base pose (submap_i_j_k_to_xyz)
    s = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=False, max_ray_length=4.0, max_submaps=4)
    R, T = rot_xyz(0.1, -0.2, 0.4), np.array([0.5, -1.0, 0.25])
    s.set_submap_pose(2, R, T)
    s.integrate_depth(syn.scene_room(), np.eye(3)[None], np.zeros((1, 3)), submaps=2)
    s.esdf_update(submap=2)
    st2 = state_of(s, submap=2)
    n, xyz, val = s.esdf_slice(0.5, submap=2)
    rx, rv = eqr.slice_rows(st2, 0.5, R.astype(F), T.astype(F))
    assert n == rx.shape[0] > 0 and np.array_equal(_multiset(xyz, val), _multiset(rx, rv))


def test_dense_tsdf_esdf_flow():
    import torch
    from taichi_slam.mapping import DenseTSDF
    m = DenseTSDF(map_scale=[12.8, 12.8], voxel_scale=VS, is_global_map=True, max_ray_length=4.0, max_disp_particles=1 << 18)
    m.set_dep_camera_intrinsic(syn.K_DEPTH)
    m.set_base_pose_submap(0, np.eye(3), np.zeros(3))   # the pose table's rows start at zero
    m.recast_depth_to_map(np.eye(3), np.zeros(3), syn.scene_room(), np.array([]))
    rng = np.random.default_rng(3)
    p = rng.uniform([-3, -2, -0.5], [3, 2, 5.5], size=(50000, 3)).astype(F)
    d, gr, v = m.esdf_query(p)
    assert isinstance(d, np.ndarray) and 0.05 < v.mean() < 0.95 and np.isfinite(d[v]).all()
    dt, grt, vt = m.esdf_query(torch.from_numpy(p).cuda(), update=False)
    assert dt.is_cuda and np.array_equal(vt.cpu().numpy(), v) and np.array_equal(dt.cpu().numpy()[v], d[v])
    xyz, val = m.get_voxels_ESDF_slice(1.0)
    k = m.num_export_ESDF_particles[None]
    n, hx, hv = m._h.esdf_slice(1.0)
    assert k == n > 100 and xyz.shape == (1 << 18, 3)
    assert np.array_equal(_multiset(xyz[:k], val[:k]), _multiset(hx, hv))
    # more frames: the slice brings the field up to date first
    m.recast_depth_to_map(rot_xyz(0.0, 0.6, 0.0), np.zeros(3), syn.scene_room(), np.array([]))
    m.get_voxels_ESDF_slice(1.0)
    assert m.num_export_ESDF_particles[None] > k
