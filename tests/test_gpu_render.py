"""GPU: rendering of the TSDF's zero level (tslam_tsdf_render) against tests/render_reference.py, bit for bit: the
synthetic scenes and the box room at several poses, several submaps in one call, colour on a textured map, batches
and repeated calls, the flush of queued frames, no side effects, a rendered frame tracked back to its pose,
DenseTSDF.render on a submap with a base pose, and the refusals that need the handle."""
import numpy as np
import pytest

import render_reference as ref
import submap_register_reference as reg
import track_world as tw
from taichislam_b200 import _capi as capi
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, tri_multiset

pytestmark = pytest.mark.gpu
F = np.float32
VS = 0.05
MIN_RAY, MAX_RAY = 0.3, 6.0
K_160 = [syn.K_DEPTH[0] / 4, 0.0, syn.K_DEPTH[2] / 4, 0.0, syn.K_DEPTH[4] / 4, syn.K_DEPTH[5] / 4, 0.0, 0.0, 1.0]
GENERIC = (reg.rot([1.0, -2.0, 0.5], 6.0), np.array([0.07, -0.04, 0.11]))


def handle(N=256, Nz=256, **kw):
    from taichislam_b200.tsdf_handle import TsdfHandle
    return TsdfHandle(N, Nz, K=syn.K_DEPTH, max_ray_length=MAX_RAY, min_ray_length=MIN_RAY, max_submaps=kw.pop("max_submaps", 16), **kw)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def got(out, c=0, pixels=None):
    depth, status, nrm, col = out
    r = dict(depth=depth[c].reshape(-1).cpu().numpy(), status=status[c].reshape(-1).cpu().numpy())
    if nrm is not None:
        r["normal"] = nrm[c].reshape(-1, 3).cpu().numpy()
    if col is not None:
        r["color"] = col[c].reshape(-1, 3).cpu().numpy()
    if pixels is not None:
        r = {k: v[pixels] for k, v in r.items()}
    return r


def check(m, R, T, h, w, K9, s=0, pixels=None, color=False, out=None, c=0):
    """m's render of camera (R, T) on submap s equals the reference's, bit for bit; -> the hit fraction."""
    if out is None:
        out = m.render(R[None], T[None], h, w, K9, submaps=[s], color=color)
    g = got(out, c, pixels)
    want = ref.render(ref.from_gather(m.gather(s, color=color), m.N, m.Nz, VS), R, T, h, w, K9, MIN_RAY, MAX_RAY, VS, pixels=pixels,
                      color=color)
    for k in want:
        assert np.array_equal(bits(g[k]), bits(want[k])), (k, np.count_nonzero(~(g[k] == want[k])))
    return float((g["status"] == 1).mean())


@pytest.fixture(scope="module")
def scenes():
    out = {}
    for name, depth in (("S1", syn.scene_plane()), ("S2", syn.scene_sphere(4.0)), ("S4", syn.scene_noise()), ("room", syn.scene_room())):
        m = handle()
        m.integrate_depth(depth, np.eye(3)[None], np.zeros((1, 3)), submaps=[0])
        out[name] = m
    return out


@pytest.fixture(scope="module")
def box_room():
    m = handle()
    for k in range(0, tw.N_FRAMES, 5):
        R, t = tw.pose(k)
        m.integrate_depth(tw.render(R, t, seed=k), R[None], t[None], submaps=[0])
    return m


@pytest.mark.parametrize("name", ["S1", "S2", "S4", "room"])
def test_scenes_bit_exact(scenes, name):
    m = scenes[name]
    for R, T in ((np.eye(3), np.zeros(3)), GENERIC):
        frac = check(m, R, T, 120, 160, K_160)
        assert frac > 0.2, (name, frac)


@pytest.mark.parametrize("k", [12, 21, 33])
def test_box_room_bit_exact(box_room, k):
    R, t = tw.pose(k)
    assert check(box_room, R, t, 120, 160, K_160) > 0.9
    pix = np.sort(np.random.default_rng(k).choice(syn.H * syn.W, 4000, replace=False))
    assert check(box_room, R, t, syn.H, syn.W, syn.K_DEPTH, pixels=pix) > 0.9


def test_several_submaps_in_one_call():
    m = handle()
    bases = {0: (np.eye(3), np.zeros(3)), 3: (reg.rot([0, 1, 0], 20.0), np.array([0.3, 0.0, -0.2]))}
    for s, (Rb, Tb) in bases.items():
        for k in range(0, tw.N_FRAMES, 10):
            R, t = reg.local_pose((Rb, Tb), *tw.pose(k))
            m.integrate_depth(tw.render(*tw.pose(k), seed=k), R[None], t[None], submaps=[s])
    cams = [(0, 21), (3, 21), (3, 7), (0, 33)]
    Rs, Ts = zip(*[reg.local_pose(bases[s], *tw.pose(k)) for s, k in cams])
    out = m.render(np.stack(Rs), np.stack(Ts), 120, 160, K_160, submaps=[s for s, _ in cams])
    for c, (s, k) in enumerate(cams):
        assert check(m, Rs[c], Ts[c], 120, 160, K_160, s=s, out=out, c=c) > 0.5   # a coverage check: 0.796 measured for frame 33 on submap 0


def test_textured_map_colour_bit_exact_and_refused_without_texture(box_room):
    m = handle(texture_enabled=True)
    for k in range(0, tw.N_FRAMES, 5):
        R, t = tw.pose(k)
        m.integrate_depth(tw.render(R, t, seed=k)[None], R[None], t[None], submaps=[0], texture=syn.texture_gradient(k)[None])
    for k in (21, 33):
        assert check(m, *tw.pose(k), 120, 160, K_160, color=True) > 0.9
    with pytest.raises(capi.TslamError) as e:
        box_room.render(np.eye(3)[None], np.zeros((1, 3)), 8, 8, K_160, color=True)
    assert e.value.code == capi.E_INVALID


def test_batches_are_bit_identical_to_single_cameras_and_repeatable(box_room):
    rng = np.random.default_rng(5)
    for n in (1, 7, 64):
        ks = rng.integers(0, tw.N_FRAMES, n)
        poses = [tw.perturb(*tw.pose(int(k)), rng, dt=0.03, deg=2.0) for k in ks]
        Rs, Ts = np.stack([p[0] for p in poses]), np.stack([p[1] for p in poses])
        batch = [a.cpu().numpy() for a in box_room.render(Rs, Ts, 120, 160, K_160)[:3]]
        again = [a.cpu().numpy() for a in box_room.render(Rs, Ts, 120, 160, K_160)[:3]]
        for a, b in zip(batch, again):
            assert np.array_equal(bits(a), bits(b))
        for c in range(n):
            one = [a.cpu().numpy() for a in box_room.render(Rs[c:c + 1], Ts[c:c + 1], 120, 160, K_160)[:3]]
            for a, b in zip(batch, one):
                assert np.array_equal(bits(a[c:c + 1]), bits(b)), (n, c)


def dense(base=None):
    from taichislam_b200.mapping.dense_tsdf import DenseTSDF
    m = DenseTSDF(map_scale=[12.8, 12.8], voxel_scale=VS, num_voxel_per_blk_axis=16, max_ray_length=MAX_RAY, max_submap_num=4,
                  max_disp_particles=1 << 16)
    m.set_dep_camera_intrinsic(syn.K_DEPTH)
    if base is not None:
        m.switch_to_next_submap()
        m.set_base_pose_submap(1, *base)
    return m


def test_queued_frames_are_seen_without_a_flush():
    res = []
    for flush in (False, True):
        m = dense((np.eye(3), np.zeros(3)))
        for k in (20, 25, 30):
            R, t = tw.pose(k)
            m.recast_depth_to_map(R, t, tw.render(R, t, seed=k), None)
        if flush:
            m._flush()
        res.append(m.render(*tw.pose(27), 120, 160, K=K_160))
    assert (res[0]["status"] == 1).mean() > 0.5
    for k in res[0]:
        assert np.array_equal(bits(res[0][k]), bits(res[1][k])), k


def test_no_side_effects(box_room):
    m = box_room
    m.esdf_update()
    rows = as_dict_rows(*m.gather(0))
    esdf = as_dict_rows(*m.esdf_gather(0))
    n0, v0, _ = m.marching_cubes()
    before = m.stats()
    m.render(np.stack([tw.pose(k)[0] for k in (3, 21)]), np.stack([tw.pose(k)[1] for k in (3, 21)]), 240, 320, K_160)
    after = m.stats()
    assert after["launches"] > before["launches"]
    for k in before:
        if k != "launches":
            assert before[k] == after[k], k
    for x, y in zip(rows, as_dict_rows(*m.gather(0))):
        assert np.array_equal(bits(x), bits(y))
    for x, y in zip(esdf, as_dict_rows(*m.esdf_gather(0))):
        assert np.array_equal(bits(x), bits(y))
    n1, v1, _ = m.marching_cubes()
    assert n0 == n1 and np.array_equal(tri_multiset(v0), tri_multiset(v1))


# A rendered 640 x 480 frame at pose P (frame 21's), rounded to uint16 mm, tracks back to P from a start 3 cm and 2 degrees
# off.  The CPU reference run (tests/test_render_reference_cpu.py, oracle-integrated map, step 4) lands 1.25 mm and
# 0.031 degrees from P.
def test_rendered_frame_tracks_back_to_its_pose(box_room):
    Rt, tt = tw.pose(21)
    depth, status, _, _ = box_room.render(Rt[None], tt[None], syn.H, syn.W, syn.K_DEPTH, normals=False)
    z = depth[0].cpu().numpy().astype(np.float64)
    d = np.where(status[0].cpu().numpy() > 0, np.round(z * 1000.0), 0).astype(np.uint16)
    for s in (4, 0, 1):
        R0, T0 = tw.perturb(Rt, tt, np.random.default_rng(s), dt=0.03, deg=2.0)
        res = box_room.track_depth(d, R0[None], T0[None])
        et, er = reg.pose_error(res["R"][0], res["T"][0], Rt, tt)
        assert res["status"][0] == 0 and et < 0.25 * VS and er < 0.25, (s, et, er)


def test_dense_tsdf_render_on_a_submap_with_a_base_pose():
    base = (reg.rot([0, 1, 0], 25.0) @ reg.rot([1, 0, 0], 4.0), np.array([0.4, -0.1, 0.3]))
    m = dense(base)
    for k in range(0, tw.N_FRAMES, 5):
        R, t = tw.pose(k)
        m.recast_depth_to_map(R, t, tw.render(R, t, seed=k), None)
    Rw, tw_ = tw.pose(21)
    res = m.render(Rw, tw_, 120, 160, K=K_160)
    Rl, Tl = m.convert_by_base(Rw, tw_)
    depth, status, nrm, _ = m._h.render(Rl[None], Tl[None], 120, 160, K_160, submaps=[1])
    assert np.array_equal(bits(res["depth"]), bits(depth[0].cpu().numpy()))
    assert np.array_equal(res["status"], status[0].cpu().numpy()) and (res["status"] == 1).mean() > 0.9
    want = (nrm[0].cpu().numpy().astype(np.float64) @ base[0].T).astype(F)
    assert np.array_equal(bits(res["normal"]), bits(want))
    # world-frame normals of the room's walls face the camera
    ray = (np.asarray(Rw) @ ref.directions(np.eye(3), K_160, np.arange(160 * 120) % 160, np.arange(160 * 120) // 160).T).T
    one = res["status"].reshape(-1) == 1
    assert np.mean((res["normal"].reshape(-1, 3)[one] * ray[one]).sum(1) < 0) > 0.99


def test_refusals_that_need_the_handle(box_room):
    m = box_room
    I, Z = np.eye(3)[None], np.zeros((1, 3))

    def refused(*args, **kw):
        with pytest.raises(capi.TslamError) as e:
            m.render(*args, **kw)
        assert e.value.code == capi.E_INVALID

    refused(I, Z, 8, 8, K_160, submaps=[16])
    refused(I, Z, 8, 8, K_160, submaps=[-1])
    refused(I, np.array([[np.nan, 0, 0]]), 8, 8, K_160)
    refused(np.array([np.diag([np.inf, 1, 1])]), Z, 8, 8, K_160)
    refused(I, np.array([[1e300, 0, 0]]), 8, 8, K_160)                 # finite in f64, not in f32
    refused(I, Z, 8, 8, K_160, color=True)
    empty = m.render(I, Z, 8, 8, K_160, submaps=[5])                  # an empty submap renders nothing
    assert not empty[1].any() and not empty[0].any()
