"""The render reference (tests/render_reference.py) pinned on hand-worked answers before any GPU run is held to it:
planes with known depth and normal, a zero on a sample, back faces, invalid slabs, the depth range, absent blocks and
the volume edge, status 2, a linear colour field, the analytic box room rendered from a map the CPU oracle integrated,
and a rendered frame tracked back to the pose it was rendered at."""
import numpy as np
import pytest

import frame_track_reference as ftr
import render_reference as ref
import submap_register_reference as reg
import track_world as tw

F = np.float32
VS = 0.0625          # binary fractions: sample depths and voxel positions are exact
K_SMALL = [40.0, 0.0, 4.0, 0.0, 40.0, 3.0, 0.0, 0.0, 1.0]
H, W = 6, 8


def rows(field, lo=(-24, -24, 0), hi=(24, 24, 40), w=None):
    """Voxel rows of the TSDF field(p) (f64 in, metres) over the index box [lo, hi); w(idx) -> weights (default 1)."""
    r = [np.arange(a, b) for a, b in zip(lo, hi)]
    I, J, K = np.meshgrid(*r, indexing="ij")
    idx = np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)
    p = idx.astype(np.float64) * VS
    return idx, field(p).astype(F), (np.ones(len(idx), F) if w is None else w(idx).astype(F))


def scene(field, N=128, Nz=128, **kw):
    return ref.Scene(*rows(field, **kw), N, Nz, VS)


def plane(z0):
    return lambda p: z0 - p[:, 2]


def draw(sc, R=np.eye(3), T=np.zeros(3), z_min=0.25, z_max=3.0, step=VS, **kw):
    return ref.render(sc, R, T, H, W, K_SMALL, z_min, z_max, step, **kw)


def test_fronto_parallel_plane():
    out = draw(scene(plane(1.01)))
    assert np.all(out["status"] == 1)
    assert np.all(np.abs(out["depth"] - 1.01) < 1e-6), out["depth"]
    assert np.all(np.abs(out["normal"] - [0.0, 0.0, -1.0]) < 1e-6)


def test_tilted_plane_at_a_generic_pose():
    n = np.array([0.3, -0.2, 1.0])
    n /= np.linalg.norm(n)
    c = 1.4
    sc = scene(lambda p: c - p @ n)
    R, T = reg.rot([1.0, 2.0, 0.5], 7.0), np.array([0.11, -0.07, 0.05])
    out = draw(sc, R, T)
    d = ref.directions(R, K_SMALL, np.arange(H * W) % W, np.arange(H * W) // W).astype(np.float64)
    want = (c - n @ T.astype(F).astype(np.float64)) / (d @ n)
    assert np.all(out["status"] == 1)
    assert np.max(np.abs(out["depth"] - want)) < 1e-5
    assert np.max(np.abs(out["normal"] + n)) < 1e-5


def test_zero_on_a_sample_gives_that_sample():
    out = draw(scene(plane(1.0)))                              # z_k = 0.25 + k / 16: sample 12 is exactly 1.0, D = 0 there
    assert np.all(out["status"] == 1) and np.all(out["depth"] == F(1.0))


def test_back_face_is_not_a_hit():
    out = draw(scene(lambda p: p[:, 2] - 1.01))                # the camera is inside: D goes - -> +
    assert np.all(out["status"] == 0) and np.all(out["depth"] == 0) and np.all(np.isnan(out["normal"]))


def test_invalid_slab_hides_the_crossing_inside_it_and_not_the_one_after():
    slab = lambda idx: np.where((idx[:, 2] >= 15) & (idx[:, 2] <= 17), 0.0, 1.0)     # z in [0.9375, 1.0625]: W = 0
    out = draw(scene(plane(1.01), w=slab))
    assert np.all(out["status"] == 0)
    second = lambda p: np.where(p[:, 2] < 1.0, 1.01 - p[:, 2], 1.51 - p[:, 2])       # positive again after the slab
    out = draw(scene(second, w=slab))
    assert np.all(out["status"] == 1) and np.all(np.abs(out["depth"] - 1.51) < 1e-6)


@pytest.mark.parametrize("z_min,z_max,hit", [(0.25, 1.0625, True), (0.25, 1.06, False), (1.0, 3.0, True), (1.0125, 3.0, False)])
def test_depth_range(z_min, z_max, hit):
    # z_max 1.0625: K = 14, the last sample is 1.0625 >= 1.01; z_max 1.06: K = 13, the last is 1.0.  z_min 1.0: D_0 > 0;
    # z_min 1.0125: the first sample is already behind the surface
    out = draw(scene(plane(1.01)), z_min=z_min, z_max=z_max)
    assert np.all(out["status"] == (1 if hit else 0))
    if hit:
        assert np.all(np.abs(out["depth"] - 1.01) < 1e-6)


def test_absent_block_and_volume_edge():
    idx, t, w = rows(plane(1.51))
    gone = (idx[:, 0] >= 0) & (idx[:, 0] < 16) & (idx[:, 1] >= 0) & (idx[:, 1] < 16) & (idx[:, 2] >= 16) & (idx[:, 2] < 32)
    sc = ref.Scene(idx[~gone], t[~gone], w[~gone], 128, 128, VS)
    h, w_ = 40, 40
    K = [40.0, 0.0, 20.0, 0.0, 40.0, 20.0, 0.0, 0.0, 1.0]
    out = ref.render(sc, np.eye(3), np.zeros(3), h, w_, K, 0.25, 3.0, VS)
    j, i = np.divmod(np.arange(h * w_), w_)
    u = (i - 20.0) / 40.0 * 1.51 / VS, (j - 20.0) / 40.0 * 1.51 / VS   # voxel coordinates where the ray meets the plane
    inside = (u[0] > 0.5) & (u[0] < 14.5) & (u[1] > 0.5) & (u[1] < 14.5)
    outside = (u[0] < -1.5) | (u[0] > 16.5) | (u[1] < -1.5) | (u[1] > 16.5)
    assert inside.sum() > 20 and outside.sum() > 200
    assert np.all(out["status"][inside] == 0) and np.all(out["status"][outside] == 1)
    assert np.all(np.abs(out["depth"][outside] - 1.51) < 1e-6)
    # volume edge: Nz = 32, so a cell's low corner must be < 15 (z < 0.9375); the rows end there too
    edge = lambda z0: ref.Scene(*rows(plane(z0), hi=(24, 24, 16)), 128, 32, VS)
    assert np.all(draw(edge(0.8))["status"] == 1)
    assert np.all(draw(edge(0.95))["status"] == 0)


def test_status_2_when_a_corner_of_the_hit_cell_is_invalid():
    # samples 3 voxels apart: u = 4 + 3k, cells {16, 17} (k = 4) and {19, 20} (k = 5) are valid; the surface is at
    # u = 17.5, whose cell {17, 18} has the W = 0 voxel plane k = 18
    sc = scene(plane(17.5 * VS), w=lambda idx: np.where(idx[:, 2] == 18, 0.0, 1.0))
    out = draw(sc, step=3 * VS)
    assert np.all(out["status"] == 2) and np.all(out["depth"] == F(17.5 * VS)) and np.all(np.isnan(out["normal"]))


def test_linear_colour_field():
    idx, t, w = rows(plane(1.01))
    p = idx.astype(np.float64) * VS
    col = np.stack([100 + 10 * p[:, 0] + 20 * p[:, 1] + 30 * p[:, 2], 50 - 5 * p[:, 0], 200 + 40 * p[:, 2]], 1).astype(F)
    sc = ref.Scene(idx, t, w, 128, 128, VS, col=col)
    out = draw(sc, color=True)
    d = ref.directions(np.eye(3), K_SMALL, np.arange(H * W) % W, np.arange(H * W) // W).astype(np.float64)
    x = d * out["depth"][:, None].astype(np.float64)
    want = np.stack([100 + 10 * x[:, 0] + 20 * x[:, 1] + 30 * x[:, 2], 50 - 5 * x[:, 0], 200 + 40 * x[:, 2]], 1)
    assert np.all(out["status"] == 1) and np.max(np.abs(out["color"] - want)) < 1e-3


# The box room: the CPU oracle integrates every fifth frame of the trajectory (tests/test_frame_track_reference_cpu.py's
# map); frames 12, 21 and 33, not integrated, are rendered at 160 x 120 and compared with the exact depth on pixels whose
# 3 x 3 neighbourhood has no depth discontinuity (max - min < 5 cm).  Achieved (median / 95th percentile of |error| in mm,
# hit fraction): frame 12 2.09 / 8.78, 1.000; frame 21 1.92 / 7.34, 0.996; frame 33 2.07 / 7.95, 0.935 - the map's zero
# level is a projective TSDF of eight views; frame 33 looks partly past what they observed.
ROOM_VS = 0.05
ROOM_FRAMES = (12, 21, 33)
K_ROOM = [tw.syn.K_DEPTH[0] / 4, 0.0, tw.syn.K_DEPTH[2] / 4, 0.0, tw.syn.K_DEPTH[4] / 4, tw.syn.K_DEPTH[5] / 4, 0.0, 0.0, 1.0]
BOUND_MEDIAN, BOUND_P95, BOUND_HIT = 0.004, 0.015, 0.90


@pytest.fixture(scope="module")
def room(oracle_lib):
    from oracle.oracle import OracleTSDF
    o = OracleTSDF(map_scale=[12.8, 12.8], K=tw.syn.K_DEPTH, max_ray_length=6.0, is_global_map=True)
    for k in range(0, tw.N_FRAMES, 5):
        R, t = tw.pose(k)
        o.integrate_depth(R, t, tw.render(R, t, seed=k))
    g = o.gather(0)
    return ref.Scene(*g[:3], o.N, o.Nz, ROOM_VS)


def smooth_pixels(z):
    """Pixels whose 3 x 3 neighbourhood of the exact depth z has max - min < 5 cm (border pixels excluded)."""
    h, w = z.shape
    st = np.stack([z[1 + a:h - 1 + a, 1 + b:w - 1 + b] for a in (-1, 0, 1) for b in (-1, 0, 1)])
    ok = np.zeros((h, w), bool)
    ok[1:-1, 1:-1] = (st.max(0) - st.min(0)) < 0.05
    return ok


def room_errors(room, k):
    R, t = tw.pose(k)
    h, w = 120, 160
    out = ref.render(room, R, t, h, w, K_ROOM, 0.3, 6.0, ROOM_VS)
    z = tw.depth_m(R, t, h, w, K_ROOM)
    ok = smooth_pixels(z).ravel()
    hit = out["status"][ok] == 1
    err = np.abs(out["depth"][ok][hit] - z.ravel()[ok][hit])
    return np.median(err), np.percentile(err, 95), hit.mean()


@pytest.mark.parametrize("k", ROOM_FRAMES)
def test_box_room_depth(room, k):
    med, p95, frac = room_errors(room, k)
    assert med < BOUND_MEDIAN and p95 < BOUND_P95 and frac > BOUND_HIT, (med, p95, frac)


# Render -> track: the map's view at pose P (frame 21's), rounded to uint16 mm, is tracked from P perturbed by 3 cm and
# 2 degrees at step 4 (only the pixels the tracker samples are rendered here).  Achieved: 1.25 mm, 0.031 degrees, the
# same from three perturbed starts.
def test_rendered_frame_tracks_back_to_its_pose(room):
    h, w, step = tw.syn.H, tw.syn.W, 4
    Rt, tt = tw.pose(21)
    jj, ii = np.meshgrid(np.arange(0, h, step), np.arange(0, w, step), indexing="ij")
    pix = (jj * w + ii).ravel()
    out = ref.render(room, Rt, tt, h, w, tw.syn.K_DEPTH, 0.3, 6.0, ROOM_VS, pixels=pix)
    depth = np.zeros(h * w, np.uint16)
    depth[pix] = np.where(out["status"] > 0, np.round(out["depth"].astype(np.float64) * 1000.0), 0).astype(np.uint16)
    p = ftr.select_depth(depth.reshape(h, w), tw.syn.K_DEPTH, step, 0.3, 6.0)
    R0, T0 = tw.perturb(Rt, tt, np.random.default_rng(4), dt=0.03, deg=2.0)
    res = ftr.track(room.rd, p, R0, T0, ROOM_VS)
    et, er = reg.pose_error(res["R"], res["T"], Rt, tt)
    assert res["status"] == 0 and et < 0.25 * ROOM_VS and er < 0.25, (et, er)
