"""The bucket kernels merge the points of a CTA on chip before they probe the per-frame bucket index, and unproject depth
pixels without IEEE division.  Bucket sums are exact integers, so any grouping of the additions gives the same records:
these tests hold rays, valid pixels and voxel updates to the CPU oracle exactly, over the scenes S1-S4 and a room,
generic poses, depth frames and point clouds, textured and untextured, on an epoch-mode and a clearing-mode handle.
The CPU tests prove the division forms the kernels use against IEEE f32 division."""
import numpy as np
import pytest

from taichislam_b200 import synthetic as syn
from util import compare_voxels, key_sort, rot_xyz

CLEARING_MAX_POINTS = 1 << 21  # too few index bits left for the launch epoch: the handle runs in clearing mode
COUNTERS = ("n_px", "n_valid", "n_rays", "n_updates", "n_oob")
SCENES = {"S1": lambda: syn.scene_plane(3.0), "S2": lambda: syn.scene_sphere(4.0), "S3": lambda: syn.scene_sphere(8.0),
          "S4": lambda: syn.scene_noise(seed=5), "room": syn.scene_room}
POSES = [(rot_xyz(0.0, 0.0, 0.0), np.zeros(3)), (rot_xyz(0.13, -0.21, 0.7), np.array([0.31, -0.12, 0.07]))]
K_OTHER = [517.3, 0.0, 318.6, 0.0, 516.5, 255.3, 0.0, 0.0, 1.0]  # a second camera: focal lengths of another sensor


# ---- CPU: the division forms -----------------------------------------------------------------------------------------

def fmaf(a, b, c):
    """f32 fused multiply-add, correctly rounded: a*b is exact in f64, TwoSum gives the exact error of the f64 sum, and
    rounding that sum to odd before the f32 rounding makes the result RN(a*b + c)."""
    p = a.astype(np.float64) * b.astype(np.float64)
    cc = c.astype(np.float64)
    s = p + cc
    bv = s - p
    err = (p - (s - bv)) + (cc - bv)
    odd = np.where(err > 0, np.inf, -np.inf)
    with np.errstate(under="ignore"):  # s = 0 with err = 0 (an exact zero) steps nowhere but is computed anyway
        odd = np.nextafter(s, odd)
    s = np.where((err != 0) & ((s.view(np.int64) & 1) == 0), odd, s)
    return s.astype(np.float32)


def div_form(a, b):
    """div_vs (csrc/tslam_internal.cuh): q0 = RN(a * r), r = RN(1/b); q1 = fma(fma(-q0, b, a), r, q0)."""
    b = np.float32(b)
    r = np.float32(1.0) / b
    q0 = a * r
    return fmaf(fmaf(-q0, np.full_like(a, b), a), np.full_like(a, r), q0)


def assert_exact(a, b):
    with np.errstate(all="raise"):
        want = a / np.float32(b)
        got = div_form(a, b)
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    assert bad.size == 0, f"{bad.size} quotients differ, first {a[bad[0]]!r} / {b!r}: {got[bad[0]]!r} vs {want[bad[0]]!r}"


def all_significands(chunk=1 << 21):
    for s in range(0, 1 << 23, chunk):
        yield (np.arange(s, s + chunk, dtype=np.uint32) | np.uint32(0x3F800000)).view(np.float32)


def test_fmaf_emulation():
    """The f32 FMA the division tests rest on: exact cases, and cases where a separate product would round."""
    a = np.array([1.0 + 2.0 ** -23, 3.0, 0.1, -7.5], np.float32)
    b = np.array([1.0 - 2.0 ** -24, 1.0 / 3.0, 10.0, 2.0], np.float32)
    c = np.array([-1.0, -1.0, -1.0, 15.0], np.float32)
    want = [float(np.float32((float(x) * float(y) + float(z)))) for x, y, z in zip(a, b, c)]  # exact in f64 here
    assert fmaf(a, b, c).tolist() == want
    assert fmaf(a, b, c)[0] != np.float32(a[0] * b[0]) + c[0]


def test_depth_division_all_uint16():
    """dep = df / 1000 for every uint16 depth."""
    assert_exact(np.arange(1 << 16, dtype=np.float32), 1000.0)


@pytest.mark.parametrize("b", [syn.FX, K_OTHER[0], K_OTHER[4], 0.05, 0.2, 0.02, 0.0002])
def test_division_every_significand(b):
    """The focal lengths of both test cameras, the 0.05 m voxel of the bucket key and the other voxel sizes of the
    march audit (tests/march_cases.py; 1/16 is a power of two): every f32 significand, which by scaling covers every
    dividend whose quotient stays normal (the check ts_fill_intrin makes when a handle is set up)."""
    for a in all_significands():
        assert_exact(a, np.float32(b))
        assert_exact(-a, np.float32(b))


def test_division_random_and_edge_operands():
    """Random divisors in the ranges of focal lengths and voxel sizes, dividends in the ranges the kernels see
    ((i - cx) * dep up to 6.5e4 px m, coordinates up to 6.4e3 m), and dividends at and next to the rounding boundaries
    of the bucket key ((k + 1/2) * vs)."""
    rng = np.random.default_rng(11)
    for b in np.concatenate([rng.uniform(50.0, 3000.0, 24), rng.uniform(0.005, 1.0, 24)]).astype(np.float32):
        a = np.concatenate([rng.uniform(-6.5e4, 6.5e4, 1 << 16), rng.uniform(-1.0, 1.0, 1 << 14) * 10.0 ** rng.integers(-4, 4, 1 << 14)])
        k = np.arange(-2000, 2000, dtype=np.float64) + 0.5
        edge = (k * np.float64(b)).astype(np.float32)
        a = np.concatenate([a.astype(np.float32), edge, np.nextafter(edge, np.float32(np.inf)), np.nextafter(edge, np.float32(-np.inf))])
        assert_exact(a, b)


# ---- GPU: bucket kernels against the CPU oracle ----------------------------------------------------------------------

def pair(K=syn.K_DEPTH, max_points=0, textured=False):
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    o = OracleTSDF(map_scale=[25.6, 25.6], K=K, is_global_map=True)
    g = TsdfHandle(o.N, o.Nz, K=K, is_global_map=True, max_points=max_points, texture_enabled=textured)
    if textured:
        o.set_color(True, True, None)
        g.set_color_intrinsics([1, 0, 0, 0, 1, 0, 0, 0, 1], True)
    return g, o


def check_counters(g, o):
    sg, so = g.stats(), o.stats()
    for k in COUNTERS:
        assert sg[k] == so[k], f"{k}: gpu {sg[k]} oracle {so[k]}"
    assert sg["err_flags"] == 0 and sg["n_rays"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("max_points", [0, CLEARING_MAX_POINTS])
@pytest.mark.parametrize("scene", sorted(SCENES))
def test_depth_scenes_match_oracle(scene, max_points):
    """Each scene from the identity pose and from a generic pose, two launches on one handle."""
    g, o = pair(max_points=max_points)
    d = SCENES[scene]()
    for R, T in POSES:
        g.integrate_depth(d, R[None], T[None])
        o.integrate_depth(R, T, d)
    check_counters(g, o)
    compare_voxels(g.gather(), o.gather(), 1e-4)


@pytest.mark.gpu
def test_other_camera_matches_oracle():
    """Another camera's focal lengths (their own reciprocals in the unprojection)."""
    g, o = pair(K=K_OTHER)
    R, T = POSES[1]
    d = syn.scene_room()
    g.integrate_depth(d, R[None], T[None])
    o.integrate_depth(R, T, d)
    check_counters(g, o)
    compare_voxels(g.gather(), o.gather(), 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("max_points", [0, CLEARING_MAX_POINTS])
def test_points_match_oracle(max_points):
    """Point clouds: dense clusters (many points of a CTA in one bucket) and scattered points, generic pose."""
    g, o = pair(max_points=max_points)
    rng = np.random.default_rng(3)
    xyz = rng.normal(size=(60000, 3))
    xyz = xyz / np.linalg.norm(xyz, axis=1, keepdims=True) * rng.uniform(0.5, 9.0, size=(60000, 1))
    xyz[:20000] = np.repeat(xyz[:200], 100, axis=0) + rng.uniform(-0.01, 0.01, size=(20000, 3))
    xyz = xyz.astype(np.float32)
    for R, T in POSES:
        g.integrate_points(xyz, R, T)
        o.integrate_points(R, T, xyz)
    check_counters(g, o)
    compare_voxels(g.gather(), o.gather(), 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("max_points", [0, CLEARING_MAX_POINTS])
def test_textured_depth_and_points_match_oracle(max_points):
    """A textured handle: a textured depth frame, a coloured point cloud and an untextured frame; colours exact."""
    g, o = pair(max_points=max_points, textured=True)
    R, T = POSES[1]
    d, tex = syn.scene_room(), syn.texture_gradient(4)
    g.integrate_depth(d, R[None], T[None], texture=tex[None])
    o.integrate_depth_tex(R, T, d, tex)
    rng = np.random.default_rng(9)
    xyz = (rng.normal(size=(30000, 3)) * 2.0).astype(np.float32)
    rgb = rng.integers(1, 256, size=(30000, 3), dtype=np.uint8)
    g.integrate_points(xyz, np.eye(3), np.zeros(3), rgb=rgb)
    o.integrate_points_rgb(np.eye(3), np.zeros(3), xyz, rgb)
    d2 = syn.scene_sphere(4.0)
    g.integrate_depth(d2, R[None], T[None])
    o.integrate_depth(R, T, d2)
    check_counters(g, o)
    gi, gt, gw, go, gc = g.gather(color=True)
    compare_voxels((gi, gt, gw, go), o.gather(), 1e-4)
    oi = o.gather()[0]
    gc, oc = gc[key_sort(gi)], o.gather_color()[key_sort(oi)]
    fin = np.isfinite(oc).all(1)
    assert np.array_equal(np.isfinite(gc).all(1), fin)
    assert np.array_equal(gc[fin], oc[fin]), "voxel colours differ"
    assert (oc[fin] > 0).any()
