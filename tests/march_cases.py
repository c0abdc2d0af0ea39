"""Seeded edge-case point clouds for the ray-march audit (tests/test_march_reference_cpu.py, tests/test_gpu_march_audit.py).

Every cloud meets the input contract of march_reference: points on the 2^-20 m grid, one point per bucket, R = I.  Each
point also has a colour (a seeded draw from a small palette of distinct colours), for the textured march."""
import numpy as np

from march_reference import round_half_away

GRID = 2.0 ** -20


def snap(p):
    return (np.round(np.asarray(p, np.float64) / GRID) * GRID).astype(np.float32)


def one_per_bucket(p, vs):
    """Drop every point whose bucket (round(p/vs), f32 quotient) an earlier point already holds."""
    p = np.asarray(p, np.float32)
    key = round_half_away(p / np.float32(vs))
    _, first = np.unique(key, axis=0, return_index=True)
    return np.ascontiguousarray(p[np.sort(first)])


def on_sphere(d, r):
    """Grid points along directions d whose f32 norm ((x*x + y*y) + z*z, sqrtf) is exactly r, so that every ray of
    the cloud has the power-of-two weight 1/r^2 when r is a power of two.  Components that are zero stay zero
    (signs kept, -0.0 included); directions without a hit within +-3 grid steps per axis are dropped."""
    d = np.asarray(d, np.float64)
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    base = snap(d * r).astype(np.float64)
    off = np.stack(np.meshgrid(*[np.arange(-3, 4)] * 3, indexing="ij"), -1).reshape(-1, 3) * GRID
    cand = (base[:, None, :] + off[None]).astype(np.float32)
    cand = np.where(d[:, None, :] == 0, base[:, None, :].astype(np.float32), cand)  # base keeps the sign of a zero
    L = np.sqrt((cand[..., 0] * cand[..., 0] + cand[..., 1] * cand[..., 1]) + cand[..., 2] * cand[..., 2])
    hit = L == np.float32(r)
    ok = hit.any(1)
    return cand[ok, np.argmax(hit[ok], 1)]


def _dirs(rng, n, axis, half_angle):
    """n random unit directions within half_angle (rad) of axis."""
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    v = rng.normal(size=(n, 3))
    v -= (v @ axis)[:, None] * axis
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    t = np.arccos(rng.uniform(np.cos(half_angle), 1.0, n))
    return np.cos(t)[:, None] * axis + np.sin(t)[:, None] * v


def hot_bundle(rng):
    """>= 20 000 rays in a 25 degree cone from a sensor in the middle of a block: every ray crosses the voxels next to
    the sensor, so the origin block gets several work items and its hottest voxels thousands of samples per item."""
    vs = 0.05
    d = _dirs(rng, 40000, [1.0, 0.3, 0.2], np.radians(25.0))
    p = one_per_bucket(snap(d * rng.uniform(4.0, 7.0, (d.shape[0], 1))), vs)  # sum w ~ 850 at the hottest voxel: unclamped
    return dict(pts=p, T=np.float32([7.3, 7.6, 8.2]) * np.float32(vs), vs=vs, N=256, Nz=128)


def ties_and_axes(rng):
    """vs = 1/16 m, sensor at T/vs = (-0.5, 15.5, -16.5): exact .5 ties in every coordinate, on block edges and corners,
    next to negative block coordinates.  Rays along the axes (zero components of both signs), in the coordinate planes,
    along block edge and corner diagonals, and in random directions - all with |p| = 4 m exactly (w = 1/16)."""
    vs = 0.0625
    ax = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float64)
    ax = ax * np.where(rng.random(ax.shape) < 0.5, 1.0, -1.0) ** (ax == 0)  # -0.0 in some zero components
    diag = np.array([[a, b, c] for a in (-1, 1) for b in (-1, 1) for c in (-1, 1)], np.float64)
    edge = np.array([[a, b, 0] for a in (-1, 1) for b in (-1, 1)] + [[a, 0, b] for a in (-1, 1) for b in (-1, 1)]
                    + [[0, a, b] for a in (-1, 1) for b in (-1, 1)], np.float64)
    plane = rng.normal(size=(600, 3))
    plane[np.arange(600), rng.integers(0, 3, 600)] = 0.0
    plane[:300] *= np.where(plane[:300] == 0, -1.0, 1.0)  # -0.0
    d = np.concatenate([ax, diag, edge, plane, rng.normal(size=(3000, 3))])
    p = one_per_bucket(on_sphere(d, 4.0), vs)
    return dict(pts=p, T=np.float32([-0.5, 15.5, -16.5]) * np.float32(vs), vs=vs, N=256, Nz=128, pow2=True)


def short_rays(rng):
    """|p| in [0.3, 0.45] m < internal_voxels * vs: the scale's n*vs - L branch sets the launch's fixed point."""
    vs = 0.05
    d = rng.normal(size=(3000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = one_per_bucket(snap(d * rng.uniform(0.3, 0.45, (3000, 1))), vs)
    return dict(pts=p, T=np.float32([0.013, -0.021, 0.004]), vs=vs, N=128, Nz=128)


def anisotropic(rng):
    """N = 200, Nz = 70 (neither a multiple of 16): rays leave the volume and end in blocks cut by its boundary."""
    vs = 0.05
    d = rng.normal(size=(8000, 3))
    p = one_per_bucket(snap(d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(1.0, 7.0, (8000, 1))), vs)
    return dict(pts=p, T=np.float32([1.1, -0.7, 0.3]), vs=vs, N=200, Nz=70)


def tiny_weights(rng):
    """One launch with z ~ 0.31 m and z ~ 60 m (max_ray_length 64, vs 0.2): the far rays' weight is below MB_MIN_WQ
    fixed-point units and must take the f32 global reductions."""
    vs = 0.2
    dn = rng.normal(size=(400, 3))
    near = snap(dn / np.linalg.norm(dn, axis=1, keepdims=True) * rng.uniform(0.30, 0.32, (400, 1)))
    df = rng.normal(size=(6000, 3))
    far = snap(df / np.linalg.norm(df, axis=1, keepdims=True) * rng.uniform(59.0, 61.0, (6000, 1)))
    p = one_per_bucket(np.concatenate([near, far]), vs)
    return dict(pts=p, T=np.float32([0.37, -0.11, 0.05]), vs=vs, N=640, Nz=640, max_ray_length=64.0)


def fine_long(rng):
    """vs = 0.2 mm with a 12.5 m range (max_ray_length / vs = 62500 steps) in a 5 cm volume: points up to 0.75 m away
    (3750 voxels: the bucket key reaches 4095), so that most samples of a ray fall outside the volume."""
    vs = 0.0002
    d = rng.normal(size=(2000, 3))
    p = one_per_bucket(snap(d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.3, 0.75, (2000, 1))), vs)
    return dict(pts=p, T=np.float32([0.0013, -0.0021, 0.0004]), vs=vs, N=256, Nz=256, max_ray_length=12.5)


def long_range(rng):
    """20 000 rays in all directions at 55-60 m (vs 0.2, max_ray_length 64): w = 1/z^2 ~ 3e-4 for every ray, so the
    window next to the sensor holds thousands of tiny weights, where a fixed point too coarse for them shows.  The sensor
sits inside a block, away from its faces."""
    vs = 0.2
    d = rng.normal(size=(24000, 3))
    p = one_per_bucket(snap(d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(55.0, 60.0, (d.shape[0], 1))), vs)
    return dict(pts=p[:20000], T=np.float32([7.3, 7.6, 8.2]) * np.float32(vs), vs=vs, N=640, Nz=640, max_ray_length=64.0)


def near_sensor(rng):
    """Points 0.05-0.12 m from the sensor with internal_voxels 40 (vs 0.02): weights 70-400 (some rays w >= 120) and
    rays 0.8 m past their point, so that some samples have |w*ds| >= 120."""
    vs = 0.02
    d = rng.normal(size=(4000, 3))
    p = one_per_bucket(snap(d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.05, 0.12, (4000, 1))), vs)
    return dict(pts=p, T=np.float32([0.0031, -0.0047, 0.0013]), vs=vs, N=256, Nz=256, internal_voxels=40)


CASES = {"hot_bundle": hot_bundle, "ties_and_axes": ties_and_axes, "short_rays": short_rays, "anisotropic": anisotropic,
         "tiny_weights": tiny_weights, "fine_long": fine_long, "long_range": long_range, "near_sensor": near_sensor}
PALETTE = np.array([[230, 25, 75], [60, 180, 75], [255, 225, 25], [0, 130, 200], [245, 130, 48], [145, 30, 180],
                    [70, 240, 240], [240, 50, 230], [1, 1, 1], [255, 255, 255]], np.uint8)


def make_case(name, seed=0):
    c = dict(internal_voxels=10, max_ray_length=10.0, pow2=False)
    c.update(CASES[name](np.random.default_rng(seed)))
    c["rgb"] = PALETTE[np.random.default_rng([seed, 1]).integers(0, PALETTE.shape[0], c["pts"].shape[0])]
    return c


def reference_of(case, path="binned", seq=1):
    from march_reference import reference_march
    return reference_march(case["pts"], case["T"], case["vs"], case["N"], case["Nz"], case["internal_voxels"],
                           case["max_ray_length"], path=path, rgb=case["rgb"], seq=seq)
