"""An analytic world for frame-tracking tests: a closed box room with three axis-aligned boxes inside, rendered exactly
(f64 ray casting) at any camera pose, so that every frame agrees with every other.

Frame convention: the camera's (x right, y down, z forward), the same as integrate_depth's R, T; a camera pose (R, t)
maps camera points into the world.  The room is x in [-3, 3], y in [-1.5, 1.5] (floor at y = +1.5), z in [-2.5, 2.5];
the boxes stand on the floor or against a wall at different heights and depths, so that the planes a view sees
constrain all six pose components.
"""
import numpy as np

from taichislam_b200 import synthetic as syn

ROOM = (np.array([-3.0, -1.5, -2.5]), np.array([3.0, 1.5, 2.5]))
BOXES = [(np.array([0.9, 0.6, 1.2]), np.array([2.0, 1.5, 2.5])),       # on the floor, in the far right corner
         (np.array([-2.3, -0.4, 0.4]), np.array([-1.5, 1.5, 1.4])),    # a tall one on the floor, left
         (np.array([-0.6, -1.5, 1.9]), np.array([0.4, -0.8, 2.5]))]    # hanging from the ceiling against the far wall
N_FRAMES = 40


def rot(axis, deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    x, y, z = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.array([[c + x * x * (1 - c), x * y * (1 - c) - z * s, x * z * (1 - c) + y * s],
                     [y * x * (1 - c) + z * s, c + y * y * (1 - c), y * z * (1 - c) - x * s],
                     [z * x * (1 - c) - y * s, z * y * (1 - c) + x * s, c + z * z * (1 - c)]])


def pose(k):
    """Camera pose of frame k of the 40-frame trajectory: a slow arc through the room's middle, panning from the left
    wall to the right one (2.5 cm, about 1.5 degrees of yaw and a little pitch per frame)."""
    u = k / (N_FRAMES - 1)
    R = rot([0, 1, 0], -30.0 + 60.0 * u) @ rot([1, 0, 0], -8.0 + 6.0 * np.sin(np.pi * u))
    t = np.array([-0.5 + 1.0 * u, 0.1 * np.sin(2.0 * np.pi * u), -1.2 + 0.4 * u])
    return R, t


def _rays(h, w, K):
    fx, cx, fy, cy = K[0], K[2], K[4], K[5]
    i = np.arange(w, dtype=np.float64)[None, :]
    j = np.arange(h, dtype=np.float64)[:, None]
    d = np.stack(np.broadcast_arrays((i - cx) / fx, (j - cy) / fy, np.ones((h, w))), -1)
    return d.reshape(-1, 3)  # z = 1: the ray parameter is the depth


def _slab(o, d, lo, hi):
    """(t_near, t_far) of the rays o + t d through the box [lo, hi]."""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        t0, t1 = (lo - o) * inv, (hi - o) * inv
    tn = np.nanmax(np.minimum(t0, t1), 1)
    tf = np.nanmin(np.maximum(t0, t1), 1)
    return tn, tf


def depth_m(R, t, h=syn.H, w=syn.W, K=syn.K_DEPTH):
    """Exact depth (m, f64 [h,w]) of the world seen from camera pose (R, t)."""
    d = _rays(h, w, K) @ np.asarray(R, np.float64).T
    o = np.asarray(t, np.float64)[None, :]
    z = _slab(o, d, *ROOM)[1]                  # the room is seen from inside: its far side
    for lo, hi in BOXES:
        tn, tf = _slab(o, d, lo, hi)
        hit = (tn <= tf) & (tn > 0.0)
        z = np.where(hit & (tn < z), tn, z)
    return z.reshape(h, w)


def render(R, t, seed=0, dropout=0.02, h=syn.H, w=syn.W, K=syn.K_DEPTH):
    """uint16 mm depth frame at camera pose (R, t): the exact depth rounded to mm, seeded dropouts (0)."""
    z = depth_m(R, t, h, w, K)
    d = np.round(z * 1000.0)
    d[np.random.default_rng(seed).random((h, w)) < dropout] = 0
    return np.clip(d, 0, 65535).astype(np.uint16)


def cloud(R, t, seed=0, step=4, n_zero=300):
    """The point-cloud variant: the frame's sampled pixels (every step-th) as f32 sensor-frame points (x, y, z) =
    depth * ray, with n_zero (0, 0, 0) points (a driver's missing returns) scattered through it."""
    h, w = syn.H, syn.W
    z = depth_m(R, t)[::step, ::step]
    ray = _rays(h, w, syn.K_DEPTH).reshape(h, w, 3)[::step, ::step]
    p = (ray * z[..., None]).reshape(-1, 3)
    rng = np.random.default_rng(seed)
    at = np.sort(rng.choice(p.shape[0], n_zero, replace=False))
    p[at] = 0.0
    return np.ascontiguousarray(p.astype(np.float32))


def perturb(R, t, rng, dt=0.05, deg=3.0):
    """A left perturbation of (R, t) by a random translation of length dt and rotation of deg degrees."""
    v = rng.normal(size=3)
    ax = rng.normal(size=3)
    dR = rot(ax, deg)
    return dR @ R, dR @ t + dt * v / np.linalg.norm(v)


def odometry(seed=11, sigma_t=0.005, sigma_deg=0.2):
    """Noisy frame-to-frame deltas of the trajectory: delta_k = T_{k-1}^-1 T_k composed with a seeded error of about
    sigma_t m and sigma_deg degrees.  -> list of (dR, dt) for k = 1 .. N_FRAMES - 1."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(1, N_FRAMES):
        (Ra, ta), (Rb, tb) = pose(k - 1), pose(k)
        dR, dt = Ra.T @ Rb, Ra.T @ (tb - ta)
        E = rot(rng.normal(size=3), sigma_deg * rng.normal())
        out.append((E @ dR, E @ dt + sigma_t * rng.normal(size=3)))
    return out


def compose(R, t, dR, dt):
    return R @ dR, R @ dt + t
