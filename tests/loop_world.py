"""A world for loop-detection tests: tests/track_world.py's box room, a trajectory that leaves the start and comes back,
and a second, different room at the same nominal coordinates.

Frames are track_world's: camera (x right, y down, z forward), world up = -y (pass up = (0, -1, 0)).  Submap s is made of
FRAMES consecutive frames; its base pose is its first camera pose.  Odometry drifts from submap DRIFT_FROM on: the stored
base poses and camera poses of those submaps are the true ones moved by DRIFT, a yaw about the world vertical and a
horizontal translation, so their local content is exact and only their place in the world is wrong.  Submap N_LOOP - 1
comes back to the start with a heading 15 degrees from submap 0's.  Submaps N_LOOP .. N_LOOP + 1 are in room B, a room of
another size with other boxes, placed at the same coordinates: every pair between the rooms is a false candidate.
"""
import numpy as np

import track_world as tw
from taichislam_b200 import synthetic as syn

UP = (0.0, -1.0, 0.0)
ROOM_A = (tw.ROOM, tw.BOXES)
ROOM_B = ((np.array([-2.2, -1.5, -3.5]), np.array([2.2, 1.5, 3.5])),
          [(np.array([-2.2, 0.3, -0.5]), np.array([-1.2, 1.5, 2.0])),    # a long low bench against the left wall
           (np.array([1.0, -1.5, -3.5]), np.array([2.2, 1.5, -2.6])),    # a full-height pillar in the near right corner
           (np.array([0.3, 0.9, 2.4]), np.array([1.4, 1.5, 3.5]))])      # a low box in the far right corner
FRAMES = 3
# (x, z, heading deg) of each submap's first camera: start, a circuit through the room, back at the start
LOOP = [(-0.5, -1.2, 0.0), (0.3, -0.6, 70.0), (0.6, 0.5, 160.0), (-0.3, 0.8, 230.0), (-0.9, -0.2, 300.0), (-0.35, -1.05, 15.0)]
N_LOOP = len(LOOP)
ROOM_B_SUBMAPS = [(-0.4, -1.0, 5.0), (0.2, 0.8, 180.0)]
DRIFT_FROM = 3
DRIFT_DEG, DRIFT_T = 25.0, np.array([0.9, 0.0, -0.6])


def yaw(deg):
    """Rotation by deg about the world vertical (heading grows from +z towards +x)."""
    return tw.rot([0, 1, 0], deg)


def drift():
    return yaw(DRIFT_DEG), DRIFT_T


def true_pose(s, f):
    """True camera pose of frame f of submap s (f = 0: the submap's base pose)."""
    x, z, h = (LOOP + ROOM_B_SUBMAPS)[s]
    R = yaw(h + 4.0 * f) @ tw.rot([1, 0, 0], -4.0)
    return R, np.array([x + 0.03 * f, 0.05 * np.sin(s + f), z + 0.02 * f])


def room_of(s):
    return ROOM_A if s < N_LOOP else ROOM_B


def odometry_pose(s, f):
    """The pose odometry reports: the true one, moved by the drift for submaps DRIFT_FROM .. N_LOOP - 1."""
    R, t = true_pose(s, f)
    if DRIFT_FROM <= s < N_LOOP:
        D, dt = drift()
        return D @ R, D @ t + dt
    return R, t


def relative(sq, sd):
    """True q-local -> d-local pose of two submaps (P_d^-1 P_q)."""
    Rq, tq = true_pose(sq, 0)
    Rd, td = true_pose(sd, 0)
    return Rd.T @ Rq, Rd.T @ (tq - td)


def depth_m(R, t, room, h=syn.H, w=syn.W, K=syn.K_DEPTH):
    walls, boxes = room
    d = tw._rays(h, w, K) @ np.asarray(R, np.float64).T
    o = np.asarray(t, np.float64)[None, :]
    z = tw._slab(o, d, *walls)[1]
    for lo, hi in boxes:
        tn, tf = tw._slab(o, d, lo, hi)
        hit = (tn <= tf) & (tn > 0.0)
        z = np.where(hit & (tn < z), tn, z)
    return z.reshape(h, w)


def render(s, f, seed=0, dropout=0.02):
    """uint16 mm depth frame f of submap s, seen from its true pose in its room."""
    z = depth_m(*true_pose(s, f), room_of(s))
    d = np.round(z * 1000.0)
    d[np.random.default_rng(1000 * s + f + seed).random(d.shape) < dropout] = 0
    return np.clip(d, 0, 65535).astype(np.uint16)


def n_submaps():
    return N_LOOP + len(ROOM_B_SUBMAPS)
