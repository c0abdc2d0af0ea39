"""Seam-crossing spiral: an analytic TSDF whose ESDF wave must cross one tile cut k times.

A one-voxel-thin corridor of observed voxels in a plane z = Z, surrounded by unobserved space.  It runs along x across
the cut between voxel x = -1 and x = 0 (block -1 | block 0, the x cut of SPIRAL_CUTS), turns along y on alternate
sides, and crosses back, k times in all.  The turns lie in blocks -2 and 1, outside the one-block ghost layer of
either tile, so a rank cannot follow the corridor through its ghosts alone.  Parallel runs are DY voxels apart, so no
26-neighbour step joins them: the only way along is the corridor.  The first voxel is a fixed-band seed (|TSDF| < voxel_scale); every other corridor
voxel is outside the band, so its ESDF is the seed's plus the corridor length to it.  A tiled ESDF with the cut
between two ranks needs one exchange round per crossing (tests/test_esdf_spiral_cpu.py pins the crossings on the
oracle)."""
import numpy as np

VS = 0.05
MAP_SCALE = [12.8, 12.8]            # N = Nz = 256: blocks -8 .. 7 on every axis
MAX_RAY = 20.0                      # far value of the ESDF seeds: well above the corridor length
SPIRAL_TILES = (2, 1, 1)
SPIRAL_CUTS = ([-8, 0, 8], [-8, 8], [-8, 8])
Z, X0, X1, Y0, DY = 40, -20, 19, -20, 4


def spiral_path(k):
    """Corridor voxels (int32 [n,3]) in path order from the seed; crosses x = -1 | 0 k times."""
    pts = []
    y, xa, xb = Y0, X0, X1
    for c in range(k):
        step = 1 if xb > xa else -1
        for x in range(xa, xb + step, step):
            if not pts or pts[-1] != (x, y, Z):
                pts.append((x, y, Z))
        if c < k - 1:
            for yy in range(y + 1, y + DY + 1):
                pts.append((xb, yy, Z))
            y += DY
        xa, xb = xb, xa
    return np.asarray(pts, np.int32)


def spiral_rows(k, sign=1.0):
    """(idx, tsdf, w, occ) rows of the corridor: the seed carries sign * 0.4 * VS, the rest sign * 10 * VS."""
    idx = spiral_path(k)
    t = np.full(len(idx), sign * 10 * VS, np.float32)
    t[0] = np.float32(sign * 0.4 * VS)
    return idx, t, np.ones(len(idx), np.float32), np.zeros(len(idx), np.int8)


def crossings(idx):
    """Steps of the path that cross the x cut between voxel -1 and voxel 0."""
    side = idx[:, 0] < 0
    return int(np.count_nonzero(side[1:] != side[:-1]))
