"""The dirty rule of the incremental mesh (DESIGN.md section 4, tslam_mesh_update) stated in numpy, and a numpy
statement of which cells of marching cubes (step 1) emit how many triangles, to attribute the oracle's triangles to
cells.

Blocks are the library's 16^3 voxel blocks, keyed by (bx, by, bz) of one submap.  A block is STAMPED when a commit wrote
it since the last update.  neg(M) = block M holds an observed voxel with TSDF < 0 (NaN and -0 are not < 0).  A block B
is TOUCHED when a stamped block lies in its 27-neighbourhood, and DIRTY when it is touched and some block M of
B + {0,1}^3 has neg before or after the change.  Every block whose triangles can change is dirty."""
import os
import re

import numpy as np

B = 16
HERE = os.path.dirname(os.path.abspath(__file__))
# corner offsets V0..V7 (marching_cube_mesher.py:196-206)
GRID = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 1], [0, 1, 1]])


def block_of(idx):
    return np.floor_divide(np.asarray(idx, np.int64), B)


def neg_blocks(idx, tsdf):
    """{block}: blocks holding an observed voxel (a row of idx) with TSDF < 0."""
    t = np.asarray(tsdf, np.float32)
    return {tuple(int(x) for x in b) for b in block_of(np.asarray(idx)[t < 0])}


def touched(stamped, blocks):
    """Blocks of `blocks` with a stamped block in their 27-neighbourhood."""
    near = {(s[0] + dx, s[1] + dy, s[2] + dz) for s in stamped for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1)}
    return {b for b in blocks if b in near}


def dirty(stamped, neg_then, neg_now, blocks):
    """The blocks an update remeshes."""
    neg = set(neg_then) | set(neg_now)
    return {b for b in touched(stamped, blocks)
            if any((b[0] + dx, b[1] + dy, b[2] + dz) in neg for dx in (0, 1) for dy in (0, 1) for dz in (0, 1))}


def ntri_table():
    """Triangles per cube index, from the packed table of include/tslam_mc_cases.h."""
    txt = open(os.path.join(HERE, "..", "include", "tslam_mc_cases.h")).read()
    words = [int(w, 16) for w in re.findall(r"0x([0-9a-f]{16})ull", txt)]
    assert len(words) == 256
    return np.array([sum(((w >> (4 * q)) & 0xF) != 0xF for q in range(16)) // 3 for w in words], np.int64)


def cell_triangles(idx, tsdf, thres):
    """Cells (base voxels) that emit triangles at step 1 and how many: (cells int64[n,3], ntri int64[n]).  A cell emits
    when its base voxel is observed with TSDF < thres, all 8 corners are observed, and its cube index (corner bit set
    when TSDF < 0) has triangles (marching_cube_mesher.py:127-187)."""
    idx = np.asarray(idx, np.int64)
    t = np.asarray(tsdf, np.float32)
    lo = idx.min(0) - 1
    shape = tuple(idx.max(0) - lo + 3)
    T = np.zeros(shape, np.float32)
    O = np.zeros(shape, bool)
    p = idx - lo
    T[p[:, 0], p[:, 1], p[:, 2]] = t
    O[p[:, 0], p[:, 1], p[:, 2]] = True
    base = t < np.float32(thres)
    cube = np.zeros(len(idx), np.int64)
    allobs = np.ones(len(idx), bool)
    for c, (dx, dy, dz) in enumerate(GRID):
        q = p + (dx, dy, dz)
        allobs &= O[q[:, 0], q[:, 1], q[:, 2]]
        cube |= (T[q[:, 0], q[:, 1], q[:, 2]] < 0).astype(np.int64) << c
    n = np.where(base & allobs, ntri_table()[cube], 0)
    keep = n > 0
    return idx[keep], n[keep]


def oracle_order(cells, ob=8):
    """Order in which the CPU oracle (orc_mc2) visits cells: its ob^3 blocks sorted by key, voxels x-major inside."""
    cells = np.asarray(cells, np.int64)
    bk = np.floor_divide(cells, ob)
    lo = np.mod(cells, ob)
    o = (lo[:, 0] * ob + lo[:, 1]) * ob + lo[:, 2]
    return np.lexsort((o, bk[:, 2], bk[:, 1], bk[:, 0]))


def triangles_per_block(idx, tsdf, thres, verts, normals):
    """{16^3 block: bytes of its triangles (vertices + normals, cell order)} of an oracle mesh of the voxels idx/tsdf;
    each triangle attributed to its cell through the oracle's visiting order and the per-cell counts."""
    cells, n = cell_triangles(idx, tsdf, thres)
    order = oracle_order(cells)
    cells, n = cells[order], n[order]
    assert int(n.sum()) * 3 == len(verts), "the per-cell counts must add up to the oracle's mesh"
    first = np.concatenate([[0], np.cumsum(n)[:-1]])
    v = np.ascontiguousarray(verts, np.float32).view(np.int32).reshape(-1, 9)
    nr = np.ascontiguousarray(normals, np.float32).view(np.int32).reshape(-1, 9)
    out = {}
    blk = block_of(cells)
    for b in np.unique(blk, axis=0):
        rows = np.flatnonzero((blk == b).all(1))
        tri = np.concatenate([np.arange(first[r], first[r] + n[r]) for r in rows])
        out[tuple(int(x) for x in b)] = v[tri].tobytes() + nr[tri].tobytes()
    return out
