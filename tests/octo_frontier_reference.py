"""numpy/scipy statement of the frontiers of a log-odds Octomap (DESIGN.md section 7, "Frontiers of the log-odds
Octomap"; csrc/tslam_octo_frontier.cu).

Input: the known voxels of one submap as rows, `idx` int32[n,3] (centred cell indices) and `L` int32[n] (Q10 log-odds),
as OctoHandle.gather() returns them, plus l_occ and the volume N, Nz (cells i, j in [-N/2, N - N/2), k in
[-Nz/2, Nz - Nz/2)).  Nothing here knows about blocks.

    OCC = L > l_occ,  FREE = the other known voxels,  UNKNOWN = every in-volume cell without a row
    frontier voxel: a FREE cell with an in-volume UNKNOWN 6-neighbour (cells outside the volume do not count)
    clusters: the 26-connected components of the frontier voxels (scipy.ndimage.label, 3x3x3 structure)
    label: the smallest key ((i+hN)*N + (j+hN))*Nz + (k+hNz) of the cluster; clusters in ascending label order
    record (int64 x 16): label, n, sum i, sum j, sum k, min i, min j, min k, max i, max j, max k, faces (voxel /
        UNKNOWN in-volume 6-neighbour pairs), sum of the unit offsets towards those neighbours (x, y, z), 0
"""
import numpy as np
from scipy import ndimage

UNK, FREE, OCC, OUT = 0, 1, 2, 3
FACES = np.array([(-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1)], np.int64)


def key(idx, N, Nz):
    idx = np.asarray(idx, np.int64).reshape(-1, 3)
    hN, hNz = N // 2, Nz // 2
    return ((idx[:, 0] + hN) * N + (idx[:, 1] + hN)) * Nz + (idx[:, 2] + hNz)


def frontiers(idx, L, l_occ, N, Nz):
    """-> (fidx int32[m,3] in key order, cluster int32[m] (ordinal in rec), rec int64[c,16] in label order)"""
    idx = np.asarray(idx, np.int64).reshape(-1, 3)
    L = np.asarray(L, np.int64).reshape(-1)
    empty = (np.zeros((0, 3), np.int32), np.zeros(0, np.int32), np.zeros((0, 16), np.int64))
    if idx.shape[0] == 0:
        return empty
    lo_v = np.array([-(N // 2), -(N // 2), -(Nz // 2)], np.int64)
    hi_v = np.array([N - N // 2, N - N // 2, Nz - Nz // 2], np.int64) - 1
    lo = np.maximum(idx.min(0) - 1, lo_v)              # the known cells and their neighbours, clipped to the volume
    hi = np.minimum(idx.max(0) + 1, hi_v)
    shape = tuple(int(v) for v in hi - lo + 3)         # one more layer of OUT around the box
    cls = np.full(shape, OUT, np.uint8)
    cls[1:-1, 1:-1, 1:-1] = UNK
    p = idx - lo + 1
    cls[p[:, 0], p[:, 1], p[:, 2]] = np.where(L > int(l_occ), OCC, FREE)
    faces = np.zeros(cls.shape, np.int8)
    dirs = np.zeros(cls.shape + (3,), np.int8)
    for f in FACES:
        nb = np.roll(cls, shift=tuple(int(-v) for v in f), axis=(0, 1, 2))   # nb[c] = cls[c + f]
        u = nb == UNK
        faces += u
        for a in range(3):
            if f[a]:
                dirs[..., a] += u.astype(np.int8) * np.int8(f[a])
    front = (cls == FREE) & (faces > 0)
    front[0, :, :] = front[-1, :, :] = front[:, 0, :] = front[:, -1, :] = front[:, :, 0] = front[:, :, -1] = False
    lab, nlab = ndimage.label(front, structure=np.ones((3, 3, 3), bool))
    pos = np.argwhere(front)
    if pos.shape[0] == 0:
        return empty
    fidx = pos.astype(np.int64) + lo - 1
    comp = lab[pos[:, 0], pos[:, 1], pos[:, 2]] - 1
    k = key(fidx, N, Nz)
    label = np.full(nlab, np.iinfo(np.int64).max, np.int64)
    np.minimum.at(label, comp, k)
    order = np.argsort(label, kind="stable")
    ordinal = np.empty(nlab, np.int64)
    ordinal[order] = np.arange(nlab)
    c = ordinal[comp]
    rec = np.zeros((nlab, 16), np.int64)
    rec[:, 0] = label[order]
    np.add.at(rec[:, 1], c, 1)
    for a in range(3):
        np.add.at(rec[:, 2 + a], c, fidx[:, a])
        rec[:, 5 + a] = np.iinfo(np.int64).max
        rec[:, 8 + a] = np.iinfo(np.int64).min
        np.minimum.at(rec[:, 5 + a], c, fidx[:, a])
        np.maximum.at(rec[:, 8 + a], c, fidx[:, a])
    f_ = faces[pos[:, 0], pos[:, 1], pos[:, 2]].astype(np.int64)
    d_ = dirs[pos[:, 0], pos[:, 1], pos[:, 2]].astype(np.int64)
    np.add.at(rec[:, 11], c, f_)
    for a in range(3):
        np.add.at(rec[:, 12 + a], c, d_[:, a])
    o = np.argsort(k, kind="stable")
    return fidx[o].astype(np.int32), c[o].astype(np.int32), rec
