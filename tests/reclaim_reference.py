"""numpy statement of tslam_tsdf_reclaim's selection and compaction (include/tslam.h, DESIGN.md section 7,
"Reclaiming pool blocks").

    select(keys, empty, rules, mask, center, radius, vs) -> keep flags per pool slot
    compact(keep) -> (n_keep, pairs (hole, mover), new_order: old slot of each new slot)
    reclaim(...)  -> keep, new_order, stats6

keys: int[n, 4] rows (submap, bx, by, bz) in slot order (TsdfHandle.block_keys); empty: bool[n] per slot.
"""
import numpy as np

ALL, EMPTY, OUTSIDE = 1, 2, 4


def axis_d2(c, b, vs):
    """Squared f64 distance of c to the span of the f32 voxel positions (float)(16 b + t) * vs, t = 0 .. 15."""
    b = np.asarray(b, np.int64)
    vs32 = np.float32(vs)
    lo = ((b * 16).astype(np.float32) * vs32).astype(np.float64)
    hi = ((b * 16 + 15).astype(np.float32) * vs32).astype(np.float64)
    q = np.minimum(np.maximum(np.float64(c), lo), hi)
    d = np.float64(c) - q
    return d * d


def outside(keys, center, radius, vs):
    keys = np.asarray(keys, np.int64).reshape(-1, 4)
    c = np.asarray(center, np.float64).reshape(3)
    d2 = (axis_d2(c[0], keys[:, 1], vs) + axis_d2(c[1], keys[:, 2], vs)) + axis_d2(c[2], keys[:, 3], vs)
    return d2 > np.float64(radius) * np.float64(radius)


def candidates(keys, mask):
    keys = np.asarray(keys, np.int64).reshape(-1, 4)
    if mask is None:
        return np.ones(keys.shape[0], bool)
    return np.asarray(mask).astype(bool)[keys[:, 0]]


def select(keys, empty, rules, mask=None, center=None, radius=None, vs=0.05):
    keys = np.asarray(keys, np.int64).reshape(-1, 4)
    empty = np.asarray(empty, bool).reshape(-1)
    cand = candidates(keys, mask)
    drop = np.zeros(keys.shape[0], bool)
    if rules & ALL:
        drop |= True
    if rules & EMPTY:
        drop |= empty
    if rules & OUTSIDE:
        drop |= outside(keys, center, radius, vs)
    return ~(cand & drop)


def compact(keep):
    """-> n_keep, pairs int[m, 2] (hole, mover), new_order int[n_keep] = old slot now at each slot."""
    keep = np.asarray(keep, bool).reshape(-1)
    n_keep = int(keep.sum())
    slots = np.arange(keep.shape[0])
    holes = slots[:n_keep][~keep[:n_keep]]
    movers = slots[n_keep:][keep[n_keep:]]
    assert holes.shape == movers.shape
    order = slots[:n_keep].copy()
    order[holes] = movers
    return n_keep, np.stack([holes, movers], 1).reshape(-1, 2), order


def reclaim(keys, empty, rules, mask=None, center=None, radius=None, vs=0.05):
    """-> keep, new_order (old slot of each new slot), stats6 as the C entry reports them."""
    keys = np.asarray(keys, np.int64).reshape(-1, 4)
    empty = np.asarray(empty, bool).reshape(-1)
    keep = select(keys, empty, rules, mask, center, radius, vs)
    n_keep, pairs, order = compact(keep)
    n = keys.shape[0]
    if n_keep == n:
        order = np.arange(n)
    cand = candidates(keys, mask)
    st = np.array([n, int(cand.sum()), n - n_keep, int((~keep & ~empty).sum()), pairs.shape[0], n_keep], np.int64)
    return keep, order, st
