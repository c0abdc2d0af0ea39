"""The dirty rule of the incremental mesh (tests/mesh_dirty.py, DESIGN.md section 4) against the CPU oracle's marching
cubes, independently of the CUDA code: random perturbations of the golden crop of the reference's map (TSDF sign flips,
voxels becoming unobserved or observed, NaN, changes in all-positive free-space blocks) change the oracle's per-block
triangle lists only inside the rule's dirty set, and perturbations in free space more than one block from any negative
voxel mark nothing and change nothing."""
import os

import numpy as np
import pytest

import mesh_dirty as md
from oracle.oracle import OracleTSDF

HERE = os.path.dirname(os.path.abspath(__file__))


def load_crop():
    z = np.load(os.path.join(HERE, "golden", "ri_new_crop.npz"))
    c = {k: z[k] for k in z.files}
    idx = c["indices"].astype(np.int32)
    # free space far from the crop: two all-positive blocks (one full, one sparse), >= 3 blocks from any negative voxel
    rng = np.random.default_rng(7)
    g = np.stack(np.meshgrid(np.arange(16), np.arange(16), np.arange(16), indexing="ij"), -1).reshape(-1, 3)
    far_a = g + np.array([16 * 8, 16 * 2, 0])
    far_b = g[rng.random(len(g)) < 0.4] + np.array([16 * 8, 16 * 3, 16])
    free = np.concatenate([far_a, far_b]).astype(np.int32)
    tf = rng.uniform(0.05, 2.0, len(free)).astype(np.float32)
    return dict(vs=float(c["voxel_size"]), scale=list(c["map_scale"]),
                idx=np.concatenate([idx, free]), t=np.concatenate([c["TSDF"].astype(np.float32), tf]),
                w=np.concatenate([c["W_TSDF"].astype(np.float32), np.ones(len(free), np.float32)]),
                occ=np.concatenate([c["occupy"].astype(np.int8), np.zeros(len(free), np.int8)]),
                far=[(8, 2, 0), (8, 3, 1)])


def mesh(c, idx, t, w, occ, thres):
    m = OracleTSDF(map_scale=c["scale"], voxel_scale=c["vs"], num_voxel_per_blk_axis=16, is_global_map=True)
    m.scatter(0, idx, t, w, occ)
    n, v, nrm = m.marching_cubes(step=1, thres=thres, cap_tri=1 << 20)
    return md.triangles_per_block(idx, t, thres, v, nrm)


def blocks_of(idx):
    return {tuple(int(x) for x in b) for b in np.unique(md.block_of(idx), axis=0)}


def perturb(c, kind, rng, k=24):
    """A copy of the crop's voxels with k voxels perturbed, and the blocks those voxels lie in (the stamped blocks)."""
    idx, t, w, occ = c["idx"].copy(), c["t"].copy(), c["w"].copy(), c["occ"].copy()
    blk = md.block_of(idx)
    far = np.isin(blk[:, 0] * 10 ** 6 + blk[:, 1] * 10 ** 3 + blk[:, 2], [b[0] * 10 ** 6 + b[1] * 10 ** 3 + b[2] for b in c["far"]])
    near_surface = np.flatnonzero(~far & np.isfinite(t) & (np.abs(t) < 3 * c["vs"]))
    if kind == "sign":
        r = rng.choice(near_surface, k, replace=False)
        t[r] = -t[r]
    elif kind == "nan":
        r = rng.choice(near_surface, k, replace=False)
        t[r] = np.nan
    elif kind == "unobserve":  # observed -> unobserved: the rows go away
        r = rng.choice(near_surface, k, replace=False)
        keep = np.ones(len(idx), bool)
        keep[r] = False
        stamped = blocks_of(idx[r])
        return idx[keep], t[keep], w[keep], occ[keep], stamped
    elif kind == "observe":  # unobserved -> observed: new rows next to observed voxels, either sign
        have = {tuple(x) for x in idx}
        base = idx[rng.choice(near_surface, 4 * k, replace=False)]
        step = rng.integers(-1, 2, size=base.shape)
        new = np.array([x for x in {tuple(x) for x in base + step} if x not in have][:k], np.int32).reshape(-1, 3)
        nt = rng.uniform(-0.3, 0.3, len(new)).astype(np.float32)
        return (np.concatenate([idx, new]), np.concatenate([t, nt]), np.concatenate([w, np.ones(len(new), np.float32)]),
                np.concatenate([occ, np.zeros(len(new), np.int8)]), blocks_of(new))
    elif kind == "free_space":  # inside the far all-positive blocks: new positive values, NaN, unobserved, newly observed
        fr = np.flatnonzero(far)
        r = rng.choice(fr, 3 * k, replace=False)
        t[r[:k]] = rng.uniform(0.01, 3.0, k).astype(np.float32)
        t[r[k:2 * k]] = np.nan
        keep = np.ones(len(idx), bool)
        keep[r[2 * k:]] = False
        have = {tuple(x) for x in idx[keep]}
        g = np.stack(np.meshgrid(np.arange(16), np.arange(16), np.arange(16), indexing="ij"), -1).reshape(-1, 3)
        cand = g + 16 * np.array(c["far"][1])
        new = np.array([x for x in map(tuple, cand[rng.permutation(len(cand))]) if x not in have][:k], np.int32)
        stamped = blocks_of(np.concatenate([idx[r], new]))
        idx, t, w, occ = idx[keep], t[keep], w[keep], occ[keep]
        return (np.concatenate([idx, new]), np.concatenate([t, rng.uniform(0.01, 3.0, len(new)).astype(np.float32)]),
                np.concatenate([w, np.ones(len(new), np.float32)]), np.concatenate([occ, np.zeros(len(new), np.int8)]), stamped)
    return idx, t, w, occ, blocks_of(idx[r])


@pytest.fixture(scope="module")
def crop():
    c = load_crop()
    c["thres"] = 5 * c["vs"]
    c["mesh"] = mesh(c, c["idx"], c["t"], c["w"], c["occ"], c["thres"])
    c["neg"] = md.neg_blocks(c["idx"], c["t"])
    return c


def test_attribution_covers_the_oracle_mesh(crop):
    """Every oracle triangle is attributed to a cell (triangles_per_block asserts that the counts add up)."""
    assert sum(len(b) for b in crop["mesh"].values()) // 72 > 10000
    assert set(crop["far"]).isdisjoint(crop["mesh"]) and set(crop["far"]).isdisjoint(crop["neg"])
    for b in crop["far"]:
        assert all((b[0] + dx, b[1] + dy, b[2] + dz) not in crop["neg"]
                   for dx in range(-3, 4) for dy in range(-3, 4) for dz in range(-3, 4))


@pytest.mark.parametrize("kind", ["sign", "nan", "unobserve", "observe"])
def test_triangles_change_only_inside_the_dirty_set(crop, kind):
    rng = np.random.default_rng({"sign": 1, "nan": 2, "unobserve": 3, "observe": 4}[kind])
    n_changed = 0
    for trial in range(8):
        idx, t, w, occ, stamped = perturb(crop, kind, rng, k=24 if kind == "observe" else 6)
        after = mesh(crop, idx, t, w, occ, crop["thres"])
        before = crop["mesh"]
        changed = {b for b in set(before) | set(after) if before.get(b) != after.get(b)}
        blocks = blocks_of(crop["idx"]) | blocks_of(idx)
        d = md.dirty(stamped, crop["neg"], md.neg_blocks(idx, t), blocks)
        assert changed <= d, (kind, trial, sorted(changed - d)[:5])
        assert d <= md.touched(stamped, blocks) and len(d) < len(blocks)
        n_changed += len(changed)
    assert n_changed > 0, "the perturbations must change the mesh somewhere"


def test_free_space_far_from_negative_voxels_marks_nothing(crop):
    rng = np.random.default_rng(5)
    for trial in range(8):
        idx, t, w, occ, stamped = perturb(crop, "free_space", rng)
        assert stamped and stamped <= set(crop["far"])
        blocks = blocks_of(crop["idx"]) | blocks_of(idx)
        assert md.touched(stamped, blocks) >= stamped
        assert md.dirty(stamped, crop["neg"], md.neg_blocks(idx, t), blocks) == set()
        assert mesh(crop, idx, t, w, occ, crop["thres"]) == crop["mesh"]


def test_rule_on_hand_made_cases():
    """The corner case that makes B + {0,1}^3 necessary: a negative voxel at voxel (0,0,0) of block (1,1,1) is a corner of
    cell (15,15,15) of block (0,0,0); the negative voxel's own block being stamped marks the lower neighbour dirty."""
    blocks = {(0, 0, 0), (1, 1, 1), (-1, 0, 0), (3, 3, 3)}
    neg_now = md.neg_blocks(np.array([[16, 16, 16]]), np.array([-0.1], np.float32))
    assert neg_now == {(1, 1, 1)}
    assert md.dirty({(1, 1, 1)}, set(), neg_now, blocks) == {(0, 0, 0), (1, 1, 1)}
    # (-1,0,0) is touched only by a stamp at (0,0,0), and reads no negative voxel in (-1,0,0) + {0,1}^3 ... unless (0,0,0) has one
    assert md.dirty({(0, 0, 0)}, set(), set(), blocks) == set()
    assert md.dirty({(0, 0, 0)}, {(0, 0, 0)}, set(), blocks) == {(0, 0, 0), (-1, 0, 0)}
    # NaN and -0 are not negative
    assert md.neg_blocks(np.array([[0, 0, 0], [1, 0, 0]]), np.array([np.nan, -0.0], np.float32)) == set()
