"""The seam-crossing spiral (tests/esdf_spiral.py) pinned on the CPU oracle: its ESDF wave really travels the whole
corridor, crossing the tile cut k times, so the exchange rounds the GPU test demands rest on a checked fact."""
import numpy as np
import pytest

import esdf_spiral as sp


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_spiral_wave_crosses_the_cut_k_times(oracle_lib, sign):
    from oracle.oracle import OracleTSDF
    k = 4
    idx, t, w, occ = sp.spiral_rows(k, sign)
    assert sp.crossings(idx) == k
    assert len(np.unique(idx, axis=0)) == len(idx)
    # no shortcut: two corridor voxels are 26-neighbours only when they are consecutive on the path (or meet at a turn)
    d = np.abs(idx[:, None, :] - idx[None, :, :]).max(axis=2)
    near = np.argwhere(d == 1)
    assert np.all(np.abs(near[:, 0] - near[:, 1]) <= 2)
    o = OracleTSDF(map_scale=sp.MAP_SCALE, voxel_scale=sp.VS, max_ray_length=sp.MAX_RAY, is_global_map=True)
    o.scatter(0, idx, t, w, occ)
    o.esdf_update()
    ei, ee = o.esdf_gather()
    assert len(ei) == len(idx)
    order = {tuple(r): i for i, r in enumerate(idx)}
    e = np.empty(len(idx), np.float32)
    for r, v in zip(ei, ee):
        e[order[tuple(r)]] = v
    # the wave leaves the seed and grows strictly along the corridor: every crossing carries it on
    assert e[0] == t[0]
    steps = np.diff(sign * e)
    assert np.all(steps > 0), steps
    assert np.all(sign * e < sp.MAX_RAY)  # no voxel is left at its far seed
    # each step adds one edge cost: vs along a run, vs * sqrt(2) at most where the corridor turns
    assert np.all(steps <= np.float32(np.sqrt(2.0) * sp.VS) + 1e-6)
