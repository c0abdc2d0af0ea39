"""The numpy reference of the incremental global fusion (tests/fuse_update_reference.py) on hand-worked cases, and held
to the CPU oracle's fuse_from on the two-submap sphere scene of test_gpu_tsdf.py::test_submap_fusion."""
import numpy as np

from fuse_update_reference import fuse_reference
from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

VS = 0.25  # exact in binary: hand-worked placements stay exact
N, NZ = 64, 64
I3 = np.eye(3)


def part(idx, tsdf, w, occ, T=(0.0, 0.0, 0.0), R=I3, sign=1, color=None):
    idx = np.asarray(idx, np.int32).reshape(-1, 3)
    n = idx.shape[0]
    p = dict(idx=idx, tsdf=np.broadcast_to(np.float32(tsdf), (n,)).copy() if np.ndim(tsdf) == 0 else np.asarray(tsdf, np.float32),
             w=np.broadcast_to(np.float32(w), (n,)).copy() if np.ndim(w) == 0 else np.asarray(w, np.float32),
             occ=np.broadcast_to(np.int64(occ), (n,)).copy() if np.ndim(occ) == 0 else np.asarray(occ, np.int64),
             R=np.asarray(R, np.float32), T=np.asarray(T, np.float32), sign=sign)
    if color is not None:
        p["color"] = np.asarray(color, np.float32).reshape(n, 3)
    return p


def test_integer_offset_splats_zero_weights():
    # g lands on a grid point: every upper corner is one voxel away along some axis, so its weight is 0 (k_fuse's
    # quirk of skipping c = 0): 7 voxels observed with W = 0 and T = 0 / 0
    r = fuse_reference([part([[1, 2, 3]], 0.1, 2.0, 1, T=(2 * VS, -VS, 0.0))], N, NZ, VS)
    assert r["idx"].tolist() == sorted([[3 + a, 1 + b, 3 + c] for a in (0, 1) for b in (0, 1) for c in (0, 1) if a or b or c])
    assert np.all(r["w"] == 0.0) and np.all(np.isnan(r["tsdf"])) and np.all(r["occ"] == 1)
    assert r["splatted"] == 1 and r["skipped"] == 0


def test_half_voxel_offset_weights_are_one_eighth():
    r = fuse_reference([part([[0, 0, 0]], 0.1, 2.0, -1, T=(VS / 2, VS / 2, VS / 2))], N, NZ, VS)
    assert r["idx"].shape[0] == 7 and [0, 0, 0] not in r["idx"].tolist()
    w = np.float32(2.0) * np.float32(0.125)
    assert np.all(r["w"] == w)                                  # 0.25 * 2^24 is an integer: W is exact
    qwt = np.rint(np.float64(w * np.float32(0.1)) * 2.0 ** 24)
    assert np.all(r["tsdf"] == np.float32(qwt / (0.25 * 2.0 ** 24)))
    assert np.all(r["occ"] == -1)


def test_weight_that_quantises_to_zero_gives_nan():
    r = fuse_reference([part([[0, 0, 0]], 0.1, 1e-10, 0, T=(VS / 2, VS / 2, VS / 2))], N, NZ, VS)
    assert r["idx"].shape[0] == 7 and np.all(r["w"] == 0.0) and np.all(np.isnan(r["tsdf"]))


def test_occ_saturates_once_on_the_total():
    # 100 + 100 would saturate a running i8 sum at 127 (then 127 - 100 = 27); the total is 100
    ps = [part([[0, 0, 0]], 0.1, 1.0, o, T=(VS / 2, VS / 2, VS / 2)) for o in (100, 100, -100)]
    r = fuse_reference(ps, N, NZ, VS)
    assert np.all(r["occ"] == 100)
    ps = [part([[0, 0, 0]], 0.1, 1.0, 100, T=(VS / 2, VS / 2, VS / 2)) for _ in range(3)]
    assert np.all(fuse_reference(ps, N, NZ, VS)["occ"] == 127)


def test_non_finite_source_voxel_is_skipped():
    idx = [[0, 0, 0], [10, 10, 10], [20, 20, 20], [-10, 5, 5]]
    r = fuse_reference([part(idx, [0.1, np.nan, 0.2, 0.1], [1.0, 1.0, 1.0, 1e8], 0, T=(VS / 2, VS / 2, VS / 2))], N, NZ, VS)
    assert r["skipped"] == 2 and r["splatted"] == 2                # NaN T, and W * wt >= 2^23
    near = [tuple(v) for v in r["idx"].tolist()]
    assert all(max(abs(a - b) for a, b in zip(v, (10, 10, 10))) > 1 for v in near)
    assert all(max(abs(a - b) for a, b in zip(v, (-10, 5, 5))) > 1 for v in near)
    assert r["idx"].shape[0] == 14


def test_add_then_subtract_leaves_nothing():
    rng = np.random.default_rng(3)
    idx = rng.integers(-20, 20, (500, 3))
    R = rot_xyz(0.1, -0.2, 0.3)
    p = part(idx, rng.normal(0, 0.1, 500), rng.uniform(0.5, 3.0, 500), rng.integers(-3, 4, 500), T=(0.13, -0.07, 0.31), R=R)
    q = dict(p, sign=-1)
    r = fuse_reference([p, q], N, NZ, VS)
    assert r["idx"].shape[0] == 0 and r["splatted"] == 1000
    keep = fuse_reference([p], N, NZ, VS)
    both = fuse_reference([p, dict(p, T=np.float32([0.2, 0.0, 0.0])), dict(p, T=np.float32([0.2, 0.0, 0.0]), sign=-1)], N, NZ, VS)
    for k in ("idx", "w", "occ"):
        assert np.array_equal(keep[k], both[k])
    assert np.array_equal(np.isnan(keep["tsdf"]), np.isnan(both["tsdf"]))


def test_matches_oracle_fusion_on_sphere_submaps(oracle_lib):
    """Same voxel set as the oracle's fuse_from; W within test_submap_fusion's TOL, and T within it where the oracle is
    finite and the voxel's weight is >= 1e-3.  Lighter voxels carry the quantisation error of the contract: each term is
    rounded to 2^-24, so T = S_wT / S_w moves by at most count * 2^-25 * (1 + |T|) / W (count <= 64 per submap)."""
    OracleTSDF = oracle_lib.OracleTSDF
    d = syn.scene_sphere(2.0, 240, 320)
    K = [syn.FX / 2, 0, syn.CX / 2, 0, syn.FY / 2, syn.CY / 2, 0, 0, 1]
    so = OracleTSDF(map_scale=[6.4, 6.4], K=K, max_ray_length=3.0)
    go = OracleTSDF(map_scale=[12.8, 12.8], is_global_map=True)
    poses = {0: (rot_xyz(0.1, 0.2, 0.3), np.array([0.5, 0.1, -0.2])), 1: (rot_xyz(-0.3, 0.1, 1.0), np.array([-0.4, 0.6, 0.3]))}
    parts = []
    for s, (R, T) in poses.items():
        so.integrate_depth(np.eye(3), np.zeros(3), d, submap=s)
        go.set_submap_pose(s, R, T)
    for s, (R, T) in poses.items():
        idx, t, w, occ = so.gather(s)
        parts.append(part(idx, t, w, occ, T=np.float32(T), R=np.float32(R)))
    go.fuse_from(so)
    oi, ot, ow, _ = as_dict_rows(*go.gather())
    r = fuse_reference(parts, go.N, go.Nz, np.float32(0.05))
    assert np.array_equal(r["idx"], oi.astype(np.int32))
    fin = np.isfinite(ot)
    assert fin.mean() > 0.99
    assert np.all(np.isfinite(r["tsdf"][fin]))
    err = np.abs(r["tsdf"] - ot)
    heavy = fin & (ow >= 1e-3)
    assert heavy.sum() > 0.99 * fin.sum()
    assert err[heavy].max() <= 1e-4
    bound = 128 * 2.0 ** -25 * (1.0 + np.abs(ot[fin])) / ow[fin]
    assert np.all(err[fin] <= 1e-4 + bound)
    assert np.all(np.abs(r["w"][fin] - ow[fin]) <= 1e-4 * np.maximum(1.0, ow[fin]))
