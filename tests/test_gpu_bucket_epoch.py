"""The per-frame bucket grid is never cleared between launches: its index entries carry a launch epoch, and a record is
stored whole by the lane that opens its bucket.  A handle whose record slots leave too few bits for the epoch
(max_points >= 2^21) runs in clearing mode instead.  These tests run the same launches through both modes - across
epoch wraps, errors, point clouds and textured frames - and against the CPU oracle; plus a CPU test of the bounds that
size the packed record and index fields (csrc/tslam_bucket.cuh)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from taichislam_b200 import synthetic as syn
from util import compare_voxels, key_sort, rot_xyz

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "taichislam_b200", "csrc")
CLEARING_MAX_POINTS = 1 << 21  # 22 slot bits: 3 left for the epoch, fewer than the 4 the epoch mode needs
EPOCHS_DEFAULT = 15            # default handle: max_points 2^20 -> 21 slot bits -> 4 epoch bits


def frames(k):
    """Frame k of a varied stream: scene, pose."""
    d = [syn.scene_room(), syn.scene_sphere(4.0), syn.scene_noise(seed=k), syn.scene_plane(3.0)][k % 4]
    R = rot_xyz(0.05 * (k % 7), -0.03 * (k % 5), 0.11 * k)
    T = np.array([0.02 * (k % 9), -0.015 * (k % 4), 0.01 * (k % 3)])
    return d, R, T


def cloud(k, n=20000):
    rng = np.random.default_rng(100 + k)
    xyz = rng.normal(size=(n, 3))
    xyz = (xyz / np.linalg.norm(xyz, axis=1, keepdims=True) * rng.uniform(1.0, 6.0, size=(n, 1))).astype(np.float32)
    rgb = rng.integers(0, 256, size=(n, 3), dtype=np.uint8)
    return xyz, rgb


def counters(g):
    s = g.stats(clear=True)
    return {k: s[k] for k in ("n_px", "n_valid", "n_rays", "n_updates", "n_oob", "err_flags")}


def same_map(a, b, color=False):
    if color:
        ai, at, aw, ao, ac = a.gather(color=True)
        bi, bt, bw, bo, bc = b.gather(color=True)
        ca, cb = ac[key_sort(ai)], bc[key_sort(bi)]
        fin = np.isfinite(ca).all(1)
        assert np.array_equal(fin, np.isfinite(cb).all(1))
        assert np.array_equal(ca[fin], cb[fin]), "voxel colours differ"
    else:
        ai, at, aw, ao = a.gather()
        bi, bt, bw, bo = b.gather()
    compare_voxels((ai, at, aw, ao), (bi, bt, bw, bo), 1e-4)


@pytest.mark.gpu
def test_epoch_wraps_twice_equals_clearing_mode():
    """More launches than the epoch counts (it wraps twice): every launch's statistics and the final map equal those of
    a clearing-mode handle fed the same launches."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    ge = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    gc = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True, max_points=CLEARING_MAX_POINTS)
    for k in range(2 * EPOCHS_DEFAULT + 7):
        d, R, T = frames(k)
        for g in (ge, gc):
            if k % 5 == 3:
                g.integrate_points(cloud(k)[0], R, T)
            else:
                g.integrate_depth(d, R[None], T[None])
        ce, cc = counters(ge), counters(gc)
        assert ce == cc, f"launch {k}: {ce} vs {cc}"
        assert ce["err_flags"] == 0 and ce["n_rays"] > 0
    same_map(ge, gc)


@pytest.mark.gpu
@pytest.mark.parametrize("max_points", [0, CLEARING_MAX_POINTS])
def test_mixed_batches_match_oracle(max_points):
    """Depth batches, a point cloud and another depth batch on one handle, in both modes, against the CPU oracle."""
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    o = OracleTSDF(map_scale=[25.6, 25.6], K=syn.K_DEPTH, is_global_map=True)
    g = TsdfHandle(o.N, o.Nz, K=syn.K_DEPTH, is_global_map=True, max_points=max_points)
    for k in (0, 1):
        d, R, T = frames(k)
        g.integrate_depth(d, R[None], T[None])
        o.integrate_depth(R, T, d)
    xyz, _ = cloud(2)
    R, T = rot_xyz(0.2, 0.1, -0.3), np.array([0.1, 0.2, -0.05])
    g.integrate_points(xyz, R, T)
    o.integrate_points(R, T, xyz)
    d, R, T = frames(5)
    g.integrate_depth(d, R[None], T[None])
    o.integrate_depth(R, T, d)
    sg, so = g.stats(), o.stats()
    for k in ("n_px", "n_valid", "n_rays", "n_updates", "n_oob"):
        assert sg[k] == so[k], f"{k}: gpu {sg[k]} oracle {so[k]}"
    assert sg["err_flags"] == 0
    compare_voxels(g.gather(), o.gather(), 1e-4)


@pytest.mark.gpu
def test_textured_and_points_mixed_with_depth():
    """Textured frames, coloured and uncoloured point clouds and untextured depth frames on one textured handle: both
    modes give the same map and colours, across an epoch wrap."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    hs = [TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True, texture_enabled=True, max_points=mp) for mp in (0, CLEARING_MAX_POINTS)]
    for g in hs:
        g.set_color_intrinsics([1, 0, 0, 0, 1, 0, 0, 0, 1], True)
    for k in range(EPOCHS_DEFAULT + 3):
        d, R, T = frames(k)
        xyz, rgb = cloud(k, 5000)
        for g in hs:
            if k % 3 == 0:
                g.integrate_depth(d, R[None], T[None], texture=syn.texture_gradient(k)[None])
            elif k % 3 == 1:
                g.integrate_points(xyz, R, T, rgb=rgb if k % 2 else None)
            else:
                g.integrate_depth(d, R[None], T[None])
        assert counters(hs[0]) == counters(hs[1]), f"launch {k}"
    same_map(hs[0], hs[1], color=True)


@pytest.mark.gpu
@pytest.mark.parametrize("max_points", [0, CLEARING_MAX_POINTS])
def test_max_points_cloud_with_count_plane_matches_oracle(max_points):
    """2^20 points at 9.5 m, 900 000 of them in one bucket: more than the packed count word can hold next to their depth
    sum (it would need 2^43 > 9.5 m * 2^20 * 900 000), so the launch keeps its counts in a plane of their own.  On a
    default handle (max_points = 2^20, max_ray 10 m) and in clearing mode, the map matches the CPU oracle."""
    from oracle.oracle import OracleTSDF
    from taichislam_b200.tsdf_handle import TsdfHandle
    o = OracleTSDF(map_scale=[25.6, 25.6], K=syn.K_DEPTH, is_global_map=True)
    g = TsdfHandle(o.N, o.Nz, K=syn.K_DEPTH, is_global_map=True, max_points=max_points)
    rng = np.random.default_rng(7)
    n = 1 << 20
    centres = np.array([[9.5, 0.5, 0.25], [0.0, 9.5, 0.5], [-9.0, 1.0, 2.0], [6.0, -7.0, 1.0],
                        [3.0, 3.0, 8.5], [-2.0, -9.0, -1.0], [5.0, 5.0, -6.0], [-6.0, 6.0, 4.0]])
    which = np.concatenate([np.zeros(900000, np.int64), rng.integers(1, len(centres), n - 900000)])
    xyz = (centres[which] + rng.uniform(-0.01, 0.01, size=(n, 3))).astype(np.float32)
    assert (np.linalg.norm(xyz, axis=1) < 10.0).all()
    g.integrate_points(xyz, np.eye(3), np.zeros(3))
    o.integrate_points(np.eye(3), np.zeros(3), xyz)
    sg, so = g.stats(), o.stats()
    for k in ("n_px", "n_valid", "n_rays", "n_updates", "n_oob"):
        assert sg[k] == so[k], f"{k}: gpu {sg[k]} oracle {so[k]}"
    assert sg["err_flags"] == 0 and sg["n_rays"] == len(centres)
    compare_voxels(g.gather(), o.gather(), 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("max_points", [0, CLEARING_MAX_POINTS])
def test_clean_launch_after_capacity_error_is_exact(max_points):
    """A launch that drops points and raises E_CAPACITY (bucket key range), then a clean launch: the clean launch's
    statistics and map equal a fresh handle's.  (The points are dropped before they are probed, so this checks the error
    path's bookkeeping, not a dirty index: every launch in epoch mode leaves its entries behind, and the launch sequences
    above check that the next launch ignores them.)"""
    from taichislam_b200.tsdf_handle import TsdfHandle
    from taichislam_b200 import _capi as capi
    g = TsdfHandle(512, 512, voxel_scale=0.002, K=syn.K_DEPTH, is_global_map=True, max_points=max_points)
    far = syn.scene_room()
    far[:, : far.shape[1] // 2] = 9000  # half the frame beyond the key range, half inside it
    g.integrate_depth(far, np.eye(3)[None], np.zeros((1, 3)), commit=False)
    with pytest.raises(capi.TslamError) as e:
        g.sync()
    assert e.value.code == capi.E_CAPACITY
    g.reset()
    g.stats(clear=True)
    f = TsdfHandle(512, 512, voxel_scale=0.002, K=syn.K_DEPTH, is_global_map=True, max_points=max_points)
    d = syn.scene_sphere(4.0)
    for h in (g, f):
        h.integrate_depth(d, np.eye(3)[None], np.zeros((1, 3)))
        h.sync()
    cg, cf = counters(g), counters(f)
    assert cg == cf and cg["n_rays"] > 1000
    same_map(g, f)


def _bounds_program(body):
    src = "#include <cstdio>\n#include \"tslam_bucket.cuh\"\nint main() {\n" + body + "\n  return 0;\n}\n"
    with tempfile.TemporaryDirectory() as tmp:
        c, exe = os.path.join(tmp, "t.cpp"), os.path.join(tmp, "t")
        with open(c, "w") as fh:
            fh.write(src)
        subprocess.run(["g++", "-std=c++17", "-O1", "-I", CSRC, c, "-o", exe], check=True)
        return subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()


def test_count_depth_packing_bounds():
    """cnt << shift | sum(d): at the configuration limits the shift leaves both fields room, and where no shift can
    (-1) the launch keeps its counts in a plane of their own instead of packing a sum that could carry into the count."""
    cases = [(640 * 480 // 4, 10.0), (640 * 480, 64.0), ((1 << 19) - 1, 63.99), (1 << 20, 10.0), (1 << 20, 3.9), (1 << 25, 1.0), (1, 1e6)]
    out = _bounds_program("\n".join(f'  printf("%d\\n", ts_bucket_cnt_shift({n}ull, {dm!r}));' for n, dm in cases))
    for (n, dm), s in zip(cases, map(int, out)):
        q = int(np.ceil(dm * 2**20)) + 1
        fits = [k for k in range(1, 64) if n < 2 ** (64 - k) and n * q < 2 ** k]
        want = 64 - n.bit_length()
        if want in fits:
            assert s == want, (n, dm, s)
        else:
            assert s == -1, (n, dm, s)
    assert list(map(int, out)) == [47, 45, 45, -1, 43, -1, 63]


def test_index_slot_bits():
    """The slot field holds slot + 1 of a depth frame (< bucket_cap) or a point cloud (<= max_points); fewer than 4 bits
    left for the epoch select clearing mode (25)."""
    cases = [(1 << 17, 1 << 20), (1 << 17, 1000), (1 << 17, 1 << 21), (1 << 21, 1000), (1 << 20, (1 << 21) - 1)]
    out = _bounds_program("\n".join(f'  printf("%d\\n", ts_bucket_slot_bits({b}u, {p}u));' for b, p in cases))
    assert list(map(int, out)) == [21, 18, 25, 25, 21]
