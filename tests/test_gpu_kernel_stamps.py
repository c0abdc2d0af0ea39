"""Kernel times from the kernels' own %globaltimer stamps (kernel_ms2): every column of a profiled launch is positive, the
parts of the ray march fit inside it, and the columns fit inside the launch's span as a pair of CUDA events around the
launch measures it.  Profiling changes no result."""
import numpy as np
import pytest

from taichislam_b200 import synthetic as syn
from util import as_dict_rows, rot_xyz

pytestmark = pytest.mark.gpu
TOL = 1e-4
REL = 1e-5  # float32 rounding of the columns


def _frames(n, start):
    import torch
    d = syn.scene_sphere(4.0)
    Rs, Ts = syn.stream_poses(n, start=start)
    return torch.from_numpy(np.stack([d] * n).view(np.int16)).cuda(), Rs, Ts


def _timed_launch(g, dev, Rs, Ts, commit=True):
    """One launch between two CUDA events, each recorded on an idle device: ms of the launch's whole span."""
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    g.integrate_depth(dev, Rs, Ts, commit=commit)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def test_kernel_ms2_columns_fit_the_launch():
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    dev, Rs, Ts = _frames(64, 0)
    g.integrate_depth(dev, Rs, Ts, commit=True)  # first launch: module load, march workspace
    g.set_profiling(True)
    spans = [_timed_launch(g, dev, Rs, Ts) for _ in range(3)]
    k = g.kernel_ms2(8)
    assert k.shape == (3, 7)
    k3 = g.kernel_ms(8)
    assert np.array_equal(k3, k[:, :3])
    for row, span in zip(k[::-1], spans):  # kernel_ms2 lists the most recent launch first
        bucket, march, commit, zero, walk, scatter, blocks = (float(x) for x in row)
        assert min(bucket, march, commit, walk, scatter, blocks) > 0.0, row
        assert zero == 0.0
        assert walk + scatter + blocks <= march * (1 + REL), row       # the march's parts are disjoint parts of it
        assert bucket + march + commit <= span * (1 + REL), (row, span)  # the stages are disjoint parts of the span

    # a launch without commit charges nothing to the commit column
    span = _timed_launch(g, dev, Rs, Ts, commit=False)
    row = g.kernel_ms2(1)[0]
    assert row[2] == 0.0 and row[0] > 0.0 and row[1] > 0.0 and row[0] + row[1] <= span * (1 + REL)
    g.commit()
    g.sync()


def test_kernel_ms2_of_textured_and_point_cloud_launches():
    """Textured maps march with k_raymarch (one kernel: the march's parts are 0); point clouds take the depth chain."""
    from taichislam_b200.tsdf_handle import TsdfHandle
    d = syn.scene_sphere(3.0)
    tex = np.full(d.shape + (3,), 90, np.uint8)
    Rs, Ts = syn.stream_poses(4, start=1)
    t = TsdfHandle(256, 256, K=syn.K_DEPTH, is_global_map=True, texture_enabled=True)
    t.set_profiling(True)
    t.integrate_depth(np.stack([d] * 4), Rs, Ts, texture=np.stack([tex] * 4))
    row = t.kernel_ms2(1)[0]
    assert row[0] > 0.0 and row[1] > 0.0 and row[2] > 0.0
    assert np.all(row[3:] == 0.0)

    rng = np.random.default_rng(5)
    u = rng.normal(size=(20000, 3))
    pts = (u / np.linalg.norm(u, axis=1, keepdims=True) * rng.uniform(0.5, 6.0, size=(20000, 1))).astype(np.float32)
    p = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    p.set_profiling(True)
    p.integrate_points(pts, rot_xyz(0.1, 0.2, -0.3), np.array([0.1, -0.2, 0.3]))
    row = p.kernel_ms2(1)[0]
    assert min(row[0], row[1], row[2], row[4], row[5], row[6]) > 0.0 and row[3] == 0.0
    assert row[4] + row[5] + row[6] <= row[1] * (1 + REL)


def _run(profiling):
    from taichislam_b200.tsdf_handle import TsdfHandle
    g = TsdfHandle(512, 512, K=syn.K_DEPTH, is_global_map=True)
    g.set_profiling(profiling)
    a, Ra, Ta = _frames(32, 3)
    b = syn.scene_room()
    Rb = np.stack([rot_xyz(0.1 * q, -0.05, 0.2) for q in range(8)])
    Tb = np.stack([np.array([0.3, -0.2, 0.1]) * q / 8 for q in range(8)])
    g.integrate_depth(a, Ra, Ta, commit=True)
    g.integrate_depth(np.stack([b] * 8), Rb, Tb, commit=False)  # host frames, committed with the next launch
    g.integrate_depth(a[:16], Ra[16:], Ta[16:], commit=True)
    g.sync()
    return g.stats(), g.march_stats(), g.gather()


def test_profiling_changes_no_result():
    s0, m0, v0 = _run(False)
    s1, m1, v1 = _run(True)
    assert s0 == s1
    assert m0 == m1 and m0["n_seg_guard"] == 0
    x, y = as_dict_rows(*v0), as_dict_rows(*v1)
    assert np.array_equal(x[0], y[0]) and np.array_equal(x[3], y[3])
    # TSDF and weight: the march's f32 reductions into acc are order-dependent, as between any two runs
    assert np.abs(x[1] - y[1]).max() <= TOL
    assert np.all(np.abs(x[2] - y[2]) <= TOL * np.maximum(1.0, np.abs(y[2])))
