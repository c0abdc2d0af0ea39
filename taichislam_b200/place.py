"""Place matching between TSDF submap descriptors (tslam_place_match, include/tslam.h; DESIGN.md section 7, "Loop
detection").  The descriptors come from TsdfHandle.place_describe; this stage reads them only, so a caller can keep them
across calls."""
import numpy as np

from . import _capi as capi

RINGS, SECTORS, WORDS = 20, 60, 512


def level(up=(0.0, 0.0, 1.0)):
    """L f64 [3,3]: the minimal rotation that takes the world unit vector along `up` to +z (the identity for +z, a half
    turn about x for -z).  Raises ValueError for an `up` that is not finite or has zero length."""
    u = np.asarray(up, np.float64).reshape(3)
    n = float(np.linalg.norm(u)) if np.all(np.isfinite(u)) else float("nan")
    if not n > 0.0 or not np.isfinite(n):
        raise ValueError(f"up must be finite and of non-zero length, not {tuple(u)}")
    u = u / n
    v = np.array([u[1], -u[0], 0.0])  # u x z
    s2, c = float(v @ v), float(u[2])
    if s2 == 0.0:
        return np.eye(3) if c > 0.0 else np.diag([1.0, -1.0, -1.0])
    K = np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])
    return np.eye(3) + K + K @ K * ((1.0 - c) / s2)


def coarse_pose(Mq, Md, yaw_deg, dx, dy, r_max):
    """The q-local -> d-local pose of a match, in f64 from the f64 levelled rotations Mq = L R_q, Md = L R_d: levelled
    points satisfy x_d = Rz(yaw) x_q + (dx c, dy c, 0), c = f32(r_max) / 64, so T0 = (Md^T Rz Mq, Md^T (dx c, dy c, 0))."""
    a = np.deg2rad(float(yaw_deg))
    Rz = np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])
    c = float(np.float32(r_max) / np.float32(64.0))
    Mq, Md = np.asarray(Mq, np.float64), np.asarray(Md, np.float64)
    return Md.T @ Rz @ Mq, Md.T @ np.array([dx * c, dy * c, 0.0])


def match(sc, ring, bev, n_points, ids, queries, top_k=8, min_gap=1, min_points=200):
    """Match database entries `queries` (indices) against the whole database of n descriptors: sc f32 [n,20,60], ring f32
    [n,20], bev int32 [n,512] torch CUDA tensors (place_describe's), n_points and ids int64 [n] (any array).  Entry d is
    eligible for query q when d != q, |ids[q] - ids[d]| >= min_gap and both have >= min_points points.  Returns a dict of
    numpy arrays [n_q, top_k]: match (database index, -1 past the eligible entries), ring_dist, sc_dist (D at the best
    shift), shift (m*), yaw_idx (0, 1, 2: yaw (2 m* + yaw_idx - 1) x 3 degrees), yaw_deg, dx, dy (cells), score,
    overlap.  Raises TslamError (E_INVALID) on an argument the contract refuses."""
    import torch
    dev = sc.device
    n = int(sc.shape[0])
    q = np.ascontiguousarray(np.asarray(queries, dtype=np.int32).reshape(-1))
    nq, k = q.shape[0], int(top_k)
    npts = torch.as_tensor(np.asarray(n_points, np.int64).reshape(-1), device=dev).contiguous()
    idt = torch.as_tensor(np.asarray(ids, np.int64).reshape(-1), device=dev).contiguous()
    if npts.numel() != n or idt.numel() != n:
        raise ValueError(f"n_points and ids need {n} entries")
    rows = max(nq * k, 1)
    info = torch.empty((rows, 6), dtype=torch.int32, device=dev)
    dist = torch.empty((rows, 3), dtype=torch.float32, device=dev)
    L = capi.load()
    capi.check(L.tslam_place_match(n, capi.tptr(sc.contiguous()), capi.tptr(ring.contiguous()), capi.tptr(bev.contiguous()),
                                   capi.tptr(npts), capi.tptr(idt), nq, capi.np_ptr(q), k, int(min_gap), int(min_points),
                                   capi.tptr(info), capi.tptr(dist), capi.stream_ptr()))
    info = info[:nq * k].cpu().numpy().reshape(nq, k, 6)
    dist = dist[:nq * k].cpu().numpy().reshape(nq, k, 3)
    m, y = info[..., 1], info[..., 2]
    return dict(match=info[..., 0], shift=m, yaw_idx=y, yaw_deg=6.0 * m + 3.0 * (y - 1.0), dx=info[..., 3], dy=info[..., 4],
                score=info[..., 5], ring_dist=dist[..., 0], sc_dist=dist[..., 1], overlap=dist[..., 2], info6=info, dist3=dist)
