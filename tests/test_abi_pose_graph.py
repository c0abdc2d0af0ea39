"""Refusals of tslam_pose_graph_solve that need no GPU, in the header's order: every check runs on the host before any
device work, and a refused call writes nothing."""
import numpy as np

import pose_graph_reference as P
from taichislam_b200 import _capi as capi


def _call(N=3, R=None, T=None, fixed=None, ij=None, ZR=None, ZT=None, om=None, c=None, prm=None, null=None):
    I = np.eye(3)
    a = dict(R=np.ascontiguousarray(np.tile(I.ravel(), (N, 1))) if R is None else R,
             T=np.zeros((N, 3)) if T is None else T,
             fixed=np.array([1] + [0] * (N - 1), np.uint8) if fixed is None else fixed,
             ij=np.array([[0, 1], [1, 2]], np.int32) if ij is None else ij,
             ZR=np.tile(I.ravel(), (2, 1)) if ZR is None else ZR, ZT=np.zeros((2, 3)) if ZT is None else ZT,
             om=np.tile(np.eye(6).ravel(), (2, 1)) if om is None else om, c=np.zeros(2) if c is None else c)
    E = len(a["ij"])
    out = dict(Ro=np.full((max(N, 1), 9), 7.0), To=np.full((max(N, 1), 3), 7.0), chi2=np.full(max(E, 1), 7.0),
               w=np.full(max(E, 1), 7.0), f3=np.full(3, 7.0), info=np.full(5, 7, np.int64))
    p = prm if prm is not None else capi.PgParams(1e-6, 1e-8, 1e-10, 10, 100, 0)
    ptr = {k: capi.np_ptr(np.ascontiguousarray(v)) for k, v in {**a, **out}.items()}
    if null:
        ptr[null] = None
    rc = capi.load().tslam_pose_graph_solve(N, ptr["R"], ptr["T"], ptr["fixed"], E, ptr["ij"], ptr["ZR"], ptr["ZT"], ptr["om"],
                                            ptr["c"], p, ptr["Ro"], ptr["To"], ptr["chi2"], ptr["w"], ptr["f3"], ptr["info"],
                                            None)
    untouched = all(np.all(v == 7) for v in out.values())
    return rc, capi.load().tslam_last_error().decode(), untouched


def refused(fragment, **kw):
    rc, msg, untouched = _call(**kw)
    assert rc == capi.E_INVALID and fragment in msg and untouched, (rc, msg, kw)


def test_sizes_nulls_and_params():
    for N in (0, 1, 4097):
        refused("n_nodes", N=N)
    refused("n_edges", ij=np.zeros((0, 2), np.int32))
    for k in ("R", "T", "fixed", "ij", "ZR", "ZT", "om", "c", "Ro", "To", "chi2", "w", "f3", "info"):
        refused("NULL", null=k)
    for p in ((-1.0, 1e-8, 1e-10, 10, 100, 0), (1e-6, np.nan, 1e-10, 10, 100, 0), (1e-6, 1e-8, 1.0, 10, 100, 0),
              (1e-6, 1e-8, 1e-10, -1, 100, 0), (1e-6, 1e-8, 1e-10, 10, 0, 0), (1e-6, 1e-8, 1e-10, 10, 100, -1),
              (1e-6, 1e-8, 1e-10, 100001, 100, 0)):
        refused("solver parameters", prm=capi.PgParams(*p))
    # sizes before NULLs before params
    refused("n_nodes", N=1, null="R", prm=capi.PgParams(-1.0, 1e-8, 1e-10, 10, 100, 0))
    refused("NULL", null="R", prm=capi.PgParams(-1.0, 1e-8, 1e-10, 10, 100, 0))


def test_nodes_then_edges_then_components():
    I9 = np.tile(np.eye(3).ravel(), (3, 1))
    T = np.zeros((3, 3)); T[1, 2] = np.inf
    refused("node 1: pose not finite", T=T)
    R = I9.copy(); R[2] *= 1.0001
    refused("node 2: rotation", R=R)
    refused("node 1: pose not finite", T=T, R=R)  # nodes in order
    for ij in ([[0, 3], [1, 2]], [[0, -1], [1, 2]], [[0, 1], [2, 2]]):
        refused("endpoints", ij=np.array(ij, np.int32))
    refused("node 1", T=T, ij=np.array([[0, 0], [1, 2]], np.int32))  # nodes before edges
    om = np.tile(np.eye(6).ravel(), (2, 1)); om[1, 5] = np.nan  # (0, 5): upper triangle
    refused("edge 1: measurement, information or Cauchy scale not finite", om=om)
    refused("not finite", c=np.array([0.0, np.inf]))
    refused("Cauchy scale", c=np.array([-1.0, 0.0]))
    ZR = np.tile(np.eye(3).ravel(), (2, 1)); ZR[0] = (P.rot([0, 0, 1], 5.0) * 1.001).ravel()
    refused("edge 0: rotation", ZR=ZR)
    om = np.tile(np.eye(6).ravel(), (2, 1)); om[0, 21] = -1.0  # (3, 3)
    refused("negative diagonal", om=om)
    refused("no fixed node", fixed=np.zeros(3, np.uint8))
    refused("no fixed node", ij=np.array([[0, 1], [0, 1]], np.int32))  # node 2 alone and free
    refused("edge 0: endpoints", ij=np.array([[0, 0], [0, 1]], np.int32), fixed=np.zeros(3, np.uint8))  # edges first
