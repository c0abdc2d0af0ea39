"""The frontier-viewpoint reference (octo_viewpoint_reference.py) on hand-worked answers.  Volume 32^3 (cells in
[-16, 16)), voxels of 0.5 m.  The scene is a FREE box, cells i in [-6, 0], j in [-3, 3], k in [-2, 2], walled by OCC
cells on every side but +i, where unknown space begins: its frontier is the 7 x 5 face i = 0, one cluster with its
centroid at the origin."""
import numpy as np

import octo_frontier_reference as fr
import octo_viewpoint_reference as vp

N = NZ = 32
VS = 0.5
FREE_L, OCC_L, L_OCC = -415, 868, 0
# fx = fy = 4 at 2 m: frontier voxel (0, j, k) projects to u = 3 - j, v = 2 - k, so a 7 x 5 image sees the whole face
CAM = dict(fx=4.0, fy=4.0, cx=3.0, cy=2.0, width=7, height=5, step=1, max_range=3.0)
AHEAD = (-2.0, 0.0, 0.0)   # 2 m from the centroid on -x: cell (-4, 0, 0), looking along +x


def box():
    g = np.stack(np.meshgrid(np.arange(-7, 1), np.arange(-4, 5), np.arange(-3, 4), indexing="ij"), -1).reshape(-1, 3)
    inner = (g[:, 0] >= -6) & (np.abs(g[:, 1]) <= 3) & (np.abs(g[:, 2]) <= 2)
    idx = np.concatenate([g[inner], g[~inner]]).astype(np.int32)
    L = np.concatenate([np.full(inner.sum(), FREE_L), np.full((~inner).sum(), OCC_L)]).astype(np.int32)
    return idx, L


def run(offsets, cam=CAM, **kw):
    idx, L = box()
    return vp.viewpoints(idx, L, L_OCC, N, NZ, VS, np.asarray(offsets, np.float32).reshape(-1, 3), cam, **kw)


def test_the_scene_has_one_cluster_on_the_open_face():
    idx, L = box()
    fidx, fcl, rec = fr.frontiers(idx, L, L_OCC, N, NZ)
    assert rec.shape[0] == 1 and rec[0, 1] == 35 and (fidx[:, 0] == 0).all()
    assert vp.centroids(rec, VS).tolist() == [[0.0, 0.0, 0.0]]


def test_free_face_seen_from_a_sample_at_a_known_distance():
    out = run([AHEAD])
    assert out["count"].tolist() == [1] and out["sample"].tolist() == [[0]] and out["visible"].tolist() == [[35]]
    assert out["pos"][0, 0].tolist() == [-2.0, 0.0, 0.0]
    assert out["R"][0, 0].tolist() == [[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]]   # camera z along +x
    narrow = run([AHEAD], cam=dict(CAM, width=3, cx=1.0))        # u = 1 - j in [0, 2]: j in {-1, 0, 1}, every k
    assert narrow["visible"].tolist() == [[15]]
    short = run([AHEAD], cam=dict(CAM, max_range=1.5))          # the face is 2 m ahead
    assert short["count"].tolist() == [0] and short["score"].tolist() == [[0]] and short["valid"].tolist() == [[True]]


def test_sample_above_the_centroid_has_no_heading():
    out = run([(0.0, 0.0, 1.0), AHEAD])                         # cell (0, 0, 2) is FREE, but h = 0
    assert out["valid"].tolist() == [[False, True]]
    assert out["sample"].tolist() == [[1]]


def test_samples_in_occ_unknown_outside_and_non_finite_are_invalid():
    offs = [(-3.5, 0.0, 0.0), (1.0, 0.0, 0.0), (20.0, 0.0, 0.0), (np.nan, 0.0, 0.0), (0.0, np.inf, 0.0), AHEAD]
    out = run(offs)                                               # OCC (-7,0,0), UNKNOWN (2,0,0), outside, NaN, inf
    assert out["valid"].tolist() == [[False] * 5 + [True]]
    assert out["score"][0, :5].tolist() == [0] * 5
    assert out["count"].tolist() == [1] and out["sample"].tolist() == [[5]]


def test_clearance_excludes_the_sample_next_to_the_wall():
    idx, L = box()
    esdf = vp.esdf_rows(idx, L, L_OCC, VS, 2.0)
    wall = (-3.0, 0.0, 0.0)                                       # cell (-6, 0, 0), 0.5 m from the OCC wall at i = -7
    assert run([wall, AHEAD])["valid"].tolist() == [[True, True]]
    out = run([wall, AHEAD], clearance=0.6, esdf=esdf)            # cell (-4, 0, 0) is 1.5 m from every wall
    assert out["valid"].tolist() == [[False, True]] and out["sample"].tolist() == [[1]]
    assert run([wall, AHEAD], clearance=1.5, esdf=esdf)["valid"].tolist() == [[False, True]]
    assert run([wall, AHEAD], clearance=1.6, esdf=esdf)["valid"].tolist() == [[False, False]]


def test_min_visible_cut():
    offs = [AHEAD, (-1.0, 0.0, 0.0)]        # from 1 m, fx = 4 maps j to u = 3 - 2j: j in {-1, 0, 1}, k in {-1, 0, 1}
    out = run(offs, min_visible=1, top_k=2)
    assert out["score"].tolist() == [[35, 9]] and out["count"].tolist() == [2]
    assert run(offs, min_visible=9, top_k=2)["count"].tolist() == [2]
    cut = run(offs, min_visible=10, top_k=2)
    assert cut["count"].tolist() == [1] and cut["sample"].tolist() == [[0, -1]]
    assert run(offs, min_visible=36)["count"].tolist() == [0]


def test_ties_are_ranked_by_sample_index():
    offs = [(-1.0, 0.0, 0.0), AHEAD, AHEAD, (-1.0, 0.0, 0.0)]
    out = run(offs, top_k=4)
    assert out["sample"].tolist() == [[1, 2, 0, 3]] and out["visible"].tolist() == [[35, 35, 9, 9]]


def test_top_k_above_the_kept_count():
    out = run([AHEAD, (1.0, 0.0, 0.0)], top_k=5)
    assert out["count"].tolist() == [1]
    assert out["sample"].tolist() == [[0, -1, -1, -1, -1]] and out["visible"].tolist() == [[35, 0, 0, 0, 0]]
    assert not out["pos"][0, 1:].any() and not out["R"][0, 1:].any()


def test_rotation_is_orthonormal_and_faces_the_centroid_level():
    ang = 2 * np.pi * np.arange(16) / 16
    offs = np.stack([1.3 * np.cos(ang), 1.3 * np.sin(ang), np.full(16, 0.4)], 1).astype(np.float32)
    m = np.array([[0.1, -0.2, 0.3]], np.float32)
    p, R, h = vp.poses(m, offs)
    assert (h > 0).all()
    for q in range(16):
        Rq = R[0, q].astype(np.float64)
        assert np.allclose(Rq @ Rq.T, np.eye(3), atol=1e-6) and abs(np.linalg.det(Rq) - 1.0) < 1e-6
        z = Rq[:, 2]
        d = (m[0] - p[0, q]).astype(np.float64)
        d[2] = 0.0
        assert z[2] == 0.0 and np.allclose(z, d / np.linalg.norm(d), atol=1e-6)
        assert Rq[:, 1].tolist() == [0.0, 0.0, -1.0]               # camera y (image down) points down: level
