"""GPU: the marching-cubes kernels (k_mc_count / k_mc_scan / k_mc_emit at step 1, k_mc_generic at step > 1, the colour
path, the incremental mesh) against tests/mc_reference.py, bit for bit.  Maps are scattered so that every value is
chosen, or integrated and gathered back; triangles are compared as sorted uint32 rows with NaN made canonical, and the
triangle count exactly.  Each case asserts, from the reference's own tags, that it produced what it is there for."""
import ctypes as C
import gc

import numpy as np
import pytest

import mc_reference as mcr
import track_world as tw
from taichislam_b200 import _capi as capi
from taichislam_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
F = np.float32
VS = 0.05


@pytest.fixture(autouse=True)
def release_maps():
    gc.collect()
    yield
    gc.collect()


def handle(N=256, Nz=256, **kw):
    from taichislam_b200.tsdf_handle import TsdfHandle
    return TsdfHandle(N, Nz, voxel_scale=VS, is_global_map=True, **kw)


def generate(g, step, thres, cap, color=False):
    """tslam_mc_generate2 -> (rc, demand, verts, normals, colors or None) of the min(demand, cap) emitted triangles."""
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    bufs = [torch.empty((3 * max(cap, 1), 3), dtype=torch.float32, device=dev) for _ in range(3 if color else 2)]
    n = C.c_int64(0)
    rc = g.L.tslam_mc_generate2(g.h, int(step), float(F(thres)), int(cap), capi.tptr(bufs[0]), capi.tptr(bufs[1]),
                                capi.tptr(bufs[2]) if color else None, C.byref(n), capi.stream_ptr())
    if rc != capi.E_CAPACITY:
        capi.check(rc)
    k = 3 * min(int(n.value), cap)
    out = [b[:k].cpu().numpy().reshape(-1, 3, 3) for b in bufs]
    return rc, int(n.value), out[0], out[1], (out[2] if color else None)


def reference(g, submaps, step, thres, color=False):
    return mcr.mesh({s: g.gather(s, color=color) for s in submaps}, g.N, g.Nz, VS, step, thres, color=color)


def ref_rows(ref):
    return mcr.sorted_rows(ref["verts"], ref["normals"], ref.get("colors"))


def audit(g, submaps, step, thres, color=False):
    """The one-shot mesh of g equals the reference's: count and every word.  -> the reference's mesh."""
    ref = reference(g, submaps, step, thres, color)
    n = ref["tag"].shape[0]
    rc, demand, v, nrm, col = generate(g, step, thres, n + 4096, color)
    assert rc == 0 and demand == n, (demand, n)
    got = mcr.sorted_rows(v, nrm, col)
    want = ref_rows(ref)
    bad = np.any(got != want, 1)
    assert not bad.any(), f"{int(bad.sum())} of {n} triangle rows differ, first got {got[bad][0]} want {want[bad][0]}"
    return ref


def box(lo, hi):
    r = [np.arange(a, b) for a, b in zip(lo, hi)]
    I, J, K = np.meshgrid(*r, indexing="ij")
    return np.stack([I.ravel(), J.ravel(), K.ravel()], 1).astype(np.int32)


def rows_of(idx, t):
    return idx, np.asarray(t, F), np.ones(len(idx), F), np.zeros(len(idx), np.int8)


def sphere_rows(c, r, half):
    c0 = np.floor(c).astype(int)
    idx = box(c0 - half, c0 + half + 1)
    d = np.sqrt(((idx - np.asarray(c)) ** 2).sum(1))
    return idx, ((d - r) * VS).astype(F)


# -- spheres across block corners, edges and faces, at negative coordinates -------------------------------------------
SPHERES = [((-32.0, -16.0, -48.0), 5.3),      # centred on a block corner: cells straddle 8 blocks
           ((-64.0, -48.0, -70.3), 5.7),      # on a block edge
           ((-88.6, -24.2, -41.1), 4.9)]      # inside one block


@pytest.fixture(scope="module")
def spheres():
    g = handle()
    idx, t = zip(*[sphere_rows(c, r, int(r) + 3) for c, r in SPHERES])
    g.scatter(0, *rows_of(np.concatenate(idx), np.concatenate(t)))
    return g


@pytest.mark.parametrize("step", [1, 2, 3])
@pytest.mark.parametrize("thres", ["0.1", "stored"])
def test_spheres_across_blocks(spheres, step, thres):
    g = spheres
    t = g.gather(0)[1]
    # "stored": a threshold equal to a stored T (the smallest T above 0.02): the cells whose corner 0 holds it are out
    th = F(0.1) if thres == "0.1" else F(np.min(t[t > F(0.02)]))
    ref = audit(g, [0], step, th)
    tag = ref["tag"]
    assert tag.shape[0] > 100
    nb = mcr.block_count(tag, step)
    assert {2, 4, 8} <= set(nb.tolist())
    local = ref["at"] - ((tag[:, None, 1:4] >> 4) << 4)
    assert (local == 16).any() and (local == 0).any()  # normals read the +17 and the -1 halo layers
    if thres == "stored" and step == 1:
        more = reference(g, [0], step, np.nextafter(th, F(1)))
        assert more["tag"].shape[0] > tag.shape[0]  # the strict test excluded cells


# -- N = 200, Nz = 70: the surface leaves the volume ------------------------------------------------------------------
@pytest.mark.parametrize("step", [1, 2, 3])
def test_volume_edges(step):
    g = handle(200, 70)
    cx, cy, r = -20.3, 13.7, 9.4   # a cylinder along z through the whole volume (k = -35 .. 34)
    idx = box((-33, 1, -35), (-7, 27, 35))
    t1 = (np.hypot(idx[:, 0] - cx, idx[:, 1] - cy) - r) * VS
    c2 = np.array([95.2, -40.5, 10.1])  # a sphere through the upper x face (i < 100)
    idx2 = box((86, -50, 0), (100, -30, 21))
    t2 = (np.sqrt(((idx2 - c2) ** 2).sum(1)) - 6.2) * VS
    g.scatter(0, *rows_of(np.concatenate([idx, idx2]), np.concatenate([t1, t2]).astype(F)))
    ref = audit(g, [0], step, 0.1)
    assert ref["edge_skipped"] > 0 and ref["tag"].shape[0] > 500
    top = ref["tag"][:, 3].max()
    assert top == 34 - step and ref["tag"][:, 3].min() == -35 and ref["tag"][:, 1].max() == 99 - step


# -- the special-value plane -----------------------------------------------------------------------------------------
def special_plane(rng):
    """A wavy plane between k = -1 and k = 0 over blocks bx -3 .. -1, by -2 .. 0, with exact zeros, +-5e-7, +-1e-6, -0.0,
    NaN, v2 = -v1 pairs (vertices at k = -0.5 at step 1 and 3), holes of unobserved voxels inside allocated blocks, and
    the column of blocks (bx, by) = (-1, -1) missing."""
    idx = box((-40, -24, -6), (-8, 8, 6))
    t = ((idx[:, 2] + 0.37 + 0.25 * rng.uniform(-1, 1, len(idx))) * VS).astype(F)
    cols = {}
    for n, (i, j, k) in enumerate(idx.tolist()):
        cols.setdefault((i, j), {})[k] = n
    keys = list(cols)
    pick = rng.permutation(len(keys))
    specials = [F(0), F(5e-7), F(-5e-7), F(1e-6), F(-1e-6), F(-0.0), F(np.nan)]
    drop = []
    for q, c in enumerate(pick):
        col = cols[keys[c]]
        kind = q % 12
        if kind < len(specials):
            t[col[-1 if q % 2 else 0]] = specials[kind]
        elif kind == 7:  # v2 = -v1 on the k edge -1 .. 0: the vertex is at k = -0.5
            a = F(rng.uniform(0.1, 0.6) * VS)
            t[col[0]], t[col[-1]] = a, -a
        elif kind == 8:  # and on the step-3 edge -2 .. 1: at -2 + 0.5 * 3
            a = F(rng.uniform(0.1, 0.6) * VS)
            t[col[1]], t[col[-2]] = a, -a
        elif kind == 9:
            drop.append(col[1])       # a hole above the surface
        elif kind == 10:
            drop.append(col[-2])      # and one below
        if kind == 11:
            t[col[2]] = F(np.nan)     # a NaN a normal reads
    keep = np.ones(len(idx), bool)
    keep[drop] = False
    keep &= ~((idx[:, 0] >= -16) & (idx[:, 1] >= -16) & (idx[:, 1] < 0))  # block column (-1, -1) absent
    return rows_of(idx[keep], t[keep])


@pytest.fixture(scope="module")
def plane_map():
    g = handle()
    g.scatter(0, *special_plane(np.random.default_rng(7)))
    return g


@pytest.mark.parametrize("step", [1, 2, 3])
def test_special_values(plane_map, step):
    ref = audit(plane_map, [0], step, 0.1)
    assert ref["tag"].shape[0] > 500
    assert (ref["snap"] == 1).any() and (ref["snap"] == 2).any()
    assert ref["hole"].any() and np.isnan(ref["normals"]).any() and np.isnan(ref["verts"]).any()
    if step != 2:  # (at step 2 a tie lands on a voxel)
        fin = np.isfinite(ref["normals"]).all(2)
        assert (ref["half"] & fin).any()  # .5 ties on negative coordinates with a finite normal to tell roundf by


# -- submaps 0 and 1023 at overlapping coordinates -------------------------------------------------------------------
def two_submaps():
    i0, t0 = sphere_rows((-20.2, -9.7, -14.4), 7.1, 10)
    i1, t1 = sphere_rows((-18.9, -11.3, -12.6), 5.2, 8)
    shell = np.abs(t1) < F(1.8 * VS)   # submap 1023 holds a thin shell: most of its box is unobserved
    return rows_of(i0, t0), rows_of(i1[shell], t1[shell])


@pytest.fixture(scope="module")
def two_map():
    g = handle()
    a, b = two_submaps()
    g.scatter(0, *a)
    g.scatter(1023, *b)
    return g


@pytest.mark.parametrize("step", [1, 2])
def test_submaps_do_not_mix(two_map, step):
    ref = audit(two_map, [0, 1023], step, 0.1)
    s = ref["tag"][:, 0]
    assert (s == 1023).sum() > 50 and (s == 0).sum() > 50
    # reading submap 0's voxels where submap 1023 has none would mesh cells the reference skips
    a, b = two_submaps()
    have = {tuple(v) for v in b[0].tolist()}
    fill = np.array([n for n, v in enumerate(a[0].tolist()) if tuple(v) not in have])
    mixed = mcr.mesh({1023: tuple(np.concatenate([x, y[fill]]) for x, y in zip(b, a))}, 256, 256, VS, step, 0.1)
    assert mixed["tag"].shape[0] != (s == 1023).sum()


# -- colour ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("step", [1, 2])
def test_textured(step):
    rng = np.random.default_rng(3)
    g = handle(texture_enabled=True)
    idx = box((-24, -8, -5), (0, 16, 5))
    t = ((idx[:, 2] + 0.41 + 0.3 * rng.uniform(-1, 1, len(idx))) * VS).astype(F)
    snap = rng.random(len(t)) < 0.06
    t[snap] = rng.choice([F(5e-7), F(-5e-7), F(0)], int(snap.sum()))
    col = rng.uniform(1, 255, (len(t), 3)).astype(F)
    col[rng.random(len(t)) < 0.3, 0] = F(0)
    g.scatter(0, *rows_of(idx, t), color=col)
    ref = audit(g, [0], step, 0.1, color=True)
    assert ref["tag"].shape[0] > 300
    assert {0, 1, 2} <= set(np.unique(ref["cbranch"]).tolist())
    assert ((ref["snap"] > 0) & (ref["cbranch"] == 1)).any()  # a snapped vertex whose colour uses mu = 0


# -- integrated maps, gathered back ----------------------------------------------------------------------------------
def test_integrated_c2_stream():
    g = handle(512, 512, K=syn.K_DEPTH)
    n = 6
    Rs, Ts = syn.stream_poses(n)
    g.integrate_depth(np.stack([syn.scene_sphere(4.0)] * n), Rs, Ts)
    for step in (1, 2):
        ref = audit(g, [0], step, 0.25)
        assert ref["tag"].shape[0] > 10000 / step ** 2


def test_integrated_box_room():
    g = handle(256, 256, K=syn.K_DEPTH, max_ray_length=6.0, min_ray_length=0.3)
    for k in range(0, tw.N_FRAMES, 5):
        R, t = tw.pose(k)
        g.integrate_depth(tw.render(R, t, seed=k), R[None], t[None])
    ref = audit(g, [0], 1, 0.1)
    assert ref["tag"].shape[0] > 10000 and ref["hole"].any()


def test_integrated_bench_stream():
    """Two 64-frame launches of the benchmark's stream (sphere radius varying by frame) into 512^3, recast_step 2."""
    g = handle(512, 512, K=syn.K_DEPTH, recast_step=2)
    for start in (0, 64):
        d = np.stack([syn.scene_sphere(4.0 + 0.04 * ((((t % 256) * 7) % 11) - 5)) for t in range(start, start + 64)])
        Rs, Ts = syn.stream_poses(64, start=start)
        g.integrate_depth(d, Rs, Ts)
    ref = audit(g, [0], 1, 0.25)
    assert ref["tag"].shape[0] > 10000


# -- saturated output ------------------------------------------------------------------------------------------------
def test_saturation_step1(plane_map):
    g = plane_map
    rc, n, v, nrm, _ = generate(g, 1, 0.1, 1 << 20)
    assert rc == 0
    full = mcr.rows(v, nrm)
    assert np.array_equal(full[np.lexsort(full.T[::-1])], ref_rows(reference(g, [0], 1, 0.1)))
    raw = np.concatenate([v.reshape(-1, 9).view(np.uint32), nrm.reshape(-1, 9).view(np.uint32)], 1)
    for cap in (1, n // 3, n - 1):
        rc, demand, v2, n2, _ = generate(g, 1, 0.1, cap)
        assert rc == capi.E_CAPACITY and demand == n and v2.shape[0] == cap
        got = np.concatenate([v2.reshape(-1, 9).view(np.uint32), n2.reshape(-1, 9).view(np.uint32)], 1)
        assert np.array_equal(got, raw[:cap])  # the prefix of the full output, bit for bit


def test_saturation_generic(plane_map):
    g = plane_map
    ref = reference(g, [0], 2, 0.1)
    n = ref["tag"].shape[0]
    want = ref_rows(ref)
    for cap in (1, n // 3, n - 1):
        rc, demand, v, nrm, _ = generate(g, 2, 0.1, cap)
        assert rc == capi.E_CAPACITY and demand == n and v.shape[0] == cap
        assert mcr.rows_in(mcr.rows(v, nrm), want).all()


# -- the incremental mesh --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["plane", "two_submaps"])
def test_mesh_cache_matches_reference(plane_map, two_map, which):
    import torch
    from taichislam_b200.mesh_handle import MeshCache
    g, subs = (plane_map, [0]) if which == "plane" else (two_map, [0, 1023])
    ref = reference(g, subs, 1, 0.1)
    n = ref["tag"].shape[0]
    cap = n + 4096
    dev = torch.device("cuda", torch.cuda.current_device())
    v = torch.empty((3 * cap, 3), dtype=torch.float32, device=dev)
    nrm = torch.empty((3 * cap, 3), dtype=torch.float32, device=dev)
    c = MeshCache(g)
    demand, rc = c.update_into(0.1, cap, v, nrm)
    c.close()
    assert rc == 0 and demand == n
    got = mcr.sorted_rows(v[:3 * n].cpu().numpy(), nrm[:3 * n].cpu().numpy())
    assert np.array_equal(got, ref_rows(ref))
