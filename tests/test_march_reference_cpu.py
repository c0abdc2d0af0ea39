"""The f64 march reference (tests/march_reference.py) pinned to the CPU oracle on every edge-case cloud of the audit,
before any GPU run trusts it: same voxel set, same per-voxel sample counts (recovered from W where every weight is a
power of two), same in-bounds and out-of-bounds sample totals, TSDF and W within the bounds of util.march_bounds.  The
textured path of the reference is pinned the same way, and its colour words to the oracle's colours exactly."""
import numpy as np
import pytest

from march_cases import CASES, make_case, reference_of
from util import as_dict_rows, compare_to_reference


def oracle_map(case, mode):
    from oracle.oracle import OracleTSDF
    vs, N, Nz = case["vs"], case["N"], case["Nz"]
    # num_voxel_per_blk_axis = 1 and a map scale half a voxel short of N*vs: N and Nz exactly as given
    return OracleTSDF(map_scale=[(N - 0.5) * vs, (Nz - 0.5) * vs], voxel_scale=vs, num_voxel_per_blk_axis=1,
                      max_ray_length=case["max_ray_length"], internal_voxels=case["internal_voxels"], is_global_map=True,
                      mode=mode)


@pytest.fixture(scope="module", params=sorted(CASES))
def case_ref(request):
    c = make_case(request.param)
    return c, reference_of(c)


def assert_pow2_counts(c, ref, oi, ot, ow):
    w = np.unique(ref["w32"])
    assert w.shape == (1,) and np.log2(w[0]) == np.round(np.log2(w[0]))
    _, _, ws = as_dict_rows(oi, ot, ow)
    free = ref["sw"] < 999.0
    assert free.mean() > 0.99
    assert np.array_equal(ws[free] / w[0], ref["count"][free]), "per-voxel sample counts differ"


@pytest.mark.parametrize("mode", ["canonical", "f32_literal"])
def test_reference_matches_oracle(case_ref, mode):
    from oracle.oracle import MODE_CANONICAL, MODE_F32_LITERAL
    c, ref = case_ref
    o = oracle_map(c, {"canonical": MODE_CANONICAL, "f32_literal": MODE_F32_LITERAL}[mode])
    assert (o.N, o.Nz) == (c["N"], c["Nz"])
    o.integrate_points(np.eye(3), c["T"], c["pts"])
    o.commit()
    st = o.stats()
    assert st["n_rays"] == ref["n_rays"] == c["pts"].shape[0]
    assert st["n_updates"] == ref["n_updates"] and st["n_oob"] == ref["n_oob"]
    oi, ot, ow, _ = o.gather()
    compare_to_reference((oi, ot, ow), ref, sequential=(mode == "f32_literal"), sharp=(mode == "canonical"))
    if c["pow2"]:
        assert_pow2_counts(c, ref, oi, ot, ow)


@pytest.mark.parametrize("name", sorted(CASES))
def test_textured_reference_matches_oracle(name):
    """The textured path of the reference against the canonical oracle with colours: same sample totals and voxel set,
    values within the textured bounds (sharp at the hottest voxel), colours equal wherever the reference's f32 and
    exact closeness bins agree on the winner - and they must agree almost everywhere."""
    from oracle.oracle import MODE_CANONICAL
    c = make_case(name)
    ref = reference_of(c, "textured")
    o = oracle_map(c, MODE_CANONICAL)
    o.set_color(True, True)
    o.integrate_points_rgb(np.eye(3), c["T"], c["pts"], c["rgb"])
    o.commit()
    st = o.stats()
    assert st["n_rays"] == ref["n_rays"] and st["n_updates"] == ref["n_updates"] and st["n_oob"] == ref["n_oob"]
    oi, ot, ow, _ = o.gather()
    compare_to_reference((oi, ot, ow), ref, sharp=name != "hot_bundle")
    if c["pow2"]:
        assert_pow2_counts(c, ref, oi, ot, ow)
    _, oc = as_dict_rows(oi, o.gather_color())
    bad = (oc != ref["color"]).any(1)
    assert not (bad & ~ref["color_amb"]).any(), f"{int(bad.sum())} colours differ from the reference's words"
    assert ref["color_amb"].mean() < (0.5 if c["pow2"] else 0.01)  # pow2: |ds| sits on the bin edges by construction
    assert len(np.unique(ref["color"], axis=0)) >= 5  # several colours compete: a wrong winner shows

def test_cases_reach_their_edges():
    """Each cloud exercises what it is there for (numbers from the reference alone)."""
    from march_reference import ray_setup
    hot = make_case("hot_bundle")
    ref = reference_of(hot)
    assert hot["pts"].shape[0] >= 20000 and ref["count"].max() >= 20000
    c = make_case("ties_and_axes")
    t = c["T"].astype(np.float64) / np.float32(c["vs"])
    assert np.all(t - np.floor(t) == 0.5)
    assert (c["pts"] == 0).any(1).sum() >= 300 and np.signbit(c["pts"][c["pts"] == 0]).sum() >= 100
    c = make_case("short_rays")
    r = ray_setup(c["pts"], c["vs"], c["internal_voxels"], c["max_ray_length"])
    assert np.all(c["internal_voxels"] * c["vs"] > r["L"])
    c = make_case("anisotropic")
    assert c["N"] % 16 and c["Nz"] % 16 and c["N"] != c["Nz"] and reference_of(c)["n_oob"] > 0
    c = make_case("tiny_weights")
    ref = reference_of(c)
    r = ray_setup(c["pts"], c["vs"], c["internal_voxels"], c["max_ray_length"])
    assert 0 < r["tiny"].sum() < r["tiny"].shape[0] and ref["n_tiny"] > 0
    c = make_case("fine_long")
    assert c["max_ray_length"] / c["vs"] > 60000
    assert np.all(np.abs(np.round(c["pts"] / np.float32(c["vs"]))) <= 4095)  # inside the bucket key range
    ref = reference_of(c)
    assert ref["n_updates"] > 0 and ref["n_oob"] > ref["n_updates"]
    c = make_case("long_range")
    r = ray_setup(c["pts"], c["vs"], c["internal_voxels"], c["max_ray_length"])
    assert c["pts"].shape[0] == 20000 and np.all((r["L"] >= 55.0) & (r["L"] <= 60.0)) and c["max_ray_length"] == 64.0
    ref = reference_of(c, "textured")
    assert ref["nwin"].max() >= 1000 and r["w32"].max() < 4e-4  # thousands of tiny weights in one window voxel
    c = make_case("near_sensor")
    r = ray_setup(c["pts"], c["vs"], c["internal_voxels"], c["max_ray_length"])
    assert c["internal_voxels"] == 40 and np.all((r["L"] >= 0.05) & (r["L"] <= 0.12))
    assert 0 < (r["w32"] >= 120.0).sum() < r["w32"].shape[0]
    ref = reference_of(c, "textured")
    assert np.any(r["w32"][:, None] * (r["L"][:, None] - np.arange(1, 19) * c["vs"]) <= -120.0)  # samples with |w*ds| >= 120
