"""CPU: the oracle's robust-cost SparseImgAlign (orc_sparse_img_align_robust: MAD scale with unit, Tukey or Huber weights)
against the compiled reference's own SparseImgAlign with setRobustCostFunction set (oracle/_ref, recorded in
tests/golden/ref/test_sia_robust_pins.npz) on the cases of tests/sia_robust_cases.py."""
import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import sia_robust_cases as rc
from tests.ref_golden import ref  # noqa: F401 (ref: fixture)

NAMES = [k["name"] for k in rc.cases()]


@pytest.mark.parametrize("name", [n for n in NAMES if n not in rc.NO_REF])
def test_robust_oracle_equals_reference(oracle, name, ref):
    """Mask, patch count and per-level scales bit for bit, pose within 1e-9, H within the residual pin's 1e-9 (NaN where
    the reference has NaN).  Fewer than RANK_OK features: the mask, the count and the first level's scale."""
    k = rc.case(name)
    o = rc.oracle_run(k)
    r = rc.ref_run(ref, k)
    p = k["p"]
    n = len(p["px"])
    assert o["n_tracked"] == r["n_tracked"]
    assert np.array_equal(o["visible"], r["visible"][:n])
    if 0 < n < rc.RANK_OK:  # rank-deficient H: only what the initial pose decides (the first level's scale)
        assert rc.same_bits(o["scales"][k["max_level"]], r["scales"][k["max_level"]])
        return
    assert rc.same_bits(o["scales"], r["scales"]), (o["scales"], r["scales"])
    assert np.allclose(r["T_cur_w"], synth.se3_mul(o["T"], p["T_ref_w"]), rtol=0, atol=1e-9)
    if name not in rc.NO_H and n >= rc.RANK_OK:
        assert np.array_equal(np.isnan(o["H"]), np.isnan(r["H"]))
        m = ~np.isnan(o["H"])
        assert np.allclose(r["H"][m], o["H"][m], rtol=1e-9, atol=1e-9)


def test_robust_scale_rules_seen_on_the_oracle(oracle):
    """The [EXT] rules the cases are built to show: with 30 iterations the coarsest level's scale carries through every
    finer level; with none, every level recomputes it and run() returns what the pre-passes counted; a MAD scale of 0 makes
    every Tukey weight 0 (x = 0, accepted) and Huber's H NaN (stop_ latches, every pass rejected)."""
    s30 = rc.oracle_run(rc.case("tukey"))["scales"][:5]
    assert np.all(s30 == s30[4]) and s30[4] > 0
    o0 = rc.oracle_run(rc.case("iters_0"))
    assert len(np.unique(o0["scales"][:5])) == 5 and o0["n_tracked"] > 4 * rc.oracle_run(rc.case("tukey"))["n_tracked"]
    t = rc.oracle_run(rc.case("zero_median_tukey"))
    assert np.all(t["scales"][:5] == 0) and all(x["accepted"] and not np.any(x["x"]) for x in t["trace"])
    assert [x["iter"] for x in t["trace"]] == [0] * 5
    h = rc.oracle_run(rc.case("zero_median_huber"))
    assert np.isnan(h["H"]).all() and not any(x["accepted"] for x in h["trace"]) and len(h["trace"]) == 5


def test_robust_no_patch_keeps_the_scale(oracle):
    """No patch in the image: the scale stays at its initial 0 (not pinned against the reference), the pose at the start."""
    o = rc.oracle_run(rc.case("no_points"))
    assert o["n_tracked"] == 0 and np.all(o["scales"][:5] == 0) and np.allclose(o["T"], synth.se3_identity())


def test_robust_tukey_beats_plain_gauss_newton_on_occlusion(oracle):
    """A quarter of the features occluded in the current image: Tukey ends far closer to the ground-truth pose than plain
    Gauss-Newton (observed: 1.8e-3 m against 1.3 m)."""
    k = rc.case("occluded_tukey")
    p = k["p"]
    gt = p["T_cur_ref_gt"]
    e_t = synth.pose_error(rc.oracle_run(k)["T"], gt)[0]
    u = oracle.sparse_img_align(p["ref_pyr"], p["cur_pyr"], p["cam"], synth.se3_identity(), p["px"], p["f"], p["pos"],
                                p["has_point"], p["ref_pos"], 4, 0)
    e_u = synth.pose_error(u["T"], gt)[0]
    assert e_t < 0.01 and e_u > 0.5, (e_t, e_u)


def test_robust_unit_weight_equals_plain_gauss_newton(oracle):
    """MAD with unit weights is plain Gauss-Newton: the same pose bit for bit as the unweighted oracle."""
    k = rc.case("unit")
    p = k["p"]
    u = oracle.sparse_img_align(p["ref_pyr"], p["cur_pyr"], p["cam"], synth.se3_identity(), p["px"], p["f"], p["pos"],
                                p["has_point"], p["ref_pos"], 4, 0)
    assert np.array_equal(rc.oracle_run(k)["T"], u["T"])
