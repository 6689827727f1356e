"""CPU: the robust-cost oracle on the edge cases of tests/sia_robust_edge_cases.py, against the compiled reference's own
SparseImgAlign with setRobustCostFunction set (oracle/_ref, recorded in tests/golden/ref/test_sia_robust_edge_pins.npz) on
the cases that start from a pyramid the reference builds itself, and its MAD scale against an exact numpy median on every
case."""
import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import sia_cases as sc
from tests import sia_robust_cases as rc
from tests import sia_robust_edge_cases as ec
from tests.ref_golden import ref  # noqa: F401 (ref: fixture)

NAMES = ec.names()


@pytest.mark.parametrize("name", [n for n in NAMES if n not in ec.NO_REF])
def test_robust_edge_oracle_equals_reference(oracle, name, ref):
    """As test_sia_robust_pins.py: mask, patch count and per-level scales bit for bit, pose within 1e-9, H within 1e-9 (NaN
    where the reference has NaN)."""
    k = ec.case(name)
    o = ec.oracle_run(k)
    r = ec.ref_run(ref, k)
    p = k["p"]
    n = len(p["px"])
    assert o["n_tracked"] == r["n_tracked"]
    assert np.array_equal(o["visible"], r["visible"][:n])
    assert rc.same_bits(o["scales"], r["scales"]), (o["scales"], r["scales"])
    assert np.allclose(r["T_cur_w"], synth.se3_mul(o["T"], p["T_ref_w"]), rtol=0, atol=1e-9)
    if name not in ec.NO_H:
        assert np.array_equal(np.isnan(o["H"]), np.isnan(r["H"]))
        m = ~np.isnan(o["H"])
        assert np.allclose(r["H"][m], o["H"][m], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("name", NAMES)
def test_robust_edge_scale_is_the_exact_median(oracle, name):
    """scale_ = 1.48 * the upper median of the f32 |res| of the in-image patches at T0 (numpy's partition), bit for bit, at
    the first level and -- n_iter 0 -- at every level; 0 (the initial scale_) where no patch is in the image."""
    k = ec.case(name)
    o = ec.oracle_run(k)
    for level, m in ec.numpy_scales(oracle, k).items():
        assert rc.same_bits(o["scales"][level], np.float32(0.0) if m is None else m), (level, o["scales"][level], m)


@pytest.mark.parametrize("name", NAMES)
def test_robust_edge_case_decisions_are_clear(name):
    """No Gauss-Newton decision of the oracle's run is within ec.MARGIN of flipping (the cases' seeds are chosen so), so
    test_sia_robust_edges_gpu.py compares the kernel's whole trace, H and pose with the oracle's."""
    k = ec.case(name)
    if len(k["p"]["px"]) >= rc.RANK_OK:
        assert sc.decision_margin(ec.oracle_run(k)) >= ec.MARGIN, ec.seed_of(name)


def test_robust_edge_cases_reach_their_edges(oracle):
    """What the cases are built to show, on the oracle: slot-edge features are tracked in the live variant and not where
    has_point is cleared; features one pixel past the coarsest level's admissible border are not visible there but are at
    level 0; the strip case sees no patch at level 4 (scale 0) and recomputes the scale at level 3; two grey values give a
    MAD scale of exactly 0 with more than half the residuals 0, four give a positive one with
    ties (over a third of the level-0 residuals repeat a value)."""
    edges = [e for e in ec.ROBUST_EDGES if e < 1024]
    live = ec.oracle_run(ec.case("slots_1024_live_tukey"))["visible"]
    assert live[edges].all() and not ec.oracle_run(ec.case("slots_1024_tukey"))["visible"][edges].any()
    k = ec.case("admissible_tukey")
    p = k["p"]
    inner = oracle.sparse_residuals(p["ref_pyr"][4], p["cur_pyr"][4], 4, p["cam"], k["T0"], p["px"], p["f"], p["pos"],
                                    p["has_point"], p["ref_pos"])
    assert inner["visible"][150:198].all() and not inner["visible"][198:].any()
    assert ec.oracle_run(k)["visible"][198:].all()
    for n_iter in (0, 30):
        s = ec.oracle_run(ec.case(f"coarse_empty_iters_{n_iter}"))["scales"]
        assert s[4] == 0 and s[3] > 0
    k2, k4 = ec.case("ties_2_tukey"), ec.case("ties_4_tukey")
    assert np.all(ec.oracle_run(k2)["scales"][:5] == 0)
    p = k4["p"]
    r = oracle.sparse_residuals(p["ref_pyr"][0], p["cur_pyr"][0], 0, p["cam"], k4["T0"], p["px"], p["f"], p["pos"],
                                p["has_point"], p["ref_pos"])
    a = np.abs(r["residuals"][r["in_image"].astype(bool)])
    assert ec.oracle_run(k4)["scales"][0] > 0 and a.size - len(np.unique(a)) > a.size // 3  # repeated values
