"""CPU: the oracle's Matcher::findEpipolarMatchDirect and DepthFilter::updateSeeds under every Matcher::Options setting
(oracle/svo_oracle_epipolar.cpp) pinned bit for bit against the compiled reference's own matcher.cpp and depth_filter.cpp
with options_ set (oracle/ref_wrap_epipolar.cpp, recorded in tests/golden/ref/test_epipolar_options_pins.npz), on the grid
of tests/epipolar_options_cases.py."""
import math

import numpy as np
import pytest

from oracle import binding, binding_epipolar
from tests import epipolar_options_cases as ec
from tests.ref_golden import ref  # noqa: F401 (ref: fixture)

CAMS = list(ec.CAMERAS)


@pytest.fixture(scope="module")
def epi():
    binding_epipolar.build()
    return binding_epipolar


def _same(a, b):
    """Equal as f64 bit patterns, any NaN equal to any NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)].view(np.uint64),
                                                                        b[~np.isnan(b)].view(np.uint64))


def _check_match(o, r, what):
    """Outcome, branch and h_inv_ bit for bit; the f64 geometry at the tolerances of the default matcher's pins
    (tests/test_oracle_pins.py): the oracle sums without the reference build's contractions, a few ulp apart."""
    assert o["success"] == r["success"] and o["reject"] == r["reject"], what
    assert o["search_level"] == r["search_level"], what
    assert o["ran_1d"] == r["ran_1d"], what
    assert _same(o["h_inv"], r["h_inv"]), (what, o["h_inv"], r["h_inv"])
    assert np.isclose(o["epi_length"], r["epi_length"], rtol=1e-9, atol=0), what
    assert np.allclose(o["A_cur_ref"], r["A_cur_ref"], rtol=1e-9, atol=1e-12), what
    assert np.allclose(o["px_cur"], r["px_cur"], rtol=0, atol=1e-9, equal_nan=True), (what, o["px_cur"], r["px_cur"])
    assert np.isclose(o["depth"], r["depth"], rtol=1e-9, atol=0), (what, o["depth"], r["depth"])


def _runs(name):
    """(candidate, label, options) of the grid: every candidate at the eight flag settings, the edgelets at the angles."""
    c = ec.candidates(name)
    for label, opt in ec.settings():
        default_angle = opt["edgelet_max_angle"] == 0.7
        for j in range(len(c["kind"])):
            if default_angle or c["ftr_type"][j] == 1:
                yield j, label, opt


@pytest.mark.parametrize("name", CAMS)
def test_epipolar_options_oracle_equals_reference(epi, ref, name):
    c = ec.candidates(name)
    seen = {"reject": 0, "ran_1d": 0, "nan_h_inv": 0, "success_no_subpix": 0}
    for j, label, opt in _runs(name):
        o = ec.oracle_match(epi, name, j, opt)
        r = ec.ref_match(ref, name, j, opt)
        _check_match(o, r, (name, j, c["kind"][j], label))
        seen["reject"] += o["reject"]
        seen["ran_1d"] += o["ran_1d"]
        seen["nan_h_inv"] += o["ran_1d"] and math.isnan(o["h_inv"])
        seen["success_no_subpix"] += o["success"] and not opt["subpix_refinement"] and c["kind"][j] == "scan"
    print(name, seen)
    assert all(v > 0 for v in seen.values()), seen


@pytest.mark.parametrize("name", CAMS)
def test_epipolar_options_the_zero_length_line(epi, ref, name):
    """d_min == d_max: px_A == px_B, epi_length 0, the short-line branch.  With align_1d the direction is (0, 0) / 0 = NaN:
    align1D runs with it, sets a NaN h_inv_ and fails, so the match fails with px_cur_ at the segment's point -- in the
    reference as in the oracle."""
    c = ec.candidates(name)
    for j in [j for j, k in enumerate(c["kind"]) if k == "zero"][:6]:
        opt = dict(binding_epipolar.DEFAULTS, align_1d=True, edgelet_filtering=False)
        o = ec.oracle_match(epi, name, j, opt)
        r = ec.ref_match(ref, name, j, opt)
        _check_match(o, r, (name, j))
        assert o["epi_length"] == 0.0 and o["ran_1d"] and math.isnan(o["h_inv"]) and not o["success"]


def _ref_cosangle(ref, name, j, base):
    """The reference's cosangle of candidate j: the largest angle its filter keeps the edgelet at, found by bisecting the
    doubles of [0, 1] with reference calls (each call's angle follows from the previous outputs, so the recorded outputs
    replay the same sequence)."""
    lo, hi = np.float64(0.0).view(np.int64), np.float64(1.0).view(np.int64)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if ec.ref_match(ref, name, j, dict(base, edgelet_max_angle=float(np.int64(mid).view(np.float64))))["reject"]:
            hi = mid
        else:
            lo = mid
    return float(np.int64(lo).view(np.float64))


@pytest.mark.parametrize("name", CAMS)
def test_epipolar_options_edgelet_angle_at_cosangle(epi, ref, name):
    """The filter compares cosangle < max_angle strictly: at max_angle == cosangle the edgelet is kept, at the next double
    above (cosangle is then the next double below the angle) it is rejected -- in the reference and in the oracle, each at
    its own cosangle.  The two cosangles are a few hundred ulp apart at most (A_cur_ref_ and epi_dir_ round differently in
    the last bits, as the default pins' 1e-9 tolerance on A_cur_ref_ allows), so an angle within that margin of an
    edgelet's cosangle is the one setting on which the oracle and the reference may disagree."""
    n = 0
    for j in ec.threshold_candidates(name):
        for a1 in (False, True):
            base = dict(binding_epipolar.DEFAULTS, align_1d=a1)
            assert not ec.oracle_match(epi, name, j, dict(base, edgelet_max_angle=0.0))["reject"]
            assert ec.oracle_match(epi, name, j, dict(base, edgelet_max_angle=1.0))["reject"]
            rc, oc = _ref_cosangle(ref, name, j, base), ec.cosangle_threshold(epi, name, j, base)
            assert abs(rc - oc) <= 1e-12 * oc, (name, j, rc, oc)
            for cos, run in ((rc, lambda o: ec.ref_match(ref, name, j, o)), (oc, lambda o: ec.oracle_match(epi, name, j, o))):
                kept = run(dict(base, edgelet_max_angle=cos))
                rejected = run(dict(base, edgelet_max_angle=float(np.nextafter(cos, 2.0))))
                assert not kept["reject"] and rejected["reject"] and not rejected["success"], (name, j, cos)
                n += 1
    assert n == 8


@pytest.mark.parametrize("name", CAMS)
def test_epipolar_options_defaults_are_the_default_oracle(epi, name):
    """At the defaults (and with align_1d alone, which the existing oracle entry point takes) the options oracle is the
    existing one bit for bit."""
    s, c = ec.scene(name), ec.candidates(name)
    for j in range(len(c["kind"])):
        r = int(c["ref_index"][j])
        T = ec.synth.se3_mul(s["T_cur_w"], ec.synth.se3_inv(s["kf_T"][r]))
        for a1 in (False, True):
            o = ec.oracle_match(epi, name, j, dict(binding_epipolar.DEFAULTS, align_1d=a1))
            b = binding.find_epipolar_match_direct(s["kf_pyr"][r], s["cur_pyr"], s["cam"], T, c["ftr_px"][j], c["ftr_f"][j],
                                                   int(c["ftr_level"][j]), int(c["ftr_type"][j]), c["ftr_grad"][j],
                                                   c["d_est"][j], c["d_min"][j], c["d_max"][j], ec.N_LEVELS - 1, align_1d=a1)
            for k in ("success", "reject", "search_level", "n_zmssd"):
                assert o[k] == b[k], (j, k)
            for k in ("epi_length", "px_cur", "depth", "h_inv", "A_cur_ref"):
                assert _same(o[k], b[k]), (j, k)
    k = ec.seeds(name)
    o = ec.oracle_update(epi, name, None)
    b = binding.depth_filter_update(s["kf_pyr"], s["kf_T"], s["cur_pyr"], s["T_cur_w"], s["cam"], k["ref_index"], k["ftr_px"],
                                    k["ftr_f"], k["ftr_level"], k["ftr_type"], k["ftr_grad"], k["batch_id"], k["batch_counter"],
                                    k["seeds"], max_search_level=ec.N_LEVELS - 1)
    for key in ("a", "b", "mu", "sigma2", "status", "px_cur", "z", "n_zmssd"):
        assert np.array_equal(o[key], b[key]), key


def _ref_status(st):
    """The oracle's per-seed status as the reference wrapper reports it: 1 converged, 2 erased otherwise, 0 kept."""
    return np.where(st == 6, 1, np.where((st == 1) | (st == 7), 2, 0)).astype(np.uint8)


DF_SETTINGS = [(lab, opt) for lab, opt in ec.settings() if opt["edgelet_max_angle"] == 0.7 or lab.startswith("a1s0")]


@pytest.mark.parametrize("name", CAMS)
def test_depth_filter_options_oracle_equals_reference(epi, ref, name):
    """DepthFilter::updateSeeds with matcher_.options_ set, two keyframes: statuses, and a, b, mu, sigma2 of every kept
    seed bit for bit (of the converged ones sigma2 as the callback received it)."""
    moved = 0
    d = ec.oracle_update(epi, name, None)
    for label, opt in DF_SETTINGS:
        o = ec.oracle_update(epi, name, opt)
        r = ec.ref_update(ref, name, opt)
        assert np.array_equal(_ref_status(o["status"]), r["status"]), label
        assert (o["status"] >= 5).sum() > 5, label
        for k in ("a", "b", "mu", "sigma2"):  # kept seeds; of the converged ones sigma2 (the erased seed's other fields are gone)
            m = r["status"] != 2 if k == "sigma2" else r["status"] == 0
            assert np.array_equal(o[k][m].view(np.uint32), r[k][m].view(np.uint32)), (label, k)
        moved += not np.array_equal(o["mu"], d["mu"])
    assert moved >= 4  # the options change the filter's result
