"""CPU: the oracle's align2D / align1D / findMatchDirect against the compiled reference (recorded outputs,
tests/golden/ref/test_align_pins.npz) on the edge cases of tests/align_cases.py, and the oracle's warp matrix and search
level against an independent float64 numpy statement.  The GPU edge tests (test_align_edges_gpu.py) replay the same
recorded outputs."""
import numpy as np
import pytest

from tests import align_cases as ac
from tests.ref_golden import ref  # noqa: F401 (ref: fixture)

ALIGN_NAMES = [c["name"] for c in ac.align_cases()]
# the compiled reference's Matcher keeps its default align_max_iter (10): the max_iter cases are the GPU tests' alone
MATCH_NAMES = [c["name"] for c in ac.match_cases() if c["align_max_iter"] == 10]

# Problems on which the oracle (and with it the kernels, which equal the oracle bit for bit) is known to end elsewhere than
# the compiled reference: (case, problem index, "1d" / "2d").  A patch constant along y, aligned in 1-D along a direction
# close to y, makes each step a division by a tiny H; the two agree bit for bit for three steps and part at the fourth,
# where a one-rounding difference is amplified into a different path (DESIGN.md 4.2).
KNOWN_ALIGN_DIFFS = {("singular", 15, "1d")}


def align_case(name):
    return next(c for c in ac.align_cases() if c["name"] == name)


def match_case(name):
    return next(c for c in ac.match_cases() if c["name"] == name)


def align_diffs(c, o, r):
    """{(case, index, "2d" / "1d")} where the oracle's outputs o and the reference's r are not bit-identical (NaN = NaN)."""
    conv2, px2, conv1, px1, h1 = r
    out = set()
    for i in range(len(conv2)):
        if conv2[i] != o["conv2"][i] or not ac.same_bits(px2[i], o["px2"][i]):
            out.add((c["name"], i, "2d"))
        if conv1[i] != o["conv1"][i] or not ac.same_bits(px1[i], o["px1"][i]) or not ac.same_bits(h1[i], o["h1"][i]):
            out.add((c["name"], i, "1d"))
    return out


@pytest.mark.parametrize("name", ALIGN_NAMES)
def test_align_case_oracle_equals_reference(oracle, name, ref):
    """px as bits (any NaN equals any NaN), converged and h_inv bit for bit."""
    c = align_case(name)
    o = ac.run_oracle_align(oracle, c)
    d = align_diffs(c, o, ac.run_ref_align(ref, c))
    assert d == {k for k in KNOWN_ALIGN_DIFFS if k[0] == name}, sorted(d)


def test_align_big_batch_sample_oracle_equals_reference(oracle, ref):
    c = ac.batch_problems(ac.BIG_BATCH)
    rows = ac.sample_rows(ac.BIG_BATCH)
    o = ac.run_oracle_align(oracle, c, rows)
    assert not align_diffs(c, o, ac.run_ref_align(ref, c, rows))


def check_match(o, r, c):
    """Where Point::getCloseViewObs rejects the point (a point at the reference camera centre, or between the cameras) the
    reference fails before the matcher; elsewhere o and r must agree."""
    seen = ac.close_view(c)
    assert not r["success"][~seen].any()
    o, r = ({k: v[seen] for k, v in x.items()} for x in (o, r))
    assert np.array_equal(o["success"], r["success"])
    assert np.array_equal(o["search_level"], r["search_level"])
    dA = np.abs(o["A_cur_ref"] - r["A_cur_ref"]).max(axis=(1, 2))
    assert np.all(dA <= 1e-12 * np.abs(r["A_cur_ref"]).max(axis=(1, 2))), dA.max(initial=0)  # relative to the largest entry
    either = o["success"] | r["success"]
    assert np.max(np.abs(o["px_cur"][either] - r["px_cur"][either]), initial=0.0) <= 1e-4
    assert np.array_equal(np.isnan(o["px_cur"]), np.isnan(r["px_cur"]))


@pytest.mark.parametrize("name", MATCH_NAMES)
def test_match_case_oracle_equals_reference(oracle, name, ref):
    """success and search level exactly, A to 1e-12 relative, px_cur to 1e-4 px where either succeeds."""
    c = match_case(name)
    check_match(ac.run_oracle_match(oracle, c), ac.run_ref_match(ref, c), c)


@pytest.mark.parametrize("n_ref", [3, 4])
def test_match_multi_ref_oracle_equals_reference(oracle, n_ref, ref):
    c = ac.multi_ref_case(n_ref)
    o = ac.run_oracle_match(oracle, c)
    check_match(o, ac.run_ref_match(ref, c), c)
    assert o["success"].sum() > 0.25 * c["M"]


def test_numpy_warp_statement_equals_oracle(oracle):
    """The float64 numpy statement of getWarpMatrixAffine / getBestSearchLevel (synth.Camera, no oracle) against the
    oracle on every matcher case: A to 1e-9 relative, the search level exactly; every level 0..4 is chosen somewhere.
    Candidates outside isInFrame never reach the warp: A and the search level stay 0."""
    levels, n_out = set(), 0
    for c in ac.match_cases() + [ac.multi_ref_case(3), ac.multi_ref_case(4)]:
        o = ac.run_oracle_match(oracle, c)
        for i in range(c["M"]):
            if not ac.in_frame(c, i):
                assert not o["A_cur_ref"][i].any() and o["search_level"][i] == 0 and not o["success"][i], (c["name"], i)
                n_out += 1
                continue
            A, s = ac.numpy_warp(c, i)
            assert np.allclose(A, o["A_cur_ref"][i], rtol=1e-9, atol=1e-12), (c["name"], i)
            assert s == o["search_level"][i], (c["name"], i)
            levels.add(s)
    assert levels == {0, 1, 2, 3, 4} and n_out > 0
