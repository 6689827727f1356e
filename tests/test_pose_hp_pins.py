"""CPU: the high-precision statement of pose_optimizer::optimizeGaussNewton (tests/pose_hp.py) against the oracle and
the compiled reference's recorded outputs on the case catalogue of tests/pose_hp_cases.py, and against itself at 60
digits; and that every catalogue case is pinned by the statement (a finite bound, no open culling test).

The oracle and the reference take the median of a vector holding a NaN with std::nth_element; where that NaN's place
decides the median (pose_hp_cases.NAN_MEDIAN), the statement -- and the kernel -- sort NaN above +inf instead, so only the
medians are left out there."""
import math

import numpy as np
import pytest
from mpmath import mp

from rpg_svo_b200 import synth
from tests import pose_hp as hp
from tests import pose_hp_cases as pc
from tests.ref_golden import RefCalls

CASES = pc.all_cases()
# cases whose last decisions are near-ties (a chi2 comparison within its uncertainty once the steps are rounding-sized):
# the kernel may take either branch, each within its own bound
NEAR_TIES = {"n40", "n512", "n513", "iters30", "rollback_at_switch"}
# cases that end in a roll-back and whose covariance -- the inverse of the rejected iteration's A -- the statement pins
ROLLBACK_COV = {"rollback_at_switch", "n511", "iters30", "z_2^-130", "z_2^128", "behind"}


def _without_nan_medians(o, r):
    return dict(o, estimated_scale=r["est_out"], error_init=r["error_init"][0], error_final=r["error_final"][0])


def reference_outputs(r):
    """The compiled reference's outputs on every catalogue case, in catalogue order (recorded or replayed by r)."""
    return [r.pose_optimize(*pc.ref_args(c)) for c in CASES]


def same_as_reference(g, rr, c):
    """An implementation's outputs g against the reference's rr on case c: flags and counts exact, the scalars to 1e-9
    relative (error_final with a 1e-9 px floor: where the observations are fitted exactly it is rounding noise), the pose
    to 1e-8 where A has full rank, the covariance where A is invertible and was formed (n_iter > 0 and an observation:
    the reference leaves Cov_ as it was otherwise)."""
    name = c["name"]
    assert np.array_equal(g["has_point"], rr["has_point"]) and g["num_obs"] == rr["num_obs"], name
    if name not in pc.NAN_MEDIAN:
        for k in ("estimated_scale", "error_init", "error_final"):
            floor = 1e-9 if k == "error_final" else 0.0
            rel = 1e-3 if name in pc.NOISE_FREE else 1e-9
            assert abs(g[k] - rr[k]) <= rel * abs(rr[k]) + floor or (math.isnan(g[k]) and math.isnan(rr[k])), (name, k, g[k], rr[k])
    assert np.array_equal(np.isfinite(g["T"]), np.isfinite(rr["T"])), name
    if name not in pc.RANK_DEFICIENT and np.isfinite(rr["T"]).all():
        dt, dr = synth.pose_error(g["T"], rr["T"])
        assert dt < 1e-8 and dr < 1e-8, (name, dt, dr)
    if c["args"][1] > 0 and c["args"][7].any() and name not in pc.RANK_DEFICIENT and np.isfinite(rr["cov"]).all():
        # noise-free frames: the Tukey weights of ~1e-11 errors are known to ~1e-4, and A and its inverse with them
        assert np.allclose(g["cov"], rr["cov"], rtol=1e-3 if name in pc.NOISE_FREE else 1e-6, atol=1e-12), name


def test_pose_oracle_matches_reference(oracle):
    """The oracle against the compiled reference's outputs on every case (recorded with SVO_REF_RECORD; the replay checks
    that the inputs hash to the recorded ones)."""
    r = RefCalls("test_pose_hp_pins", "test_pose_oracle_matches_reference")
    refs = reference_outputs(r)
    r.finish()
    for c, rr in zip(CASES, refs):
        same_as_reference(oracle.pose_optimize(*c["args"]), rr, c)


@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_pose_statement_matches_oracle(oracle, name):
    c = next(x for x in CASES if x["name"] == name)
    runs = hp.branches(*c["args"], exact=c["exact"])
    o = oracle.pose_optimize(*c["args"])
    if name in pc.NAN_MEDIAN:
        o = _without_nan_medians(o, runs[0])
    if name in pc.RANK_DEFICIENT:
        hp.assert_rank_deficient(o, runs[0])
        return
    run, ratio, why = hp.match_any(o, runs, c["args"][2])
    assert run is not None, (name, why, ratio)
    if hp.decisive(runs[0]) and name not in pc.RANK_DEFICIENT:
        assert run is runs[0], name
    ok, cratio, checked = hp.cov_check(o, run, c["args"][2])
    assert ok, (name, cratio)
    if name in ROLLBACK_COV:
        assert checked and run["trace"][-1]["decision"] == "rollback", name


@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_pose_catalogue_case_is_pinned(name):
    """Every case has a finite bound far below its pose's size and no culling test left open; the pose is bounded
    wherever A has full rank; every case but the named near-ties is decisive."""
    c = next(x for x in CASES if x["name"] == name)
    runs = hp.branches(*c["args"], exact=c["exact"])
    r = runs[0]
    assert hp.defined(r) and r["bound"] < 1e-6, (name, r["bound"])
    assert not r["cull_open"].any(), name
    assert name in NEAR_TIES or name in pc.RANK_DEFICIENT or hp.decisive(r), (name, [x["tie"] for x in r["trace"]])
    full_rank = all(rec["cond"] < 1e12 for rec in r["trace"] if not math.isnan(rec["cond"]))
    assert full_rank or name in pc.RANK_DEFICIENT, name


@pytest.mark.parametrize("name", ["iters7", "n41", "rollback_at_switch"])
def test_pose_statement_at_60_digits(name):
    """Away from the branch points the 40-digit statement is the exact iteration: 60 digits move its pose by far less
    than the kernel's bound."""
    c = next(x for x in CASES if x["name"] == name)
    r40 = hp.optimize(*c["args"])
    old = mp.dps
    try:
        mp.dps = 60
        r60 = hp.optimize(*c["args"])
    finally:
        mp.dps = old
    assert [x["decision"] for x in r40["trace"]] == [x["decision"] for x in r60["trace"]]
    d = max(abs(a - b) for ra, rb in zip(r40["R"], r60["R"]) for a, b in zip(ra, rb))
    d = max(d, max(abs(a - b) for a, b in zip(r40["t"], r60["t"])))
    assert float(d) < 1e-30, float(d)
    assert math.isfinite(r40["bound"])


def test_pose_every_ending_occurs():
    """The five ways optimizeGaussNewton ends, each reached decisively by some case at full rank: the EPS stop, the
    roll-back on chi2, the roll-back on a NaN step, n_iter exhausted, and no observations."""
    ends = {"stop": [], "rollback": [], "nan": [], "out_of_iterations": [], "empty": []}
    for c in CASES:
        r = hp.branches(*c["args"], exact=c["exact"])[0]
        if r["empty"]:
            ends["empty"].append(c["name"])
        elif r["trace"] and hp.decisive(r) and c["name"] not in pc.RANK_DEFICIENT:
            ends[r["trace"][-1]["decision"]].append(c["name"])
    print("decisive endings:", ends)
    assert all(ends.values()), ends
