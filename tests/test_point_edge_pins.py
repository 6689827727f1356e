"""CPU: the point optimizer's oracle (orc_point_optimize) against the compiled reference's Point::optimize (recorded in
tests/golden/ref/test_point_edge_pins.npz) and against the high-precision statement of tests/point_hp.py, on the
degenerate and non-finite points of tests/point_cases.py."""
import numpy as np
import pytest

from tests import point_cases as pc
from tests import point_hp as hp
from tests.ref_golden import ref  # noqa: F401 (fixture)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def test_point_edge_cases_oracle_equals_reference(oracle, ref):
    """For every case: the oracle and the reference agree on which coordinates are finite; both end where one of the
    exact runs the kernel may take ends (tests/point_hp.branches) -- bit for bit where that run returns the untouched
    start, within the run's bound where that bound is defined (see point_hp.defined).  Where it is not, the step divided by
    a pivot that is rounding noise (one camera centre, the 4 um baseline): the stand-in's Eigen LDLT and the oracle's
    then end metres apart along the ray, and only finiteness is defined."""
    refs = pc.ref_outputs(ref)
    seen = {}
    for (name, n_iter, s, Ts, fs), r in zip(pc.edge_cases(), refs):
        o = oracle.point_optimize(n_iter, s, Ts, fs)
        assert np.array_equal(np.isfinite(o), np.isfinite(r)), (name, o, r)
        runs = hp.branches(n_iter, s, Ts, fs)
        for who, x in (("oracle", o), ("reference", r)):
            run, ratio = hp.match_any(x, runs)
            assert run is not None, (name, who, x, [hp.as_float(q) for q in runs], ratio)
        if runs[0]["untouched"] and hp.decisive(runs[0]):
            assert np.array_equal(_bits(o), _bits(s)) and np.array_equal(_bits(r), _bits(s)), name
        seen[name] = [rec["decision"] for rec in runs[0]["trace"]]
    print({k: v for k, v in seen.items()})


@pytest.mark.parametrize("name", ["one_centre_axis", "baseline_0.26", "baseline_0.008", "baseline_0.00026", "baseline_8e-06",
                                  "start_z0", "bearing_fz0", "start_nan", "pose_t_inf"])
def test_point_edge_cases_reach_their_branches(name):
    """Each case reaches what it was built for, in the exact trace: the exactly-zero pivot on the common optical axis
    (its component of the step is 0, the other two are not), cond(A) of ~1e3 / 1e6 / 1e9 / 1e12 for the four baselines,
    a NaN step at iteration 0 for a start at z = 0, a bearing with f_z = 0 and a NaN start, a finite run past an infinite
    pose translation (that observation's Jacobian and residual are 0 and 0 - 0)."""
    case = {c[0]: c for c in pc.edge_cases()}[name]
    _, n_iter, s, Ts, fs = case
    r = hp.optimize(n_iter, s, Ts, fs)
    t0 = r["trace"][0]
    if name == "one_centre_axis":
        assert t0["pivots"][2] == 0 and t0["dp"][2] == 0 and t0["dp"][0] != 0
        assert hp.decisive(r) and r["trace"][-1]["decision"] == "out_of_iterations"
    elif name.startswith("baseline_"):
        want = {"0.26": 1e3, "0.008": 1e6, "0.00026": 1e9, "8e-06": 1e12}[name.split("_")[1]]
        assert want / 3 <= t0["cond"] <= want * 3, t0["cond"]
        if name == "baseline_0.00026":  # the second step overshoots: chi2 rises, decisively
            assert hp.decisive(r) and [x["decision"] for x in r["trace"]] == ["step", "rollback"]
    elif name == "pose_t_inf":
        assert all(np.isfinite(hp.as_float(r))) and r["trace"][-1]["decision"] == "stop"
    else:
        assert [x["decision"] for x in r["trace"]] == ["nan"] and r["untouched"]
