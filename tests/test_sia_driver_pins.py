"""CPU: the alignment oracle on the Gauss-Newton driver's corner cases (tests/sia_driver_cases.py) against the compiled
reference's own SparseImgAlign::run (oracle/_ref, recorded in tests/golden/ref/test_sia_driver_pins.npz), and the oracle's
iteration trace against the float64 statement of the driver: every pose update, roll-back, termination decision and 6x6
solve."""
import numpy as np
import pytest

from oracle import binding as ob
from rpg_svo_b200 import synth
from tests import sia_driver_cases as dc
from tests.ref_golden import ref  # noqa: F401 (ref: fixture)


@pytest.mark.parametrize("name", dc.REF_CASES)
def test_driver_oracle_equals_reference(name, ref):
    """Mask and patch count exact, the final pose within 1e-9 (1e-8 from the far starts; NaN where the reference's is), H of
    the last pass within 1e-9 (NaN where the reference's is) wherever an iteration ran.  Below RANK_OK features the pose
    is rounding noise of a (nearly) singular solve and is not compared."""
    k = dc.case(name)
    o = dc.oracle_run(k)
    r = dc.ref_run(ref, k)
    p = k["p"]
    n = len(p["px"])
    assert o["n_tracked"] == r["n_tracked"], (o["n_tracked"], r["n_tracked"])
    assert np.array_equal(o["visible"], r["visible"][:n])
    T = synth.se3_mul(o["T"], p["T_ref_w"])
    assert np.array_equal(np.isnan(T), np.isnan(r["T_cur_w"]))
    if n >= dc.RANK_OK and not np.isnan(T).any():
        far = name.startswith(("rollback", "large_angle")) or name == "zero_depth"
        assert np.allclose(T, r["T_cur_w"], rtol=0, atol=1e-8 if far else 1e-9)
    if o["trace"] and n >= dc.RANK_OK:
        assert np.array_equal(np.isnan(o["H"]), np.isnan(r["H"]))
        m = ~np.isnan(o["H"])
        assert np.allclose(r["H"][m], o["H"][m], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("name", dc.NAMES)
def test_driver_statement_holds_on_the_oracle(name):
    """The oracle's trace against the float64 statement: T_k = T_(k-1) exp(-x_k) to 1e-13 with |R^T R - I| <= 2e-15, the
    roll-backs bit for bit, the termination rule, and x = H^-1 Jres of the oracle's own residual pass to 1e-14 cond(H)
    (cond(H) <= 1e12).  The cases compared iteration by iteration are clear of near-ties (margin > dc.MARGIN)."""
    k = dc.case(name)
    o = dc.oracle_run(k)
    err, orth = dc.pose_update_errors(o["trace"], k["T0"])
    assert err <= 1e-13 and orth <= 2e-15, (err, orth)  # orth: 1.1e-15 after theta_above's steps of theta^2 up to 5
    dc.check_flags(o["trace"], k)
    p = k["p"]
    if len(p["px"]) >= dc.RANK_OK:
        assert dc.margin(o, k["eps"]) > dc.MARGIN, dc.margin(o, k["eps"])

    def residuals(level, T, vis):
        return ob.sparse_residuals(p["ref_pyr"][level], p["cur_pyr"][level], level, p["cam"], T, p["px"], p["f"], p["pos"],
                                   p["has_point"], p["ref_pos"], visible_in=vis)

    for e, kappa in dc.solve_errors(o["trace"], k, residuals):
        assert e <= 1e-14 * kappa, (e, kappa)


def test_driver_cases_reach_their_edges():
    """What the cases are built to show, on the oracle."""
    run = lambda name: dc.oracle_run(dc.case(name))  # noqa: E731
    assert run("iters_0")["trace"] == [] and run("iters_0")["n_tracked"] == 0 and not run("iters_0")["visible"].any()
    assert len(run("iters_neg")["trace"]) > 5 * 2  # no limit: the levels end by roll-back or eps
    assert [t["iter"] for t in run("iters_1")["trace"]] == [0] * 5
    assert all(len([t for t in run("eps_huge")["trace"] if t["level"] == lv]) == 1 for lv in range(5))
    for name in ("eps_zero", "eps_nan"):  # nothing stops a level but a roll-back or the limit (6 iterations)
        tr = run(name)["trace"]
        for lv in range(5):
            last = [t for t in tr if t["level"] == lv][-1]
            assert not last["accepted"] or last["iter"] == 5, (name, lv)
    for name in dc.ROLLBACK:
        tr = run(name)["trace"]
        assert not [t for t in tr if t["level"] == 4][-1]["accepted"]  # the first level rolls back ...
        dt, dr = synth.pose_error(run(name)["T"], dc.scene()["T_cur_ref_gt"])
        assert dt < 2e-3 and dr < 2e-3  # ... and the finer levels still converge
    for name in ("no_points", "nan_ref_pos", "nan_T0"):
        assert all(t["n_meas"] == 0 and not np.any(t["x"]) for t in run(name)["trace"]) and run(name)["n_tracked"] == 0
    assert [t["n_meas"] for t in run("coarse_empty")["trace"] if t["level"] == 4] == [0]
    z = run("zero_residual")["trace"]
    assert all(t["chi2"] == 0 and not np.any(t["x"]) for t in z) and len(z) == 5
    assert [t["iter"] for t in run("zero_eps_neg")["trace"]] == list(range(5)) * 5
    # the pivoted factorisation: H of the textureless pair is 0, one or two features give rank 2 / 4
    for name in ("textureless", "few_1", "few_2"):
        assert dc.min_pivot_ratio(run(name)["H"]) <= 1e-13, name
    assert np.linalg.matrix_rank(run("few_1")["H"]) == 2 and np.linalg.matrix_rank(run("few_2")["H"]) == 4
    first = next(t for t in run("large_angle")["trace"] if t["accepted"])
    assert first["iter"] == 0 and np.linalg.norm(first["x"][3:]) >= 0.5  # se3_exp's closed form, not the series
    zd = run("zero_depth")["trace"]
    assert len(zd) == 5 and all(np.isnan(t["x"][0]) and not t["accepted"] for t in zd)  # stop latched over the levels
    d = dc.case("behind")["p"]
    assert (d["f"][:, 2] < 0).sum() == 10 and run("behind")["n_tracked"] == 300  # behind the camera, still in the image
    assert run("far_proj")["n_tracked"] == 290
    # points at zero depth from the identity, and bearings with f_z == 0: never in the image, no NaN in H, tracked as the rest
    for name in ("zero_depth_id", "fz_zero"):
        o = run(name)
        assert o["visible"][dc.POISONED].all() and o["n_tracked"] == 295 and np.isfinite(o["H"]).all(), name
    # an accepted step just below / just above theta^2 = 0.25, where se3_exp changes form
    for name, lo, hi in (("theta_below", 0.24, 0.25), ("theta_above", 0.25, 0.26)):
        th2 = [float(t["x"][3:] @ t["x"][3:]) for t in run(name)["trace"] if t["accepted"]]
        assert any(lo <= v < hi for v in th2), (name, th2)
    for name in ("nan_px", "inf_px"):
        assert not run(name)["visible"][dc.POISONED].any()
    for name in ("nan_f", "inf_f", "nan_pos", "inf_pos"):
        assert run(name)["visible"][dc.POISONED].all() and run(name)["n_tracked"] == 295
