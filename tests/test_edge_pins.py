"""CPU: the oracle against the compiled reference (recorded outputs, tests/golden/ref/test_edge_pins.npz) at corners the
older pins do not cover -- degenerate pose problems and seeds in every DepthFilter status, bad variances included.  The GPU
tests of the same corners (test_pose_edges_gpu.py, test_depth_edges_gpu.py) replay these recorded outputs too."""
import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests.ref_golden import ref  # noqa: F401 (ref: fixture)
from tests.pose_cases import args, degenerate_cases, first_normal_matrix, zero_error_case


@pytest.mark.parametrize("idx", range(6))
def test_pose_degenerate_oracle_equals_reference(oracle, idx, ref):
    """1 and 2 observations, points on one 3D line, and observations in a 20, 4 and 1 px window of a distant plane: the
    oracle's pivoted LDL^T against Eigen's in the reference.  Both are backward-stable solves of the same A, so the poses
    agree to ~cond(A) * eps relative to the step."""
    name, c = degenerate_cases()[idx]
    r = ref.pose_optimize(*(args(c)[:2] + (c["cam"],) + args(c)[3:]))
    o = oracle.pose_optimize(*args(c))
    assert np.array_equal(r["has_point"], o["has_point"]) and r["num_obs"] == o["num_obs"], name
    cond = np.linalg.cond(first_normal_matrix(c))
    step = max(synth.pose_error(o["T"], c["T_init"]))
    bound = 1e-10 + 100 * cond * 2.2e-16 * max(step, 1e-6)
    dt, dr = synth.pose_error(r["T"], o["T"])
    assert dt <= bound and dr <= bound, (name, dt, dr, bound)
    assert np.array_equal(np.isfinite(r["cov"]), np.isfinite(o["cov"])), name
    for k in ("estimated_scale", "error_init"):  # before the first solve: the same to rounding
        assert np.isclose(r[k], o[k], rtol=1e-9), (name, k)
    # error_final is measured at a pose known only to `bound` along the nearly unobservable direction
    assert np.isclose(r["error_final"], o["error_final"], rtol=1e-9 if cond < 1e10 else 1e-3), name


@pytest.mark.parametrize("n", [41, 40])
def test_zero_mad_scale_oracle_equals_reference(oracle, n, ref):
    """Exactly zero reprojection errors for most observations: MAD scale 0, every Tukey weight from a division by 0."""
    c = zero_error_case(n, seed=n)
    r = ref.pose_optimize(*(args(c)[:2] + (c["cam"],) + args(c)[3:]))
    o = oracle.pose_optimize(*args(c))
    assert r["estimated_scale"] == 0.0 == o["estimated_scale"]
    assert np.array_equal(r["T"], o["T"]) and np.array_equal(r["has_point"], o["has_point"]) and r["num_obs"] == o["num_obs"]
    assert r["error_init"] == o["error_init"] and r["error_final"] == o["error_final"]
    assert np.array_equal(np.isfinite(r["cov"]), np.isfinite(o["cov"]))


def test_depth_seed_statuses_oracle_equals_reference(oracle, ref):
    """Seeds in every status of DepthFilter::updateSeeds in one call, and seeds whose sigma2 is negative, NaN or infinite.
    For a bad sigma2 the reference computes z_inv_max with std::max, which passes a NaN through, where the kernel's fmaxf
    returns 1e-8; z_inv_min is NaN (negative, NaN) or inf (inf) either way, so the epipolar segment has a NaN or zero-depth
    end, the scan never starts, and the seed ends in NO_MATCH with b + 1 in both."""
    c = synth.make_seed_status_case(91)
    r = ref.depth_filter_update([c["ref_pyr"][0]], [c["T_ref_w"]], c["cur_pyr"][0], c["T_cur_w"], c["n_levels"], c["cam"],
                                c["ref_index"], c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"],
                                c["batch_id"], c["batch_counter"], c["seeds"])
    o = oracle.depth_filter_update([c["ref_pyr"]], [c["T_ref_w"]], c["cur_pyr"], c["T_cur_w"], c["cam"], c["ref_index"],
                                   c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"],
                                   c["batch_counter"], c["seeds"])
    st = o["status"]
    for s in (1, 2, 3, 4, 5, 6):
        assert (st == s).sum() > 0, s
    assert not (st == 7).any()
    s2 = c["seeds"]["sigma2"]
    nan_min = c["bad_sigma2"] & ~(s2 > 0) & (st >= 4)  # negative or NaN sigma2 that reached the matcher: z_inv_min is NaN
    assert nan_min.sum() > 5 and np.all(st[nan_min] == 4)
    assert np.array_equal(r["status"], np.where(st == 6, 1, np.where((st == 1) | (st == 7), 2, 0)))
    keep = r["status"] == 0
    for k in ("a", "b", "mu", "z_range", "sigma2"):
        assert np.array_equal(r[k][keep].view(np.uint32), o[k][keep].view(np.uint32)), k


@pytest.mark.parametrize("kind", ["render", "noise", "checker", "low_contrast"])
def test_fast_numpy_statement_equals_oracle(oracle, kind):
    """The oracle's detector against the independent numpy statement (tests/fast_numpy.py: the segment test from the
    ring's definition, the library's literal bisection, dense 3x3 suppression, Shi-Tomasi in float64) for every FAST
    threshold b from 0 to 254 and both tie modes.  x, y and level must agree on every cell float64 decides."""
    from tests import fast_numpy as fn

    pyr = fn.images(1)[kind]
    n_corners = 0
    for b in (0, 1, 19, 20, 21, 60, 200, 254):
        for ties in (0, 1):
            r = fn.detect(pyr, 3, 8, 0.0, b=b, ties_suppress=bool(ties))
            o = oracle.fast_detect(pyr, 3, 8, 0.0, nonmax_ties_suppress=ties, fast_threshold=b)
            assert len(r["ambiguous"]) <= 2
            assert fn.agree(r, o, 64, 8) >= 46
            n_corners += len(o["x"])
            if kind == "low_contrast" and b == 0:
                assert (r["fast_score"] == 0).sum() >= 20                    # score-0 corners win their cells
    assert n_corners > 0


def test_fast_detect_thresholds_oracle_equals_reference(oracle, ref):
    """The compiled reference's FastDetector (b = 20, as it hard-codes) on a tiled 16x16 motif, whose cells hold equal
    Shi-Tomasi scores, and at detection thresholds around a winner's float32 score.  A threshold whose float32 rounding
    lies above it leaves the initial Corner(0, 0, threshold, 0) of every cell no corner beat above the threshold, and the
    reference emits it."""
    motif = np.random.default_rng(4).integers(0, 256, (16, 16), dtype=np.uint8)
    pyr = synth.build_pyramid(np.tile(motif, (6, 8)), 3)
    a, b = oracle.fast_detect(pyr, 3, 32, 0.0), ref.fast_detect(pyr[0], 3, 3, 32, 0.0)
    assert all(np.array_equal(a[k], b[k]) for k in ("x", "y", "level")) and len(a["x"]) == 12
    pyr = synth.make_two_view(5, width=320, height=240, n_levels=3)["ref_pyr"]
    s = float(np.median(oracle.fast_detect(pyr, 3, 30, 0.0)["score"]))
    for thr in (0.0, -0.0, s, np.nextafter(s, np.inf), np.nextafter(s, -np.inf), 1e30):
        a, b = oracle.fast_detect(pyr, 3, 30, thr), ref.fast_detect(pyr[0], 3, 3, 30, float(thr))
        assert all(np.array_equal(a[k], b[k]) for k in ("x", "y", "level")), thr
    assert ((b["x"] == 0) & (b["y"] == 0)).sum() == 11 * 8                    # 1e30: placeholders only


def test_many_observations_reprojection_oracle_equals_reference(oracle, ref):
    """Points with 32 to ~70 observations, exactly equal viewing angles (duplicated keyframe poses) and points seen
    only from behind: Point::getCloseViewObs and the cell policy of the compiled reference against the oracle."""
    from tests import reproject_cases as rc

    c = rc.many_obs_case()
    c = dict(c, options=dict(c["options"], max_fts=1000))
    r, o = ref.reproject_map(c), oracle.reproject_map(c)
    for k in ("n_matches", "n_trials", "n_new", "n_overlap"):
        assert r[k] == o[k], k
    for k in ("overlap_kf", "overlap_count", "new_point", "new_level", "new_type", "pt_type", "pt_n_failed", "pt_n_succeeded"):
        assert np.array_equal(r[k], o[k]), k
    assert np.max(np.abs(r["new_px"] - o["new_px"]), initial=0.0) <= 1e-9
    assert np.allclose(r["new_grad"], o["new_grad"], rtol=0, atol=1e-9)
    assert o["n_new"] > 30
