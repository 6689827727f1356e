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
