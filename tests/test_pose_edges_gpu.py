"""GPU: pose_opt_kernel and point_optimize_kernel at the corners the default cases never reach -- few observations,
singular and ill-conditioned normal matrices (both sides of the unpivoted LDL^T's pivot test), the shared-memory
capacity, noise-free frames (MAD scale 0), tied medians, few iterations and multi-wave batches -- against the oracle and,
where the oracle's pin does not cover the corner, against the compiled reference's recorded outputs."""
import numpy as np
import pytest

from rpg_svo_b200 import synth
from rpg_svo_b200.capi import SvoB200Error
from tests.pose_cases import (PIVOT_THRESH, args, backward_error, degenerate_cases, first_normal_matrix, first_normal_system,
                               first_step, min_pivot_ratio, pivot_sweep_cases, zero_error_case)
from tests.ref_golden import RefCalls

pytestmark = pytest.mark.gpu


def _finite_cov_equal(a, b, rtol=1e-6, atol=1e-12):
    """A singular A has no inverse: both sides then hold inf / NaN / huge entries.  They must agree on which entries are
    finite, and the finite ones must agree when the matrix is invertible at all."""
    fa, fb = np.isfinite(a), np.isfinite(b)
    assert np.array_equal(fa, fb), (a, b)
    return np.allclose(a[fa], b[fb], rtol=rtol, atol=atol)


def _same_as_oracle(g, o, pose_tol=1e-8, cov=True):
    assert np.array_equal(g["has_point"], o["has_point"])
    assert g["num_obs"] == o["num_obs"] and g["n_iter_done"] == o["n_iter_done"], (g["n_iter_done"], o["n_iter_done"])
    dt, dr = synth.pose_error(g["T"], o["T"])
    assert dt < pose_tol and dr < pose_tol, (dt, dr)
    for k in ("estimated_scale", "error_init", "error_final"):
        assert abs(g[k] - o[k]) <= 1e-9 * max(1.0, abs(o[k])), k
    if cov:
        assert _finite_cov_equal(g["cov"], o["cov"])


# ---- 1a: the corners where the oracle is pinned to the compiled reference -----------------------------------------------
@pytest.mark.parametrize("n,outliers,noise,n_iter", [(8, 0.0, 0.5, 10), (40, 0.3, 1.0, 10), (1000, 0.1, 2.0, 3), (250, 0.03, 1.0, 1)])
def test_pose_oracle_pinned_corners(ctx, oracle, n, outliers, noise, n_iter):
    """The four cases of test_oracle_pose_optimizer_edge_cases_equal_reference_source_compiled_here on the kernel: the
    oracle bit for bit on the mask, and the compiled reference's outputs recorded for that pin (replayed here)."""
    c = synth.make_pose_opt_case(90 + n, n=n, width=752, height=480, px_noise=noise, outlier_frac=outliers)
    g = ctx.pose_optimize(*args(c, n_iter))
    o = oracle.pose_optimize(*args(c, n_iter))
    _same_as_oracle(g, o)
    assert g["n_iter_done"] <= n_iter
    r = RefCalls("test_oracle_pins", f"test_oracle_pose_optimizer_edge_cases_equal_reference_source_compiled_here[{n}-{outliers}-{noise}-{n_iter}]")
    rr = r.pose_optimize(2.0, n_iter, c["cam"], c["T_init"], c["f"], c["pos"], c["level"], c["has_point"])
    r.finish()
    assert np.array_equal(g["has_point"], rr["has_point"]) and g["num_obs"] == rr["num_obs"]
    dt, dr = synth.pose_error(g["T"], rr["T"])
    assert dt < 1e-8 and dr < 1e-8, (dt, dr)
    for k in ("estimated_scale", "error_init", "error_final"):
        assert abs(g[k] - rr[k]) <= 1e-9 * max(1.0, abs(rr[k])), k
    assert np.allclose(g["cov"], rr["cov"], rtol=1e-6, atol=1e-12)


# ---- 1b: singular and ill-conditioned A ----------------------------------------------------------------------------------
def _pose_bound(c, g, o):
    """Distance between the kernel's and the oracle's pose after an ill-conditioned solve: both are backward-stable
    LDL^T solves of the same A (unpivoted vs pivoted), so their steps agree to ~cond(A) * eps * |dT|.  Along A's (near)
    null space this bound is as large as the step itself -- it says nothing there; the solve is checked by its backward
    error instead (test_pose_degenerate_frames_take_both_solver_paths)."""
    A = first_normal_matrix(c)
    cond = np.linalg.cond(A)
    dT = max(synth.pose_error(o["T"], c["T_init"]))
    return 1e-9 + 100 * cond * 2.2e-16 * max(dT, 1e-6)


def test_pose_degenerate_frames_take_both_solver_paths(ctx, oracle):
    """One Gauss-Newton iteration on frames whose A sweeps across the pivot test: the kernel's branch report must be the
    one numpy predicts from A (the fast path where every pivot is clear of 1e-13 * max diagonal, the pivoted LDL^T where
    one is not), both paths must occur, and the step must solve A dT = b backward-stably: |A dT - b| / (|A| |dT| + |b|)
    <= 1e-12, with A and b formed in numpy and dT recovered from the returned pose.  That holds for any correct solve however
    ill-conditioned A is (measured: <= 1e-14 on these frames) and fails at O(1) for a wrong one."""
    counts = {"fast": 0, "pivoted": 0}
    for name, c in pivot_sweep_cases():
        g = ctx.pose_optimize(*args(c, 1))
        o = oracle.pose_optimize(*args(c, 1))
        A = first_normal_matrix(c)
        ratio = min_pivot_ratio(A)
        if c["has_point"].sum() >= 3 and (ratio > 10 * PIVOT_THRESH or ratio < 0.1 * PIVOT_THRESH):
            want = int(ratio <= PIVOT_THRESH)
            assert g["n_pivoted_solves"] == want and g["cov_pivoted"] == want, (name, ratio, g["n_pivoted_solves"])
        elif c["has_point"].sum() < 3:  # rank <= 4: some pivot is rounding noise around 0
            assert g["n_pivoted_solves"] == 1 and g["cov_pivoted"] == 1, name
        counts["pivoted" if g["n_pivoted_solves"] else "fast"] += 1
        assert g["n_iter_done"] == o["n_iter_done"] == 1, name
        assert np.array_equal(g["has_point"], o["has_point"]) and g["num_obs"] == o["num_obs"], name
        dt, dr = synth.pose_error(g["T"], o["T"])
        bound = _pose_bound(c, g, o)
        assert dt <= bound and dr <= bound, (name, dt, dr, bound)
        A, b = first_normal_system(c)
        if name not in ("window0.3", "window0.2"):
            assert backward_error(A, b, first_step(c, g["T"])) <= 1e-12, name
            assert backward_error(A, b, first_step(c, o["T"])) <= 1e-12, name
        # at 0.3 / 0.2 px, b sums errors of points 0.2 px apart carrying 0.003 px of noise: formed in double (numpy's
        # order or the kernel's) it is only good to ~1e-5 relative, so only the path choice is checked there
    print("pose optimizer solve paths:", counts)
    assert counts["fast"] > 0 and counts["pivoted"] > 0


@pytest.mark.parametrize("idx", range(6))
def test_pose_degenerate_frames_match_oracle_and_reference(ctx, oracle, idx):
    """Ten iterations on each degenerate frame against the oracle and the compiled reference's outputs (recorded by
    tests/test_edge_pins.py): mask, scale, error_init and error_final (the observable outcome), T within the
    condition-number bound, the covariance where A is invertible in double.  n_iter_done is compared where A has full
    numerical rank: with 1-2 observations or points on a line, the step along the null space is rounding noise and so is
    the iteration at which chi2 stops falling (see test_pose_optimize_ties_and_tiny_sets)."""
    name, c = degenerate_cases()[idx]
    g = ctx.pose_optimize(*args(c))
    o = oracle.pose_optimize(*args(c))
    bound = max(1e-8, _pose_bound(c, g, o))
    A = first_normal_matrix(c)
    cond = np.linalg.cond(A)
    if min_pivot_ratio(A) > PIVOT_THRESH:
        assert g["n_iter_done"] == o["n_iter_done"], (name, g["n_iter_done"], o["n_iter_done"])
    # error_final is measured at the final pose, which is known only to ~cond * eps along the weak directions; where the
    # observations are fitted exactly (1-2 observations) it is rounding noise, ~1e-13 px: hence the 1e-9 px floor
    tol_final = 1e-9 if cond < 1e10 else 1e-3
    for want in (o,):
        assert abs(g["estimated_scale"] - want["estimated_scale"]) <= 1e-9 * abs(want["estimated_scale"]), name
        assert abs(g["error_init"] - want["error_init"]) <= 1e-9 * abs(want["error_init"]), name
        assert abs(g["error_final"] - want["error_final"]) <= tol_final * abs(want["error_final"]) + 1e-9, name
    assert np.array_equal(g["has_point"], o["has_point"]) and g["num_obs"] == o["num_obs"], name
    dt, dr = synth.pose_error(g["T"], o["T"])
    assert dt <= bound and dr <= bound, (name, dt, dr, bound)
    r = RefCalls("test_edge_pins", f"test_pose_degenerate_oracle_equals_reference[{idx}]")
    rr = r.pose_optimize(*(args(c)[:2] + (c["cam"],) + args(c)[3:]))
    r.finish()
    assert np.array_equal(g["has_point"], rr["has_point"]) and g["num_obs"] == rr["num_obs"], name
    assert abs(g["estimated_scale"] - rr["estimated_scale"]) <= 1e-9 * abs(rr["estimated_scale"]), name
    assert abs(g["error_init"] - rr["error_init"]) <= 1e-9 * abs(rr["error_init"]), name
    assert abs(g["error_final"] - rr["error_final"]) <= tol_final * abs(rr["error_final"]) + 1e-9, name
    dt, dr = synth.pose_error(g["T"], rr["T"])
    assert dt <= bound and dr <= bound, (name, dt, dr, bound)
    assert np.array_equal(np.isfinite(g["cov"]), np.isfinite(rr["cov"])), name
    # the covariance is A's inverse: its relative error is ~cond(A) * eps in any implementation
    fin = np.isfinite(rr["cov"])  # at cond ~4e12 the last A can be singular in both, its inverse NaN in both
    if cond < 1e13:
        assert np.allclose(g["cov"][fin], rr["cov"][fin], rtol=max(1e-6, 1e3 * cond * 2.2e-16), atol=1e-12), (name, cond)


# ---- 1c: shared-memory capacity ------------------------------------------------------------------------------------------
def _probe(ctx, c, n):
    """True if the host accepts n observations in one frame (the shared-memory check returns ELIMIT before any launch
    when it does not; with has_point all zero an accepted frame launches a kernel that returns at once)."""
    d = dict(c, f=c["f"][:n], pos=c["pos"][:n], level=c["level"][:n], has_point=np.zeros(n, np.uint8))
    try:
        ctx.pose_optimize(*args(d))
        return True
    except SvoB200Error as e:
        assert "error -4" in str(e), e  # SVO_B200_ELIMIT
        return False


def test_pose_capacity_edge_and_counts_around_the_thread_strides(ctx, oracle):
    c = synth.make_pose_opt_case(123, 6000, 1920, 1080)
    lo, hi = 1000, 6000
    assert _probe(ctx, c, lo) and not _probe(ctx, c, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _probe(ctx, c, mid) else (lo, mid)
    n_max = lo
    print("largest frame the pose optimizer accepts:", n_max, "observations")
    assert n_max >= 3000
    assert not _probe(ctx, c, n_max + 1)
    rng = np.random.default_rng(5)
    for n in (1023, 1024, 1025, 2047, 2048, 2049, n_max):
        hp = c["has_point"][:n].copy()
        hp[rng.uniform(size=n) < 0.1] = 0  # holes
        d = dict(c, f=c["f"][:n], pos=c["pos"][:n], level=c["level"][:n], has_point=hp)
        g, o = ctx.pose_optimize(*args(d)), oracle.pose_optimize(*args(d))
        _same_as_oracle(g, o)
        assert g["num_obs"] > 0.6 * n


# ---- 1d: zero noise, odd / even counts, tied medians ---------------------------------------------------------------------
@pytest.mark.parametrize("n", [41, 40])
def test_pose_zero_mad_scale(ctx, oracle, n):
    """Reprojection errors exactly 0 for all but three observations (tests/pose_cases.zero_error_case): the MAD scale is
    exactly 0, every Tukey weight is tukey(e / 0) -- 0/0 = NaN for the exact observations, e/0 = inf for the others, both
    weight 0 -- so A = 0, the solve takes the pivoted LDL^T's all-zero early exit (dT = 0, converged after one
    iteration) and the covariance inverts a zero matrix.  Every output against the oracle and the compiled reference."""
    c = zero_error_case(n, seed=n)
    for n_iter in (1, 10):
        g, o = ctx.pose_optimize(*args(c, n_iter)), oracle.pose_optimize(*args(c, n_iter))
        assert g["estimated_scale"] == 0.0 == o["estimated_scale"]
        assert g["error_init"] == o["error_init"] and g["error_final"] == o["error_final"]
        assert g["n_iter_done"] == o["n_iter_done"] == 1 and g["n_pivoted_solves"] == 1 and g["cov_pivoted"] == 1
        assert np.array_equal(g["has_point"], o["has_point"]) and g["num_obs"] == o["num_obs"]
        assert np.array_equal(g["T"], c["T_init"]) and np.array_equal(o["T"], c["T_init"])  # dT = 0 exactly
        assert np.array_equal(np.isfinite(g["cov"]), np.isfinite(o["cov"])) and not np.isfinite(g["cov"]).any()
    r = RefCalls("test_edge_pins", f"test_zero_mad_scale_oracle_equals_reference[{n}]")
    rr = r.pose_optimize(*(args(c)[:2] + (c["cam"],) + args(c)[3:]))
    r.finish()
    assert rr["estimated_scale"] == 0.0 and np.array_equal(g["T"], rr["T"]) and np.array_equal(g["has_point"], rr["has_point"])
    assert g["error_init"] == rr["error_init"] and g["error_final"] == rr["error_final"] and g["num_obs"] == rr["num_obs"]


@pytest.mark.parametrize("n", [41, 40])
def test_pose_more_than_half_the_errors_tied(ctx, oracle, n):
    """Most observations are copies of one: the median select of the scale and of error_init / error_final meets a
    run of equal keys longer than half the array, at odd and even counts."""
    c = synth.make_pose_opt_case(400 + n, n, 752, 480, px_noise=1.0, outlier_frac=0.0)
    c["has_point"][:] = 1
    k = n // 2 + 3
    for key in ("f", "pos", "level"):
        c[key][1:k] = c[key][0]
    for n_iter in (1, 3, 10):
        g, o = ctx.pose_optimize(*args(c, n_iter)), oracle.pose_optimize(*args(c, n_iter))
        _same_as_oracle(g, o)


# ---- 1e: a batch of several waves mixing every case ----------------------------------------------------------------------
def test_pose_batch_of_several_waves_equals_single_calls(ctx, oracle):
    probe = synth.make_pose_opt_case(123, 6000, 1920, 1080)
    lo, hi = 3000, 6000
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _probe(ctx, probe, mid) else (lo, mid)
    frames = [synth.make_pose_opt_case(500, lo, 1920, 1080)]
    frames += [c for _, c in degenerate_cases()]
    for k in range(290):
        n = [0, 1, 2, 7, 40, 300, 1025][k % 7]
        c = synth.make_pose_opt_case(600 + k, max(n, 1), 752, 480, px_noise=1.0, outlier_frac=0.1)
        if n == 0:
            c["has_point"][:] = 0
        frames.append(c)
    assert len(frames) > 2 * 132
    off = np.concatenate([[0], np.cumsum([len(c["level"]) for c in frames])]).astype(np.int32)
    cat = lambda k: np.concatenate([c[k] for c in frames])
    res = ctx.pose_optimize_batch(2.0, 10, [c["cam"].fx for c in frames], np.stack([c["T_init"] for c in frames]), off,
                                  cat("f"), cat("pos"), cat("level"), cat("has_point"))
    for i, (c, r) in enumerate(zip(frames, res)):
        g = ctx.pose_optimize(*args(c))
        assert np.array_equal(r["T"], g["T"]) and np.array_equal(r["has_point"], g["has_point"]), i
        for k in ("num_obs", "n_iter_done", "n_pivoted_solves", "cov_pivoted", "estimated_scale", "error_init", "error_final"):
            assert r[k] == g[k] or (np.isnan(r[k]) and np.isnan(g[k])), (i, k)
        assert np.array_equal(r["cov"], g["cov"], equal_nan=True), i


# ---- 3: the point optimizer ----------------------------------------------------------------------------------------------
def test_point_optimize_single_observation(ctx, oracle):
    """One observation: A = J^T J has rank 2.
    * Points on the optical axis of an unrotated camera: A = diag(1/z^2, 1/z^2, 0) exactly, ldlt3_solve's third pivot is
      exactly 0 and its 1/DBL_MAX test zeroes that component -- a deterministic step, equal to the oracle's to rounding.
    * General points: the third pivot is rounding noise (~1e-17 of the others) that every implementation divides by, so
      the step along the viewing ray is arbitrary (kernel and oracle end centimetres apart on it).  Across the ray the
      step is the range-space solve: the point's projection into the observing frame must agree with the oracle's.  Moving
      along the linearised ray from the stepped point changes the projection only at second order, by <= |d| |s| / z^2
      for a difference d along the ray, a step s and a depth z; and the step must reduce the start's reprojection error
      (the oracle's leaves at most 0.47 of it on these points)."""
    rng = np.random.default_rng(23)
    P, A = 64, 8
    poses = [synth.se3_exp(np.concatenate([rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.05, 0.05, 3)])) for _ in range(4)]
    poses.append(np.hstack([np.eye(3), [[0.0], [0.0], [0.25]]]))           # unrotated camera: the axis points
    pos0 = np.stack([rng.uniform(-1, 1, P), rng.uniform(-1, 1, P), rng.uniform(3, 6, P)], 1)
    frs = rng.integers(0, 4, P).astype(np.int32)
    frs[:A] = 4
    pos0[:A, :2] = 0.0                                                      # exactly on that camera's optical axis
    fs = []
    for p in range(P):
        T = poses[frs[p]]
        pc = T[:, :3] @ (pos0[p] + rng.normal(0, 0.05, 3)) + T[:, 3]
        fs.append(pc / np.linalg.norm(pc))
    fs = np.array(fs)

    def proj(T, x):
        q = T[:, :3] @ x + T[:, 3]
        return q[:2] / q[2], q[2]

    g = ctx.point_optimize_batch(1, pos0, np.arange(P + 1), frs, fs, poses)
    for p in range(P):
        o = oracle.point_optimize(1, pos0[p], [poses[frs[p]]], fs[p:p + 1])
        T = poses[frs[p]]
        if p < A:
            assert np.allclose(g[p], o, rtol=0, atol=1e-12), (p, g[p] - o)
            assert g[p][2] == pos0[p][2] and o[2] == pos0[p][2]             # the zero-pivot component is not moved
            continue
        (pg, z), (po, _), (p0, _) = proj(T, g[p]), proj(T, o), proj(T, pos0[p])
        obs = fs[p][:2] / fs[p][2]
        d, step = np.linalg.norm(g[p] - o), np.linalg.norm(o - pos0[p])
        assert np.linalg.norm(pg - po) <= 2 * d * step / z ** 2 + 1e-12, (p, pg - po, d, step)
        assert np.linalg.norm(pg - obs) < np.linalg.norm(p0 - obs), p
    for n_iter in (3, 5):  # later iterations start from points that differ along the ray: finite where the oracle is
        g = ctx.point_optimize_batch(n_iter, pos0, np.arange(P + 1), frs, fs, poses)
        for p in range(P):
            o = oracle.point_optimize(n_iter, pos0[p], [poses[frs[p]]], fs[p:p + 1])
            assert np.array_equal(np.isfinite(g[p]), np.isfinite(o)), p


def test_point_optimize_few_iterations_match_oracle_and_reference(ctx, oracle):
    """The points of test_oracle_point_optimize_equals_reference_source_compiled_here (2-6 observations, bearing noise
    1e-3) at 1, 3 and 5 iterations.  Before convergence the kernel's matrix path and the oracle's quaternion path
    differ by the rotation matrix's rounding (~1e-16 relative per entry), amplified by the 3x3 system's condition
    number along the ray (<= ~1e4 for these baselines): 1e-10 m on positions of 3-6 m; the oracle is pinned to the
    reference at 1e-13 for 1 and 3 iterations, so the reference's recorded outputs are held to the same bound."""
    rng = np.random.default_rng(5)
    r = RefCalls("test_oracle_pins", "test_oracle_point_optimize_equals_reference_source_compiled_here")
    for _ in range(20):
        pos = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(3, 6)])
        Ts, fs = [], []
        for _ in range(int(rng.integers(2, 7))):
            T = synth.se3_exp(np.concatenate([rng.uniform(-0.5, 0.5, 3), rng.uniform(-0.05, 0.05, 3)]))
            pc = T[:, :3] @ pos + T[:, 3]
            f = pc / np.linalg.norm(pc) + rng.normal(0, 1e-3, 3)
            Ts.append(T.reshape(12)); fs.append(f / np.linalg.norm(f))
        start = pos + rng.normal(0, 0.05, 3)
        k = len(fs)
        for n_iter in (1, 3, 5):
            a = r.point_optimize(n_iter, start, np.array(Ts), np.array(fs))
            o = oracle.point_optimize(n_iter, start, np.array(Ts), np.array(fs))
            g = ctx.point_optimize_batch(n_iter, start[None], [0, k], np.arange(k), np.array(fs), [T.reshape(3, 4) for T in Ts])[0]
            tol = 1e-10 if n_iter < 5 else 1e-8  # at convergence the last roll-back compares rounding noise
            assert np.allclose(g, o, rtol=0, atol=tol), (n_iter, g - o)
            assert np.allclose(g, a, rtol=0, atol=tol), (n_iter, g - a)
    r.finish()
