"""GPU: point_optimize_kernel (Point::optimize) against the high-precision statement of tests/point_hp.py -- at 0 to
20000 observations per point, 0 to 10 iterations, each of its four ways to end, the EPS stop at its edge, degenerate
geometry, non-finite inputs and batch shapes -- and against the oracle and the compiled reference's recorded outputs on
the degenerate and non-finite points; and the refusal of malformed observation offset tables.

A point whose every decision is decisive (point_hp: margins beyond 1e-9 relative and beyond the kernel's own rounding)
must take the exact run's branches and end within that run's bound; a point with a near-tie may end on either side of
it, within the bound of the branch it took (point_hp.branches recomputes each)."""
import ctypes as C

import numpy as np
import pytest

from rpg_svo_b200.capi import _p, c64
from tests import point_cases as pc
from tests import point_hp as hp
from tests.ref_golden import RefCalls

pytestmark = pytest.mark.gpu

WORST = {"ratio": 0.0, "where": None}  # largest error / bound over this module's comparisons


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _single(ctx, n_iter, s, Ts, fs):
    return ctx.point_optimize_batch(n_iter, *pc.batch([(s, Ts, fs)]))[0]


def _check(g, n_iter, s, Ts, fs, label, counts=None):
    """g (the kernel's result) against the runs the exact reference allows; returns the run it matched."""
    runs = hp.branches(n_iter, s, Ts, fs)
    run, ratio = hp.match_any(g, runs)
    assert run is not None, (label, g, [hp.as_float(r) for r in runs], [r["bound"] for r in runs], ratio)
    if hp.decisive(runs[0]):
        assert run is runs[0], label
    if hp.defined(run) and ratio > WORST["ratio"]:
        WORST.update(ratio=ratio, where=label)
    if counts is not None:
        for rec in runs[0]["trace"]:
            if rec["tie"] is None and rec.get("decision") in counts:
                counts[rec["decision"]] += 1
    return run


def _report(what):
    print(f"{what}: largest |kernel - exact| / bound so far {WORST['ratio']:.3g} ({WORST['where']})")


# ---- observation and iteration counts --------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 2, 3, 7, 64, 1000, 20000])
def test_point_observation_counts(ctx, oracle, n):
    """0 observations: A = 0, the solve's all-zero pivot exit gives dp = 0 and the point comes back bit for bit (a -0.0
    coordinate as +0.0: -0.0 + 0.0, in the oracle too).  1 observation on the optical axis of its camera: the exactly-zero
    pivot.  2 to 20000: bearings with 1e-3 rad noise, 5 iterations (structureOptimNumIter); the bound grows with n."""
    rng = np.random.default_rng(100 + n)
    if n == 0:
        starts = np.array([[0.25, -1.5, 4.0], [-0.0, 2.0, -3.0]])
        g = ctx.point_optimize_batch(5, starts, [0, 0, 0], np.zeros(0, np.int32), np.zeros((0, 3)), np.zeros((1, 3, 4)))
        assert np.array_equal(_bits(g[0]), _bits(starts[0]))
        assert np.array_equal(_bits(g[1]), _bits(oracle.point_optimize(5, starts[1], np.zeros((0, 12)), np.zeros((0, 3)))))
        assert np.array_equal(_bits(g[1]), _bits([0.0, 2.0, -3.0]))
        return
    if n == 1:
        Ts = np.array([pc.pose_at([0.0, 0.0, 0.0])])
        s, fs, n_iter = np.array([0.0, 0.0, 3.0]), pc.bearings(Ts, np.array([0.05, 0.02, 3.5])), 1
    else:
        s, Ts, fs, _ = pc.track(rng, n)
        n_iter = 5
    g = _single(ctx, n_iter, s, Ts, fs)
    r = _check(g, n_iter, s, Ts, fs, f"n={n}")
    assert hp.defined(r), (n, r["bound"])
    if n == 1:
        assert r["trace"][0]["pivots"][2] == 0 and g[2] == s[2]  # the zero-pivot component is not moved
    print(f"n={n}: |kernel - exact| = {hp.error(g, r):.3g} m, bound {r['bound']:.3g} m, "
          f"decisions {[x['decision'] for x in r['trace']]}{' (a near-tie branch)' if r['force'] else ''}")
    _report(f"n={n}")


@pytest.mark.parametrize("n_iter", [0, 1, 2, 5, 10])
def test_point_iteration_counts(ctx, n_iter):
    """40 points (2-6 observations) in one launch at n_iter = 0 (every position bit for bit), 1, 2, 5 and 10."""
    rng = np.random.default_rng(7)
    pts = [pc.track(rng, int(rng.integers(2, 7)))[:3] for _ in range(40)]
    g = ctx.point_optimize_batch(n_iter, *pc.batch(pts))
    for p, (s, Ts, fs) in enumerate(pts):
        if n_iter == 0:
            assert np.array_equal(_bits(g[p]), _bits(s)), p
        _check(g[p], n_iter, s, Ts, fs, f"n_iter={n_iter} point {p}")
    _report(f"n_iter={n_iter}")


# ---- every way to end, and the EPS stop at its edge ------------------------------------------------------------------
def test_point_every_branch_occurs(ctx):
    """The four ways Point::optimize ends, counted where the exact trace decides them decisively: the EPS stop (tracks
    converging within 10 iterations; decisive on noise-free tracks, with noisy bearings the last chi2 comparisons are
    near-ties), the roll-back on a chi2 increase at it > 0 (the 0.26 mm baseline's second step overshoots), the roll-back
    on a NaN step at it = 0 (a start at z = 0, a bearing with f_z = 0) and running out of iterations (2 iterations on the
    same tracks).  Each must occur, and the kernel must follow every decisive one."""
    rng = np.random.default_rng(8)
    cases = {c[0]: c for c in pc.edge_cases()}
    pts = []
    for _ in range(30):
        s, Ts, fs, _ = pc.track(rng, int(rng.integers(2, 7)), noise=float(rng.choice([0.0, 1e-3])))
        pts += [(10, s, Ts, fs), (2, s, Ts, fs)]
    pts += [cases[k][1:] for k in ("baseline_0.00026", "start_z0", "bearing_fz0")]
    counts = {"stop": 0, "rollback": 0, "nan": 0, "out_of_iterations": 0}
    for j, (n_iter, s, Ts, fs) in enumerate(pts):
        _check(_single(ctx, n_iter, s, Ts, fs), n_iter, s, Ts, fs, f"branch case {j}", counts)
    print("decisive endings in the exact traces:", counts)
    assert all(v > 0 for v in counts.values()), counts
    _report("branches")


def test_point_eps_stop_at_its_edge(ctx):
    """Noise-free observations: Gauss-Newton converges quadratically, so over 400 starts 1e-4..1e-1 m off some step lands
    within a factor 10 of EPS = 1e-10 on either side.  Where that decision is decisive, the kernel must take it -- stop
    just below, one more iteration just above."""
    rng = np.random.default_rng(9)
    side = {"below": 0, "above": 0}
    picked = []
    for _ in range(400):
        s, Ts, fs, _ = pc.track(rng, int(rng.integers(2, 7)), noise=0.0, start_sigma=10 ** rng.uniform(-4, -1))
        r = hp.optimize(10, s, Ts, fs)
        edge = [d for d in r["trace"] if "eps_margin" in d and d["tie"] is None and -0.9 <= d["eps_margin"] <= 9.0]
        if edge:
            side["below" if edge[0]["eps_margin"] < 0 else "above"] += 1
            picked.append((s, Ts, fs))
    print("decisive EPS decisions within a factor 10 of EPS:", side)
    assert side["below"] > 0 and side["above"] > 0
    g = ctx.point_optimize_batch(10, *pc.batch(picked))
    for p, (s, Ts, fs) in enumerate(picked):
        _check(g[p], 10, s, Ts, fs, f"eps edge point {p}")
    _report("EPS edge")


# ---- degenerate and non-finite points --------------------------------------------------------------------------------
def test_point_degenerate_and_nonfinite_match_oracle_and_reference(ctx, oracle):
    """The cases of tests/point_cases.py against the exact runs, the oracle and the compiled reference's recorded outputs
    (tests/test_point_edge_pins.py): the same finite coordinates everywhere; bit for bit with the start (and so with both)
    where the exact run decisively returns it -- a NaN step at iteration 0 from a NaN or inf start, bearing or rotation,
    a start at z = 0, a bearing with f_z = 0; within the bound elsewhere.  Where A's smallest pivot is rounding noise (one
    camera centre with rotated frames, the 8 um baseline) the step along the ray is that noise divided out, in the kernel,
    the oracle and the reference alike: no bound is defined there and only finiteness is compared."""
    r = RefCalls("test_point_edge_pins", "test_point_edge_cases_oracle_equals_reference")
    refs = pc.ref_outputs(r)
    r.finish()
    for (name, n_iter, s, Ts, fs), rr in zip(pc.edge_cases(), refs):
        g = _single(ctx, n_iter, s, Ts, fs)
        o = oracle.point_optimize(n_iter, s, Ts, fs)
        assert np.array_equal(np.isfinite(g), np.isfinite(o)) and np.array_equal(np.isfinite(g), np.isfinite(rr)), (name, g, o, rr)
        run = _check(g, n_iter, s, Ts, fs, name)
        if run["untouched"] and hp.decisive(run):
            assert np.array_equal(_bits(g), _bits(s)) and np.array_equal(_bits(o), _bits(s)) and np.array_equal(_bits(rr), _bits(s)), name
    _report("degenerate / non-finite")


# ---- batch shapes ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [1, 127, 128, 129, 131072])
def test_point_batch_equals_single_calls(ctx, P):
    """Points with 0-3 observations around the 128-thread block edges, and at P = 131072 three 20000-observation
    stragglers in the same launch: every point bit for bit equal to a one-point call of it."""
    rng = np.random.default_rng(P)
    pts = []
    for p in range(P):
        k = int(rng.integers(0, 4))
        X = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(3, 6)])
        Ts = np.array([pc.pose_at(rng.uniform(-0.5, 0.5, 3), rng.uniform(-0.05, 0.05, 3)) for _ in range(k)]).reshape(-1, 12)
        pts.append((X + rng.normal(0, 0.05, 3), Ts, pc.bearings(Ts, X, rng, 1e-3) if k else np.zeros((0, 3))))
    if P == 131072:
        for p in (5, 70000, P - 1):
            pts[p] = pc.track(rng, 20000)[:3]
    g = ctx.point_optimize_batch(5, *pc.batch(pts))
    for p, (s, Ts, fs) in enumerate(pts):
        assert np.array_equal(_bits(g[p]), _bits(_single(ctx, 5, s, Ts, fs))), p


def test_point_batch_offset_prefix_and_last_frame(ctx):
    """obs_offset[0] > 0: the observations before it are never read -- NaN bearings and frame indices far out of range
    there are accepted -- and the result equals the rebased call bit for bit.  Observations use every frame up to the last
    one, n_frames - 1."""
    rng = np.random.default_rng(13)
    pts = [pc.track(rng, int(rng.integers(1, 5)))[:3] for _ in range(300)]
    starts, off, frs, fs, Ts = pc.batch(pts)
    n_frames = len(Ts)
    frs = rng.permutation(n_frames).astype(np.int32)[frs]   # every frame used once, the last one included
    Ts_perm = np.empty_like(Ts)
    Ts_perm[frs] = Ts
    assert frs.max() == n_frames - 1
    want = ctx.point_optimize_batch(5, starts, off, frs, fs, Ts_perm)
    pre = 17
    frs_p = np.concatenate([np.array([-5, 10 ** 6] * 8 + [n_frames], np.int32), frs])
    fs_p = np.concatenate([np.full((pre, 3), np.nan), fs])
    got = ctx.point_optimize_batch(5, starts, off + pre, frs_p, fs_p, Ts_perm)
    assert np.array_equal(_bits(got), _bits(want))
    for p in range(0, 300, 37):
        assert np.array_equal(_bits(want[p]), _bits(_single(ctx, 5, *pts[p]))), p


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_point_and_pose_batch_refuse_malformed_offsets(ctx):
    """Offsets must satisfy 0 <= off[0] <= off[1] <= ... <= off[P]: a decreasing interior entry (point 0 would walk 100
    observations of a 6-entry table), a last entry below the first (a negative observation count) and a negative first
    entry are refused with SVO_B200_EINVAL before anything is launched or written; the pose batch refuses a negative first
    entry the same way."""
    lib = ctx.lib
    fr = np.zeros(200, np.int32)
    f = np.tile([0.0, 0.0, 1.0], (200, 1))
    T = c64(np.tile(pc.pose_at([0.0, 0.0, 0.0]), (2, 1)))
    for off in ([0, 100, 5], [5, 6, 3], [-1, 2, 3]):
        pos = c64(np.arange(6.0).reshape(2, 3))
        snap = pos.copy()
        o = np.array(off, np.int32)
        n0 = ctx.launch_count()
        rc = lib.svo_b200_point_optimize_batch(ctx.h, 2, 5, _p(o), _p(fr), _p(c64(f)), _p(T), 2, _p(pos))
        assert rc == -1, off
        assert ctx.launch_count() == n0 and np.array_equal(_bits(pos), _bits(snap)), off
    # pose batch, negative first entry
    Tp = c64(np.tile(pc.pose_at([0.0, 0.0, 0.0]), (1, 1)))
    Tsnap = Tp.copy()
    hpv = np.ones(8, np.uint8)
    hsnap = hpv.copy()
    fx = c64([300.0])
    o = np.array([-1, 3], np.int32)
    out = (C.c_byte * 4096)()
    n0 = ctx.launch_count()
    rc = lib.svo_b200_pose_optimize_batch(ctx.h, 1, C.c_double(2.0), 10, _p(fx), _p(Tp), _p(o), _p(c64(f[:8])),
                                          _p(c64(np.ones((8, 3)))), _p(np.zeros(8, np.int32)), _p(hpv), out)
    assert rc == -1
    assert ctx.launch_count() == n0 and np.array_equal(_bits(Tp), _bits(Tsnap)) and np.array_equal(hpv, hsnap)
    _report("module")
