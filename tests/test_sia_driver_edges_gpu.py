"""GPU: the plain alignment kernel's Gauss-Newton driver (gn_tail, the per-level loop, the outputs) on the corner cases of
tests/sia_driver_cases.py, in every launch geometry: against the oracle, against the float64 statement of each step, at the
exact edge of the convergence test, replaying the compiled reference's recorded outputs, and in a mixed batch of the
throughput geometry that holds every driver path at once."""
import collections

import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import sia_cases as sc
from tests import sia_driver_cases as dc
from tests.ref_golden import RefCalls

pytestmark = pytest.mark.gpu

# (ctas_per_pair, features_per_thread, upfront mode): as test_sia_geometry_gpu.GEOMETRIES
GEOMETRIES = {"auto": (-1, 0, -1), "cta-1fpt": (1, 1, -1), "cta-2fpt": (1, 2, -1), "cluster-4": (4, 0, -1),
              "cluster-4-per-level": (4, 0, 0), "cluster-8": (8, 0, -1)}
# Observed on an H100 (NVIDIA H100 80GB HBM3), maxima over the cases in parentheses:
X_ATOL = 1e-5        # trace x vs the oracle's (7.9e-7; relative to |x|_inf up to 8.5e-4 on the small last steps of a level)
POSE_STEP_TOL = 1e-13  # T_k vs T_(k-1) exp(-x_k) in float64
ORTH_TOL = 2e-15     # |R^T R - I| of every pose of the trace (the oracle's reaches 1.1e-15 after steps of theta^2 up to 5)
SOLVE_TOL = 1e-13    # |x - H^-1 Jres|_inf / |x|_inf per unit of cond(H)


def _configure(ctx, cfg):
    ctx.sia_config(cfg[0], cfg[1])
    ctx.sia_upfront(cfg[2])


@pytest.fixture(autouse=True)
def _reset_config(ctx):
    yield
    ctx.sia_config(-1, 0)
    ctx.sia_upfront(-1)


_frames = {}


@pytest.fixture(scope="module")
def frames(ctx):
    """Device frames per pyramid (keyed by the id of its level-0 array), shared by the cases."""
    yield _frames
    for r, c in _frames.values():
        r.destroy()
        if c is not r:
            c.destroy()
    _frames.clear()


def _frames_of(ctx, frames, p):
    key = (id(p["ref_pyr"][0]), id(p["cur_pyr"][0]))
    if key not in frames:
        r = ctx.frame(p["ref_pyr"])
        frames[key] = (r, r if p["cur_pyr"] is p["ref_pyr"] else ctx.frame(p["cur_pyr"]))
    return frames[key]


def gpu_run(ctx, frames, k, eps=None):
    p = k["p"]
    ref_f, cur_f = _frames_of(ctx, frames, p)
    return ctx.sparse_img_align(ref_f, cur_f, p["cam"], k["T0"], p["px"], p["f"], p["pos"], p["has_point"], p["ref_pos"],
                                k["max_level"], k["min_level"], k["n_iter"], k["eps"] if eps is None else eps,
                                want_trace=True)


_oracle = {}


def oracle_run(k):
    if k["name"] not in _oracle:
        _oracle[k["name"]] = dc.oracle_run(k)
    return _oracle[k["name"]]


def same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def assert_driver_parity(g, o, k):
    """Mask and n_tracked exact; below RANK_OK features (and on dc.NEAR_SINGULAR) the first pass's n_meas only.  Otherwise the trace's (level, iter,
    accepted, n_meas) exact, chi2 within 1e-4 relative (NaN where the oracle's is), x within X_ATOL (NaN where the oracle's
    is), the final pose within sc.POSE_TOL (NaN where the oracle's is)."""
    n = len(k["p"]["px"])
    assert np.array_equal(g["visible"], o["visible"]), "visibility mask"
    assert g["n_tracked"] == o["n_tracked"], (g["n_tracked"], o["n_tracked"])
    if n < dc.RANK_OK or k["name"] in dc.NEAR_SINGULAR:
        assert len(g["trace"]) > 0 and g["trace"][0]["n_meas"] == o["trace"][0]["n_meas"]
        return
    assert dc.margin(o, k["eps"]) > dc.MARGIN, dc.margin(o, k["eps"])
    assert len(g["trace"]) == len(o["trace"]), (len(g["trace"]), len(o["trace"]))
    for a, b in zip(g["trace"], o["trace"]):
        assert (a["level"], a["iter"], a["accepted"], a["n_meas"]) == (b["level"], b["iter"], b["accepted"], b["n_meas"])
        assert (np.isnan(a["chi2"]) and np.isnan(b["chi2"])) or abs(a["chi2"] - b["chi2"]) <= 1e-4 * max(1.0, abs(b["chi2"]))
        assert np.array_equal(np.isnan(a["x"]), np.isnan(b["x"]))
        m = ~np.isnan(b["x"])
        if m.any():
            assert np.abs(a["x"][m] - b["x"][m]).max() <= X_ATOL, (a["x"], b["x"])
    assert np.array_equal(np.isnan(g["T"]), np.isnan(o["T"]))
    if not np.isnan(o["T"]).any():
        dt, dr = synth.pose_error(g["T"], o["T"])
        assert dt <= sc.POSE_TOL and dr <= sc.POSE_TOL, (dt, dr)


def assert_driver_statement(ctx, frames, g, k, solve=True):
    """The kernel's own trace against the float64 statement (tests/sia_driver_cases.py): each accepted step is T exp(-x) to
    POSE_STEP_TOL with an orthonormal rotation, each rejected one gives back the pose its level's last accepted step started
    from bit for bit, the flags follow the termination rule, the final pose is the trace's last bit for bit, the stats
    count the trace, and x solves the residual pass's H x = Jres to SOLVE_TOL cond(H)."""
    tr = g["trace"]
    err, orth = dc.pose_update_errors(tr, k["T0"])
    assert err <= POSE_STEP_TOL and orth <= ORTH_TOL, (err, orth)
    dc.check_flags(tr, k)
    dc.check_stats(g["stats"], tr, k)
    if tr:
        assert same(g["T"], tr[-1]["T"])
    else:
        assert same(g["T"], k["T0"])
    if not solve:
        return []
    p = k["p"]
    ref_f, cur_f = _frames_of(ctx, frames, p)

    def residuals(level, T, vis):
        return ctx.sparse_residuals(ref_f, cur_f, p["cam"], level, T, p["px"], p["f"], p["pos"], p["has_point"], p["ref_pos"],
                                    visible_in=vis)

    errs = dc.solve_errors(tr, k, residuals)
    for e, kappa in errs:
        assert e <= SOLVE_TOL * kappa, (e, kappa)
    return errs


def _geom_ok(L, cfg):
    if cfg[0] > 0 and L["ctas_per_pair"] != cfg[0]:
        return False
    if cfg[1] > 0 and L["features_per_thread"] != cfg[1]:
        return False
    if cfg[0] == 4 and cfg[2] == 0 and L["upfront"]:
        return False
    return L["n_pairs"] == 1 and not L["residuals_only"]


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
@pytest.mark.parametrize("name", dc.NAMES)
def test_driver_case_equals_oracle_and_statement(ctx, frames, name, geometry):
    k = dc.case(name)
    cfg = GEOMETRIES[geometry]
    _configure(ctx, cfg)
    before = ctx.launch_count()
    g = gpu_run(ctx, frames, k)
    assert ctx.launch_count() > before  # every case has features: a launch ran, in the geometry asked for
    L = ctx.sia_last_launch()
    assert _geom_ok(L, cfg), L
    o = oracle_run(k)
    assert_driver_parity(g, o, k)
    errs = assert_driver_statement(ctx, frames, g, k)
    if errs:
        print(f"MEASURE {name}/{geometry}: solve err / cond {max(e / c for e, c in errs):.2e}")


# ---- the exact edge of the convergence test (m <= eps) ---------------------------------------------------------------------
EPS_EDGE_CASE = "levels_4_2"


def eps_edge(run):
    """`run(eps)` on the EPS_EDGE_CASE: |x|_inf m of the accepted step (level 4, iteration 1), and for eps = m and
    eps = nextafter(m, 0) whether level 4 stopped at that step (the same step, bit for bit, in all three runs)."""
    base = run(None)
    step = next(t for t in base["trace"] if t["level"] == 4 and t["iter"] == 1)
    m = dc.xmax(step["x"])
    assert step["accepted"] and m > dc.case(EPS_EDGE_CASE)["eps"]
    stopped = []
    for eps in (m, np.nextafter(m, 0.0)):
        lv4 = [t for t in run(eps)["trace"] if t["level"] == 4]
        assert dc.xmax(lv4[1]["x"]) == m, eps
        stopped.append(len(lv4) == 2)
    return m, stopped


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_eps_edge_stops_at_equality_and_not_one_ulp_below(ctx, frames, geometry):
    """eps equal to an accepted step's |x|_inf stops the level at that step; nextafter(eps, 0) does not (m <= eps).  The
    kernel's and the oracle's |x|_inf of a step on a real scene differ in the last bits (the normal matrix is summed in
    another order; within X_ATOL), so each is put at its own edge.  Where the two are the same number -- x = 0 exactly on
    the zero-residual pair, with eps 0 (stops at once) and eps -5e-324 (never stops) -- they are compared with each other."""
    _configure(ctx, GEOMETRIES[geometry])
    k = dict(dc.case(EPS_EDGE_CASE), name="eps_edge")
    mk, sk = eps_edge(lambda eps: gpu_run(ctx, frames, k, eps=eps))
    mo, so = eps_edge(lambda eps: dc.oracle_run(k, eps=eps))
    assert sk == so == [True, False], (sk, so)
    assert abs(mk - mo) <= X_ATOL, (mk, mo)
    for name, n_levels in (("zero_eps_0", 1), ("zero_eps_neg", 5)):
        kz = dc.case(name)
        g, o = gpu_run(ctx, frames, kz), oracle_run(kz)
        assert all(dc.xmax(t["x"]) == 0.0 for t in g["trace"] + o["trace"])
        assert [t["iter"] for t in g["trace"]] == [t["iter"] for t in o["trace"]] == list(range(n_levels)) * 5


# ---- the compiled reference's recorded outputs ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", dc.REF_CASES)
def test_driver_case_equals_recorded_reference(ctx, frames, name):
    """The kernel against SparseImgAlign::run of the compiled reference as test_sia_driver_pins.py recorded it: mask and
    n_tracked exact, the final pose within sc.POSE_TOL (NaN where the reference's is; below RANK_OK features not compared)."""
    k = dc.case(name)
    r = RefCalls("test_sia_driver_pins", f"test_driver_oracle_equals_reference[{name}]")
    rr = dc.ref_run(r, k)
    r.finish()
    g = gpu_run(ctx, frames, k)
    assert np.array_equal(g["visible"], rr["visible"][:len(g["visible"])])
    assert g["n_tracked"] == rr["n_tracked"]
    T = synth.se3_mul(g["T"], k["p"]["T_ref_w"])
    assert np.array_equal(np.isnan(T), np.isnan(rr["T_cur_w"]))
    if len(k["p"]["px"]) >= dc.RANK_OK and not np.isnan(T).any():
        dt, dr = synth.pose_error(T, rr["T_cur_w"])
        assert dt <= sc.POSE_TOL and dr <= sc.POSE_TOL, (dt, dr)


# ---- every branch is reached -------------------------------------------------------------------------------------------------

def test_driver_branches_are_reached(ctx, frames):
    """Each path of the driver occurs in the kernel's own traces of the cases (auto geometry): counted and printed."""
    c = collections.Counter()
    for name in dc.NAMES:
        k = dc.case(name)
        g = gpu_run(ctx, frames, k)
        tr = g["trace"]
        by_level = collections.defaultdict(list)
        for t in tr:
            by_level[t["level"]].append(t)
        for lv, ts in by_level.items():
            last = ts[-1]
            if not last["accepted"] and not np.isnan(last["x"][0]) and last["iter"] > 0:
                c["roll-back"] += 1
            if last["accepted"] and dc.xmax(last["x"]) <= k["eps"]:
                c["eps stop"] += 1
            if last["accepted"] and len(ts) == k["n_iter"] and not dc.xmax(last["x"]) <= k["eps"]:
                c["iteration limit"] += 1
            if np.isnan(ts[0]["x"][0]) and ts[0]["iter"] == 0 and not ts[0]["accepted"]:
                c["NaN step stop"] += 1
        c["level without measurement"] += sum(1 for t in tr if t["n_meas"] == 0)
        th2 = [float(np.dot(t["x"][3:], t["x"][3:])) for t in tr if t["accepted"] and np.all(np.isfinite(t["x"]))]
        c["large-angle exponential (theta^2 >= 0.25)"] += sum(1 for v in th2 if v >= 0.25)
        c["theta^2 in [0.2, 0.25)"] += sum(1 for v in th2 if 0.2 <= v < 0.25)
        c["theta^2 in [0.25, 0.3)"] += sum(1 for v in th2 if 0.25 <= v < 0.3)
        if tr and (dc.min_pivot_ratio(g["H"]) <= 1e-13 or not np.isfinite(g["H"]).all()):
            c["pivoted solve"] += 1
        if name in dc.NONFINITE or name in ("nan_ref_pos", "nan_T0"):
            c[f"non-finite input: {name}"] += 1
    c["n_iter 0"] += int(not gpu_run(ctx, frames, dc.case("iters_0"))["trace"])
    c["n_iter < 0 (no limit)"] += int(len(gpu_run(ctx, frames, dc.case("iters_neg"))["trace"]) > 5)
    k = dict(dc.case(EPS_EDGE_CASE), name="eps_edge")
    _, (at, below) = eps_edge(lambda eps: gpu_run(ctx, frames, k, eps=eps))
    c["eps stop at the edge"] += int(at)
    c["eps edge passed one ulp below"] += int(not below)
    print("\ndriver branches reached:")
    for key in sorted(c):
        print(f"  {key}: {c[key]}")
    for key in ("roll-back", "eps stop", "iteration limit", "level without measurement", "pivoted solve",
                "large-angle exponential (theta^2 >= 0.25)", "NaN step stop", "n_iter 0", "n_iter < 0 (no limit)",
                "eps stop at the edge", "eps edge passed one ulp below"):
        assert c[key] > 0, key
    for name in dc.NONFINITE + ("nan_ref_pos", "nan_T0"):
        assert c[f"non-finite input: {name}"] > 0, name


# ---- a mixed batch in the throughput geometry -------------------------------------------------------------------------------
BATCH_CASES = [n for n in dc.NAMES if n in dc.BATCHABLE]
CLEAN = "rollback_3"  # what replaces the non-finite pairs


def _stage_run_fetch(ctx, frames, ks, runs=1):
    B = len(ks)
    ns = [len(k["p"]["px"]) for k in ks]
    off = np.concatenate([[0], np.cumsum(ns)]).astype(np.int32)
    cat = {key: np.concatenate([k["p"][key] for k in ks]) for key in ("px", "f", "pos", "has_point")}
    fr = [_frames_of(ctx, frames, k["p"]) for k in ks]
    ctx.sia_batch_stage([f[0] for f in fr], [f[1] for f in fr], ks[0]["p"]["cam"], np.stack([k["T0"] for k in ks]), off,
                        cat["px"], cat["f"], cat["pos"], cat["has_point"], np.stack([k["p"]["ref_pos"] for k in ks]), 4, 0, 30)
    for _ in range(runs):
        ctx.sia_batch_run()
    r = ctx.sia_batch_fetch(want_H=True)
    L = ctx.sia_last_launch()
    return r, off, L


def test_mixed_batch_equals_single_runs_and_oracle(ctx, frames):
    """Pair b is BATCH_CASES[b % len]: roll-backs, converging pairs, no measurements, rank-deficient and textureless pairs
    and every non-finite kind in one batch of more than one wave of the throughput geometry (160 threads x 2 features, three
    CTAs per SM).  Each pair equals its single run in that geometry bit for bit (T, H, mask, stats) and the oracle (mask,
    n_tracked, the stats against the oracle's trace, the pose); replacing the non-finite pairs with clean ones leaves every
    other pair bit-identical; two back-to-back runs of the staged batch fetch exactly what one does."""
    ks = [dc.case(BATCH_CASES[b % len(BATCH_CASES)]) for b in range(3 * 132 + 37)]
    assert all((k["n_iter"], k["eps"], k["max_level"], k["min_level"]) == (30, 1e-6, 4, 0) for k in ks)
    r, off, L = _stage_run_fetch(ctx, frames, ks)
    assert (L["ctas_per_pair"], L["threads"], L["features_per_thread"]) == (1, 160, 2) and L["n_pairs"] == len(ks), L
    ctx.sia_config(1, 2)
    single = {}
    for b, k in enumerate(ks):
        if k["name"] not in single:
            g = gpu_run(ctx, frames, k)
            assert (ctx.sia_last_launch()["threads"], ctx.sia_last_launch()["features_per_thread"]) == (160, 2)
            o = oracle_run(k)
            assert_driver_parity(g, o, k)
            if len(k["p"]["px"]) >= dc.RANK_OK:
                dc.check_stats(g["stats"], o["trace"], k)
            single[k["name"]] = g
        g = single[k["name"]]
        assert same(r["T"][b], g["T"]) and same(r["H"][b], g["H"]), (b, k["name"])
        assert np.array_equal(r["visible"][off[b]:off[b + 1]], g["visible"]), (b, k["name"])
        for key in ("n_iters", "sum_visible", "sum_in_image", "n_tracked"):
            assert r["stats"][b][key] == g["stats"][key], (b, k["name"], key)
    ctx.sia_config(-1, 0)
    # the non-finite pairs replaced by clean ones: every other pair is bit-identical
    bad = {n for n in dc.NONFINITE} | {"nan_ref_pos", "nan_T0"}
    ks2 = [dc.case(CLEAN) if k["name"] in bad else k for k in ks]
    r2, off2, _ = _stage_run_fetch(ctx, frames, ks2)
    for b, k in enumerate(ks):
        if k["name"] in bad:
            continue
        assert same(r2["T"][b], r["T"][b]) and same(r2["H"][b], r["H"][b]), b
        assert np.array_equal(r2["visible"][off2[b]:off2[b + 1]], r["visible"][off[b]:off[b + 1]]), b
        assert r2["stats"][b].tobytes() == r["stats"][b].tobytes(), b
    # two chained runs (programmatic dependent launch) fetch what one run does
    r3, _, _ = _stage_run_fetch(ctx, frames, ks, runs=2)
    assert same(r3["T"], r["T"]) and same(r3["H"], r["H"]) and np.array_equal(r3["visible"], r["visible"])
    assert r3["stats"].tobytes() == r["stats"].tobytes()
