"""GPU: the robust alignment kernel (sia_robust_kernel) against the oracle on the edge cases of tests/sia_robust_edge_cases.py
(every slot edge, odd sizes, borders, level ranges, pyramid depths, initial poses, a coarsest level without patches, tie-heavy
images), its MAD scale against an exact numpy median, heterogeneous batches against single calls, and the robust mode as
a batch is staged."""
import numpy as np
import pytest

from rpg_svo_b200 import capi, synth
from tests import sia_cases as sc
from tests import sia_robust_cases as rc
from tests import sia_robust_edge_cases as ec

pytestmark = pytest.mark.gpu

# Observed on an H100 (NVIDIA H100 80GB HBM3) over every case of this file, maxima in parentheses:
POSE_TOL = 1e-9     # final pose vs the oracle
CHI2_RTOL = 5e-5    # trace chi2, relative: serial f32 sum vs per-patch f32 then f64 (5.8e-6)
H_RTOL = 1e-13      # H vs the oracle's H, relative to max |H|
KSIA_THREADS = {96, 160, 320, 384, 512}


@pytest.fixture(autouse=True)
def weights_off_after(ctx):
    yield
    ctx.sia_robust(capi.SCALE_UNIT, capi.WEIGHT_UNIT)


def gpu_run(ctx, k, frames=None):
    p = k["p"]
    ctx.sia_robust(capi.SCALE_MAD, k["weight"])
    ref, cur = frames if frames is not None else (ctx.frame(p["ref_pyr"]), ctx.frame(p["cur_pyr"]))
    g = ctx.sparse_img_align(ref, cur, p["cam"], k["T0"], p["px"], p["f"], p["pos"], p["has_point"], p["ref_pos"],
                             k["max_level"], k["min_level"], k["n_iter"], want_trace=True)
    g["scales"] = ctx.sia_last_scales(1)[0] if len(p["px"]) else None
    if frames is None:
        ref.destroy(); cur.destroy()
    return g


def same_chi2(a, b):
    """Within CHI2_RTOL, NaN (a pass without an in-image patch, or Huber with a zero scale) equal to NaN."""
    return (np.isnan(a) and np.isnan(b)) or a == b or abs(a - b) <= CHI2_RTOL * abs(b)


def assert_robust_parity(g, o, k, medians=None):
    """Kernel result `g` (with its `scales`) vs the oracle's `o` on case `k`: mask exact; the first level's scale bit for bit
    (and against `medians`, {level: numpy scale}); below RANK_OK features nothing else.  Otherwise the oracle's run is at
    least ec.MARGIN from flipping a Gauss-Newton decision, and every scale is bit for bit, n_tracked exact, the trace's
    (level, iter, accepted, n_meas) exact and chi2 within CHI2_RTOL, H within H_RTOL with NaN where the oracle has NaN, the
    pose within POSE_TOL."""
    n = len(k["p"]["px"])
    assert np.array_equal(g["visible"], o["visible"]), "visibility mask"
    if n == 0:
        assert g["n_tracked"] == 0 and np.array_equal(g["T"], k["T0"])
        return
    s = g["scales"]
    lv = k["max_level"]
    run = list(range(k["min_level"], lv + 1))
    assert rc.same_bits(s[lv], o["scales"][lv]), (s, o["scales"])
    assert np.all(np.isnan(s[[l for l in range(capi.MAX_LEVELS) if l not in run]]))
    for l, m in (medians or {}).items():
        assert rc.same_bits(s[l], 0.0 if m is None else m), (l, s[l], m)
    if n < rc.RANK_OK:
        return
    assert sc.decision_margin(o) >= ec.MARGIN, sc.decision_margin(o)
    assert rc.same_bits(s, o["scales"]), (s, o["scales"])
    assert g["n_tracked"] == o["n_tracked"], (g["n_tracked"], o["n_tracked"])
    assert len(g["trace"]) == len(o["trace"]), (len(g["trace"]), len(o["trace"]))
    for a, b in zip(g["trace"], o["trace"]):
        assert (a["level"], a["iter"], a["accepted"], a["n_meas"]) == (b["level"], b["iter"], b["accepted"], b["n_meas"])
        assert same_chi2(a["chi2"], b["chi2"]), (a["chi2"], b["chi2"])
    if k["n_iter"] > 0:
        assert np.array_equal(np.isnan(g["H"]), np.isnan(o["H"]))
        m = ~np.isnan(o["H"])
        if m.any():
            assert np.max(np.abs(g["H"][m] - o["H"][m])) <= H_RTOL * max(np.abs(o["H"][m]).max(), 1e-300)
    dt, dr = synth.pose_error(g["T"], o["T"])
    assert dt <= POSE_TOL and dr <= POSE_TOL, (dt, dr)


def report(name, g, o):
    """Observed differences, printed for the tolerances above."""
    if len(g["visible"]) < rc.RANK_OK or not o["trace"]:
        return
    dt, dr = synth.pose_error(g["T"], o["T"])
    c2 = max((abs(a["chi2"] - b["chi2"]) / abs(b["chi2"]) for a, b in zip(g["trace"], o["trace"]) if b["chi2"] and
              np.isfinite(b["chi2"])), default=0.0)
    m = ~np.isnan(o["H"])
    h = np.max(np.abs(g["H"][m] - o["H"][m])) / np.abs(o["H"][m]).max() if m.any() and np.abs(o["H"][m]).max() > 0 else 0.0
    ok = ~np.isnan(o["scales"]) & (o["scales"] != 0)
    sr = np.max(np.abs(g["scales"][ok] - o["scales"][ok]) / o["scales"][ok]) if ok.any() else 0.0
    print(f"MEASURE {name}: pose {max(dt, dr):.2e} chi2 {c2:.2e} H {h:.2e} scale {sr:.2e}")


@pytest.mark.parametrize("name", ec.names())
def test_robust_edge_case_equals_oracle(ctx, oracle, name):
    k = ec.case(name)
    o = ec.oracle_run(k)
    g = gpu_run(ctx, k)
    report(name, g, o)
    assert_robust_parity(g, o, k, ec.numpy_scales(oracle, k))


# ---- heterogeneous batches --------------------------------------------------------------------------------------------------
# The batch's pairs share the camera, the weight, the level range and n_iter: they are the 640x480 Tukey cases of
# sia_robust_edge_cases run at levels 4..0 with 30 iterations (each clear of near-ties), and pairs of 0 and 1 features.
# The cases drawn from sc.base_pair() run on FramePool frames (whose pyramids the pool builds: the oracle runs on those levels).
BATCH_CASES = ["slots_256_tukey", "t0_perturbed", "empty", "one", "slots_1024_tukey", "ties_4_tukey", "slots_255_tukey",
               "admissible_tukey", "slots_511_tukey", "t0_converged", "slots_769_tukey", "coarse_empty_iters_30",
               "slots_257_tukey", "slots_1024_live_tukey", "ties_2_tukey", "slots_767_tukey", "slots_513_tukey",
               "slots_1023_tukey", "slots_512_tukey", "slots_768_tukey"]


@pytest.fixture(scope="module")
def batch_cases(ctx):
    """{name: (case, (ref, cur) frames, oracle result)} for BATCH_CASES; frames are shared by the cases of one scene."""
    pool = capi.FramePool(ctx, 640, 480, 5, 2)
    base = sc.base_pair()
    pool.upload_array(np.stack([base["ref_pyr"][0], base["cur_pyr"][0]]))
    pool_pyr = ([pool.frames[0].download_level(l) for l in range(5)], [pool.frames[1].download_level(l) for l in range(5)])
    frames, out = {}, {}
    rng = np.random.default_rng(7)
    for name in BATCH_CASES:
        if name in ("empty", "one"):
            n = 0 if name == "empty" else 1
            xi = np.concatenate([rng.uniform(-2e-3, 2e-3, 3), np.deg2rad(rng.uniform(-0.1, 0.1, 3))])
            k = dict(name=name, p=ec.robust_subset(base, n, clear_edges=False), weight=rc.WEIGHTS["tukey"], n_iter=30,
                     max_level=4, min_level=0, T0=synth.se3_exp(xi))
        else:
            k = dict(ec.case(name))
        p = k["p"]
        if name in ("empty", "one") or (name.startswith("slots_") and ec.seed_of(name)[0] == 0):  # sc.base_pair(): the pool
            k["p"] = dict(p, ref_pyr=pool_pyr[0], cur_pyr=pool_pyr[1])
            f = (pool.frames[0], pool.frames[1])
        else:
            key = id(p["ref_pyr"])
            if key not in frames:
                frames[key] = (ctx.frame(p["ref_pyr"]), ctx.frame(p["cur_pyr"]))
            f = frames[key]
        assert k["p"]["cam"].width == 640 and k["weight"] == rc.WEIGHTS["tukey"] and k["n_iter"] == 30
        assert (k["max_level"], k["min_level"]) == (4, 0)
        out[name] = (k, f, ec.oracle_run(k))
    yield out
    for r, c in frames.values():
        r.destroy(); c.destroy()
    pool.destroy()


@pytest.mark.parametrize("B", [2, 33, 300])
def test_robust_heterogeneous_batch(ctx, batch_cases, B):
    """Pair b is BATCH_CASES[b % 20]: its own frames (single frames or a pool's), T0, ref_pos and 0-1024 features.  Pose,
    H, mask, stats and scales of each pair equal bit for bit its single call (a pair without features: the pose as given,
    H and stats 0, scales NaN, as a single call that launches nothing), and each pair passes assert_robust_parity against
    its own oracle run."""
    ks = [batch_cases[BATCH_CASES[b % len(BATCH_CASES)]] for b in range(B)]
    ns = [len(k["p"]["px"]) for k, _, _ in ks]
    off = np.concatenate([[0], np.cumsum(ns)]).astype(np.int32)
    cat = {key: np.concatenate([k["p"][key] for k, _, _ in ks]) for key in ("px", "f", "pos", "has_point")}
    ctx.sia_robust(capi.SCALE_MAD, capi.WEIGHT_TUKEY)
    ctx.sia_batch_stage([f[0] for _, f, _ in ks], [f[1] for _, f, _ in ks], ks[0][0]["p"]["cam"],
                        np.stack([k["T0"].reshape(12) for k, _, _ in ks]), off, cat["px"], cat["f"], cat["pos"],
                        cat["has_point"], np.stack([k["p"]["ref_pos"] for k, _, _ in ks]), 4, 0, 30)
    ctx.sia_batch_run()
    bt = ctx.sia_batch_fetch(want_H=True)
    bs = ctx.sia_last_scales(B)
    assert ctx.sia_last_launch()["threads"] == 256
    single = {}
    for b, (k, f, o) in enumerate(ks):
        if k["name"] not in single:
            g = gpu_run(ctx, k, frames=f)
            if ns[b] == 0:  # no launch: what the kernel must write for the pair
                g["scales"] = np.full(capi.MAX_LEVELS, np.nan, np.float32)
                assert np.array_equal(g["T"], k["T0"]) and not g["H"].any() and not any(g["stats"].values())
            assert_robust_parity(g, o, k)
            single[k["name"]] = g
        g = single[k["name"]]
        assert np.array_equal(bt["T"][b], g["T"]) and np.array_equal(bt["H"][b], g["H"], equal_nan=True), b
        assert np.array_equal(bt["visible"][off[b]:off[b + 1]], g["visible"]), b
        for key in ("n_iters", "sum_visible", "sum_in_image", "n_tracked"):
            assert bt["stats"][b][key] == g["stats"][key], (b, key)
        assert rc.same_bits(bs[b], g["scales"]), b
        if ns[b] == 0:
            assert rc.same_bits(bs[b], o["scales"]), b


# ---- the mode is what the batch was staged with ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scenes(ctx):
    d = sc.base_pair()
    frames = (ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"]))
    yield [dict(d=d, frames=frames)]
    frames[0].destroy(); frames[1].destroy()


def _stage_two(ctx, d, ref, cur):
    n = 200
    s = ec.robust_subset(d, n)
    off = np.array([0, n, 2 * n], np.int32)
    cat = {key: np.concatenate([s[key], s[key]]) for key in ("px", "f", "pos", "has_point")}
    ctx.sia_batch_stage([ref, ref], [cur, cur], d["cam"], np.tile(synth.se3_identity().reshape(1, 12), (2, 1)), off,
                        cat["px"], cat["f"], cat["pos"], cat["has_point"], np.tile(d["ref_pos"], (2, 1)), 4, 0, 10)


def test_robust_mode_is_captured_at_stage_time(ctx, scenes):
    """Staged with Tukey and run after switching to SCALE_UNIT: the robust kernel runs (256 threads) and reports scales.
    Staged unweighted and run after switching Tukey on: sia_kernel runs and there are no scales."""
    d = scenes[0]["d"]
    ref, cur = scenes[0]["frames"]
    ctx.sia_robust(capi.SCALE_MAD, capi.WEIGHT_TUKEY)
    _stage_two(ctx, d, ref, cur)
    ctx.sia_robust(capi.SCALE_UNIT, capi.WEIGHT_UNIT)
    ctx.sia_batch_run()
    weighted = ctx.sia_batch_fetch(want_H=True)
    assert ctx.sia_last_launch()["threads"] == 256
    s = ctx.sia_last_scales(2)
    assert np.all(s[:, :5] > 0) and rc.same_bits(s[0], s[1])
    _stage_two(ctx, d, ref, cur)
    ctx.sia_robust(capi.SCALE_MAD, capi.WEIGHT_TUKEY)
    ctx.sia_batch_run()
    plain = ctx.sia_batch_fetch(want_H=True)
    assert ctx.sia_last_launch()["threads"] in KSIA_THREADS
    with pytest.raises(capi.SvoB200Error, match="-1"):
        ctx.sia_last_scales(1)
    assert not np.array_equal(weighted["T"], plain["T"])


def test_robust_last_scales_errors(ctx, scenes):
    """More pairs than the last launch had is EINVAL; after an unweighted launch, any request is."""
    d = scenes[0]["d"]
    ref, cur = scenes[0]["frames"]
    ctx.sia_robust(capi.SCALE_MAD, capi.WEIGHT_HUBER)
    _stage_two(ctx, d, ref, cur)
    ctx.sia_batch_run()
    ctx.sia_batch_fetch()
    assert ctx.sia_last_scales(2).shape == (2, capi.MAX_LEVELS)
    with pytest.raises(capi.SvoB200Error, match="-1"):
        ctx.sia_last_scales(3)
    ctx.sia_robust(capi.SCALE_UNIT, capi.WEIGHT_UNIT)
    s = ec.robust_subset(d, 100)
    ctx.sparse_img_align(ref, cur, d["cam"], synth.se3_identity(), s["px"], s["f"], s["pos"], s["has_point"], d["ref_pos"], 4, 0)
    for B in (1, 2):
        with pytest.raises(capi.SvoB200Error, match="-1"):
            ctx.sia_last_scales(B)
