"""GPU: the robust alignment kernel (svo_b200_sia_robust: MAD scale with unit, Tukey or Huber weights) against the oracle
(pinned on the compiled reference by test_sia_robust_pins.py) on the cases of tests/sia_robust_cases.py, in batches, and
when the mode is switched on and off."""
import os
import struct
import subprocess

import numpy as np
import pytest

from rpg_svo_b200 import capi, synth
from tests import sia_cases as sc
from tests import sia_robust_cases as rc

pytestmark = pytest.mark.gpu

NAMES = [k["name"] for k in rc.cases()]
POSE_TOL = 1e-9  # observed on an H100 (NVIDIA H100 80GB HBM3): 1.1e-13 m (occluded_unit)
CHI2_RTOL = 5e-5  # trace chi2, relative: serial f32 sum vs per-patch f32 then f64 (observed up to 5.0e-6)
KSIA_THREADS = {96, 160, 320, 384, 512}  # block sizes of sia_kernel's instantiations (the robust kernel runs 256)


@pytest.fixture(autouse=True)
def weights_off_after(ctx):
    """The context is shared with the other GPU tests: every test leaves the robust cost off."""
    yield
    ctx.sia_robust(capi.SCALE_UNIT, capi.WEIGHT_UNIT)


def gpu_run(ctx, k, weight=None, scale=capi.SCALE_MAD, frames=None):
    p = k["p"]
    ctx.sia_robust(scale, k["weight"] if weight is None else weight)
    ref, cur = frames if frames is not None else (ctx.frame(p["ref_pyr"]), ctx.frame(p["cur_pyr"]))
    g = ctx.sparse_img_align(ref, cur, p["cam"], synth.se3_identity(), p["px"], p["f"], p["pos"], p["has_point"], p["ref_pos"],
                             k["max_level"], k["min_level"], k["n_iter"], want_trace=True)
    if frames is None:
        ref.destroy(); cur.destroy()
    return g


@pytest.mark.parametrize("name", NAMES)
def test_robust_single_call_equals_oracle(ctx, oracle, name):
    """Mask and n_tracked exact; the scale bit for bit where it comes from the initial pose (the first level) and within
    1e-5 relative where a later level recomputed it; the trace's (level, iter, accepted, n_meas) equal and its chi2 within
    CHI2_RTOL; pose within POSE_TOL."""
    k = rc.case(name)
    o = rc.oracle_run(k)
    g = gpu_run(ctx, k)
    n = len(k["p"]["px"])
    assert np.array_equal(g["visible"], o["visible"])
    if n == 0:  # no launch: nothing tracked, the pose unchanged
        assert g["n_tracked"] == 0 and np.array_equal(g["T"], synth.se3_identity())
        return
    s = ctx.sia_last_scales(1)[0]
    lv = k["max_level"]
    assert rc.same_bits(s[lv], o["scales"][lv]), (s, o["scales"])
    assert np.all(np.isnan(s[[l for l in range(capi.MAX_LEVELS) if not k["min_level"] <= l <= k["max_level"]]]))
    if n < rc.RANK_OK:
        return
    assert g["n_tracked"] == o["n_tracked"], (g["n_tracked"], o["n_tracked"])
    for l in range(k["min_level"], k["max_level"]):
        assert s[l] == o["scales"][l] or abs(s[l] - o["scales"][l]) <= 1e-5 * abs(o["scales"][l]), (l, s, o["scales"])
    assert [(t["level"], t["iter"], t["accepted"], t["n_meas"]) for t in g["trace"]] == \
        [(t["level"], t["iter"], t["accepted"], t["n_meas"]) for t in o["trace"]]
    for a, b in zip(g["trace"], o["trace"]):
        assert (np.isnan(a["chi2"]) and np.isnan(b["chi2"])) or abs(a["chi2"] - b["chi2"]) <= CHI2_RTOL * abs(b["chi2"]), \
            (a["chi2"], b["chi2"])
    dt, dr = synth.pose_error(g["T"], o["T"])
    print(f"{name}: |dt| {dt:.2e} m, dR {dr:.2e} rad vs oracle")
    assert dt <= POSE_TOL and dr <= POSE_TOL, (dt, dr)


def _batch_sets():
    d = sc.base_pair()
    counts = [0, 1, 31, 32, 33, 300, 1024]
    return d, counts


@pytest.mark.parametrize("B", [1, 7, 300])
def test_robust_batch_equals_single_calls(ctx, B):
    """B pairs with feature counts cycling through 0, 1, 31, 32, 33, 300, 1024: pose, mask, H, stats and scales of the batch
    equal bit for bit those of single calls."""
    d, counts = _batch_sets()
    d["has_point"][::13] = 0
    ns = [counts[b % len(counts)] for b in range(B)]
    off = np.concatenate([[0], np.cumsum(ns)]).astype(np.int32)
    idx = np.concatenate([np.arange(n) for n in ns]).astype(int) if off[-1] else np.zeros(0, int)
    cat = {k: np.ascontiguousarray(d[k][idx]) for k in ("px", "f", "pos", "has_point")}
    ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
    ctx.sia_robust(capi.SCALE_MAD, capi.WEIGHT_TUKEY)
    T0 = np.tile(synth.se3_identity().reshape(1, 12), (B, 1))
    ctx.sia_batch_stage([ref] * B, [cur] * B, d["cam"], T0, off, cat["px"], cat["f"], cat["pos"], cat["has_point"],
                        np.tile(d["ref_pos"], (B, 1)), 4, 0, 10)
    ctx.sia_batch_run()
    bt = ctx.sia_batch_fetch(want_H=True)
    bs = ctx.sia_last_scales(B)
    single = {}
    for b in range(B):
        n = ns[b]
        if n not in single:
            if n == 0:
                single[n] = None
            else:
                g = ctx.sparse_img_align(ref, cur, d["cam"], synth.se3_identity(), d["px"][:n], d["f"][:n], d["pos"][:n],
                                         d["has_point"][:n], d["ref_pos"], 4, 0, 10)
                single[n] = (g, ctx.sia_last_scales(1)[0], ctx.sia_last_launch())
        if n == 0:
            assert bt["stats"][b]["n_tracked"] == 0 and np.array_equal(bt["T"][b], synth.se3_identity())
            continue
        g, s, L = single[n]
        assert np.array_equal(bt["T"][b], g["T"]) and np.array_equal(bt["H"][b], g["H"]), b
        assert np.array_equal(bt["visible"][off[b]:off[b + 1]], g["visible"]), b
        assert bt["stats"][b]["n_tracked"] == g["n_tracked"] and rc.same_bits(bs[b], s), b
        assert L["threads"] == 256
    ref.destroy(); cur.destroy()


def test_robust_feature_limit(ctx):
    d, _ = _batch_sets()
    ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
    ctx.sia_robust(capi.SCALE_MAD, capi.WEIGHT_HUBER)
    with pytest.raises(capi.SvoB200Error, match="-4"):
        ctx.sparse_img_align(ref, cur, d["cam"], synth.se3_identity(), d["px"][:1025], d["f"][:1025], d["pos"][:1025],
                             d["has_point"][:1025], d["ref_pos"], 4, 0)
    ref.destroy(); cur.destroy()


def test_robust_mode_switching(ctx):
    """MAD with unit weights matches the unweighted kernel's pose within 1e-7; UnitScale with any weight is the unweighted
    launch, bit for bit what a context that never set a mode computes; weights on and then off again give the same bits."""
    k = rc.case("tukey")
    p = k["p"]
    fresh = capi.Context(0)
    try:
        ref, cur = fresh.frame(p["ref_pyr"]), fresh.frame(p["cur_pyr"])
        base = fresh.sparse_img_align(ref, cur, p["cam"], synth.se3_identity(), p["px"], p["f"], p["pos"], p["has_point"],
                                      p["ref_pos"], 4, 0, want_trace=True)
        ref.destroy(); cur.destroy()
    finally:
        fresh.close()
    u = gpu_run(ctx, k, weight=capi.WEIGHT_UNIT)
    dt, dr = synth.pose_error(u["T"], base["T"])
    print(f"MAD + unit weights vs unweighted: |dt| {dt:.2e} m, dR {dr:.2e} rad")
    assert dt <= 1e-7 and dr <= 1e-7
    for w in (capi.WEIGHT_UNIT, capi.WEIGHT_TDIST, capi.WEIGHT_TUKEY, capi.WEIGHT_HUBER):
        g = gpu_run(ctx, k, weight=w, scale=capi.SCALE_UNIT)
        assert ctx.sia_last_launch()["threads"] in KSIA_THREADS
        with pytest.raises(capi.SvoB200Error):
            ctx.sia_last_scales(1)
        assert np.array_equal(g["T"], base["T"]) and np.array_equal(g["H"], base["H"]) and g["n_tracked"] == base["n_tracked"]
    gpu_run(ctx, k, weight=capi.WEIGHT_TUKEY)
    assert ctx.sia_last_launch()["threads"] == 256
    g = gpu_run(ctx, k, weight=capi.WEIGHT_TUKEY, scale=capi.SCALE_UNIT)
    assert np.array_equal(g["T"], base["T"]) and np.array_equal(g["H"], base["H"])


def test_robust_residual_pass_ignores_the_mode(ctx):
    """svo_b200_sparse_residuals runs the unweighted residual pass whatever the mode."""
    k = rc.case("tukey")
    p = k["p"]
    ref, cur = ctx.frame(p["ref_pyr"]), ctx.frame(p["cur_pyr"])
    args = (ref, cur, p["cam"], 2, synth.se3_identity(), p["px"], p["f"], p["pos"], p["has_point"], p["ref_pos"])
    ctx.sia_robust(capi.SCALE_UNIT, capi.WEIGHT_UNIT)
    a = ctx.sparse_residuals(*args)
    ctx.sia_robust(capi.SCALE_MAD, capi.WEIGHT_TUKEY)
    b = ctx.sparse_residuals(*args)
    assert ctx.sia_last_launch()["residuals_only"] == 1
    for key in a:
        assert np.array_equal(np.asarray(a[key]), np.asarray(b[key]), equal_nan=np.asarray(a[key]).dtype.kind == "f"), key
    ref.destroy(); cur.destroy()


def test_robust_tukey_beats_plain_gauss_newton_on_occlusion(ctx):
    """As on the oracle (test_sia_robust_pins.py): Tukey ends within 0.01 m of the ground truth, plain Gauss-Newton over 0.5 m."""
    k = rc.case("occluded_tukey")
    gt = k["p"]["T_cur_ref_gt"]
    e_t = synth.pose_error(gpu_run(ctx, k)["T"], gt)[0]
    e_u = synth.pose_error(gpu_run(ctx, k, scale=capi.SCALE_UNIT)["T"], gt)[0]
    print(f"occluded pair: Tukey {e_t:.2e} m, plain Gauss-Newton {e_u:.2e} m from the ground truth")
    assert e_t < 0.01 and e_u > 0.5, (e_t, e_u)


def test_robust_argument_errors(ctx):
    for scale, weight in [(capi.SCALE_TDIST, capi.WEIGHT_TUKEY), (capi.SCALE_NORMAL, capi.WEIGHT_UNIT),
                          (capi.SCALE_MAD, capi.WEIGHT_TDIST), (4, 0), (-1, 0), (capi.SCALE_MAD, 7)]:
        with pytest.raises(capi.SvoB200Error, match="-1"):
            ctx.sia_robust(scale, weight)
    ctx.sia_robust(capi.SCALE_UNIT, capi.WEIGHT_UNIT)
    k = rc.case("tukey")
    gpu_run(ctx, k, scale=capi.SCALE_UNIT)
    with pytest.raises(capi.SvoB200Error, match="-1"):
        ctx.sia_last_scales(1)
    # weights with an active multi-GPU feature split (two contexts of this process as the split's two ranks)
    other = capi.Context(0)
    try:
        _, p0 = ctx.sia_split_create(0, 2, 1)
        _, p1 = other.sia_split_create(1, 2, 1)
        ctx.sia_split_connect(in_process_ptrs=[p0, p1])
        with pytest.raises(capi.SvoB200Error, match="-1"):
            ctx.sia_robust(capi.SCALE_MAD, capi.WEIGHT_TUKEY)
        ctx.sia_split_destroy()
        ctx.sia_robust(capi.SCALE_MAD, capi.WEIGHT_TUKEY)  # set before the split is connected: the launch is refused
        _, p0 = ctx.sia_split_create(0, 2, 1)
        ctx.sia_split_connect(in_process_ptrs=[p0, p1])
        p = k["p"]
        ref, cur = ctx.frame(p["ref_pyr"]), ctx.frame(p["cur_pyr"])
        with pytest.raises(capi.SvoB200Error, match="-1"):
            ctx.sparse_img_align(ref, cur, p["cam"], synth.se3_identity(), p["px"], p["f"], p["pos"], p["has_point"],
                                 p["ref_pos"], 4, 0)
        ref.destroy(); cur.destroy()
    finally:
        ctx.sia_split_destroy()
        other.sia_split_destroy()
        other.close()


def test_robust_host_mirror(ctx, oracle, tmp_path):
    """svo::SparseImgAlign with setRobustCostFunction(MADScale, TukeyWeight) (host_robust_demo over svo_host.h): pose, patch
    count and Fisher information as the oracle's; a second object on the same context without a robust cost runs
    unweighted."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    host = os.path.join(root, "rpg_svo_b200", "host")
    exe = os.path.join(host, "host_robust_demo")
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(exe + ".cpp"), os.path.getmtime(os.path.join(host, "svo_host.h"))):
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-pthread", "-o", exe, exe + ".cpp", "-L" + os.path.join(root, "rpg_svo_b200"),
                               "-lsvo_b200", "-Wl,-rpath,$ORIGIN/.."])
    k = rc.case("occluded_tukey")
    p = k["p"]
    cam, N = p["cam"], len(p["px"])
    inp, outp = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as fh:
        fh.write(struct.pack("7i", cam.width, cam.height, p["n_levels"], N, 4, 0, capi.WEIGHT_TUKEY))
        fh.write(struct.pack("4d", cam.fx, cam.fy, cam.cx, cam.cy))
        fh.write(p["ref_pyr"][0].tobytes()); fh.write(p["cur_pyr"][0].tobytes())
        fh.write(np.ascontiguousarray(p["T_ref_w"]).tobytes())
        for a in (p["px"], p["f"], p["pos"]):
            fh.write(np.ascontiguousarray(a, np.float64).tobytes())
        fh.write(np.ascontiguousarray(p["has_point"], np.uint8).tobytes())
    out = subprocess.run([exe, str(inp), str(outp)], check=True, capture_output=True, text=True).stdout
    print(out)
    raw = open(outp, "rb").read()
    sigma_i_sq = 5e-4 * 255 * 255
    o_r = rc.oracle_run(k)
    o_p = oracle.sparse_img_align(p["ref_pyr"], p["cur_pyr"], cam, synth.se3_identity(), p["px"], p["f"], p["pos"], p["has_point"],
                                  p["ref_pos"], 4, 0)
    for j, o in enumerate((o_r, o_p)):
        base = j * (96 + 8 + 288)
        T = np.frombuffer(raw, np.float64, 12, base).reshape(3, 4)
        n_tracked = struct.unpack_from("q", raw, base + 96)[0]
        fisher = np.frombuffer(raw, np.float64, 36, base + 104).reshape(6, 6)
        dt, dr = synth.pose_error(T, oracle.se3_mul(o["T"], p["T_ref_w"]))
        print(f"host mirror {'robust' if j == 0 else 'plain'}: |dt| {dt:.2e} m, dR {dr:.2e} rad vs oracle")
        assert dt < 1e-4 and dr < 1e-4 and n_tracked == o["n_tracked"]
        assert np.allclose(fisher, o["H"] / sigma_i_sq, rtol=1e-6, atol=1e-9 * np.abs(o["H"]).max() / sigma_i_sq)
