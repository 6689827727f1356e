"""GPU: depth_filter_kernel (DepthFilter::updateSeeds) and its match-only mode (Matcher::findEpipolarMatchDirect) on the
paths the default cases never reach or never check: several keyframes, every branch of the epipolar scan, the search-step
limit at its edge, equal ZMSSD scores, and seeds in every status (bad variances included) -- against the oracle and the
compiled reference's recorded outputs."""
import numpy as np
import pytest

from oracle import binding
from rpg_svo_b200 import synth
from tests import depth_update_hp as hp
from tests.ref_golden import RefCalls

pytestmark = pytest.mark.gpu

NO_MATCH, UPDATED = 4, 5
SEED_KEYS = ("a", "b", "mu", "sigma2")


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _check_update(g, o, c, kf_T, min_updated=0, oracle_statement=True):
    """status and n_zmssd bit-exact; seeds that never reach updateSeed bit-identical; every updated seed of the kernel
    bit for bit one of the exactly rounded statement's candidates from its own depth (tests/depth_update_hp.py: only
    expf, computeTau's acos / sin / atan and the pose product are left open), and the oracle's bit for bit its own."""
    assert np.array_equal(g["status"], o["status"])
    assert np.array_equal(g["n_zmssd"], o["n_zmssd"])
    upd = o["status"] >= UPDATED
    assert upd.sum() >= min_updated
    hp.assert_seed_updates(g, o, c["seeds"], kf_T, c["ref_index"], c["T_cur_w"], c["ftr_f"], c["cam"].fx, binding,
                           oracle_statement=oracle_statement)
    assert np.max(np.abs(g["px_cur"][upd] - o["px_cur"][upd]), initial=0.0) <= 1e-4
    assert np.allclose(g["z"][upd], o["z"][upd], rtol=1e-6)


def _run_both(ctx, oracle, kf_pyr, kf_T, c, seeds=None, **kw):
    frames = [ctx.frame(p) for p in kf_pyr]
    cur = ctx.frame(c["cur_pyr"])
    seeds = c["seeds"] if seeds is None else seeds
    a = (c["ref_index"], c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"], c["batch_counter"], seeds)
    g = ctx.depth_filter_update(frames, kf_T, cur, c["T_cur_w"], c["cam"], *a, **kw)
    o = oracle.depth_filter_update(kf_pyr, kf_T, c["cur_pyr"], c["T_cur_w"], c["cam"], *a, **kw)
    for f in frames + [cur]:
        f.destroy()
    return g, o


# ---- 2a: several keyframes ------------------------------------------------------------------------------------------------
def test_depth_filter_two_keyframes_vs_oracle_and_reference(ctx, oracle):
    """The case of test_oracle_depth_filter_two_keyframes_equals_reference_source_compiled_here (ref_index per seed, 50 %
    edgelets, baseline 0.5) on the kernel, against the oracle and the reference's outputs recorded for that pin."""
    a = synth.make_depth_case(61, n_seeds=300, baseline=0.5)
    b = synth.make_two_view(62, baseline=0.25)
    rng = np.random.default_rng(3)
    ref_index = rng.integers(0, 2, a["M"]).astype(np.int32)
    ftr_type = (rng.uniform(size=a["M"]) < 0.5).astype(np.int32)
    kf_pyr, kf_T = [a["ref_pyr"], b["ref_pyr"]], [a["T_ref_w"], b["T_ref_w"]]
    c = dict(a, ref_index=ref_index, ftr_type=ftr_type)
    g, o = _run_both(ctx, oracle, kf_pyr, kf_T, c)
    _check_update(g, o, c, kf_T, min_updated=50)
    r = RefCalls("test_oracle_pins", "test_oracle_depth_filter_two_keyframes_equals_reference_source_compiled_here")
    rr = r.depth_filter_update([k[0] for k in kf_pyr], kf_T, a["cur_pyr"][0], a["T_cur_w"], a["n_levels"], a["cam"],
                               ref_index, a["ftr_px"], a["ftr_f"], a["ftr_level"], ftr_type, a["ftr_grad"], a["batch_id"],
                               a["batch_counter"], a["seeds"])
    r.finish()
    st = g["status"]
    assert np.array_equal(rr["status"], np.where(st == 6, 1, np.where((st == 1) | (st == 7), 2, 0)))
    keep = rr["status"] == 0
    nomatch = st == NO_MATCH
    assert np.array_equal(_bits(g["b"][nomatch]), _bits(rr["b"][nomatch]))
    for k in SEED_KEYS:
        assert np.allclose(g[k][keep], rr[k][keep], rtol=2e-5, atol=1e-7), k


@pytest.mark.parametrize("n_kfs", [3, 5])
def test_depth_filter_interleaved_keyframes(ctx, oracle, n_kfs):
    """Keyframes with different poses and images, seeds interleaving them (ref_index 0, 1, 2, 0, ...): a kernel that read
    another keyframe's image or pose than ref_index names would scan the wrong patch along the wrong line."""
    c = synth.make_multi_keyframe_depth_case(70 + n_kfs, n_seeds=400, n_kfs=n_kfs)
    g, o = _run_both(ctx, oracle, c["kf_pyr"], c["kf_T"], c)
    _check_update(g, o, c, c["kf_T"], min_updated=100)
    upd = o["status"] >= UPDATED
    for r in range(n_kfs):  # every keyframe's seeds are measured, near their own true depth
        m = upd & (c["ref_index"] == r)
        assert m.sum() > 10, r
        assert np.median(np.abs(g["z"][m] - c["depth_gt"][m])) < 0.05, r


# ---- 2d: every seed status, bad variances ----------------------------------------------------------------------------------
def test_depth_filter_every_seed_status(ctx, oracle):
    """TOO_OLD, BEHIND, NOT_IN_FRAME, NO_MATCH, UPDATED and CONVERGED in one launch, plus seeds whose sigma2 is negative,
    NaN or infinite, against the oracle and the reference's outputs recorded by test_edge_pins.py."""
    c = synth.make_seed_status_case(91)
    g, o = _run_both(ctx, oracle, [c["ref_pyr"]], [c["T_ref_w"]], c)
    _check_update(g, o, c, [c["T_ref_w"]], min_updated=50)
    st = g["status"]
    counts = {s: int((st == s).sum()) for s in range(1, 8)}
    print("seed statuses (1 too old .. 6 converged, 7 NaN):", counts)
    for s in range(1, 7):
        assert counts[s] > 0, s
    # NAN (z_inv_min NaN after a successful match) cannot happen: z_inv_min = mu + sqrt(sigma2) is NaN only for a NaN mu
    # or a negative / NaN sigma2, and then d_min is NaN, the epipolar segment has a NaN end and the scan never starts.
    # For the same seeds the kernel's fmaxf gives z_inv_max = 1e-8 where the reference's std::max gives NaN; the segment is
    # NaN either way, so both end in NO_MATCH with b + 1 -- which the reference comparison below confirms.
    assert counts[7] == 0
    s2 = c["seeds"]["sigma2"]
    nan_min = c["bad_sigma2"] & ~(s2 > 0) & (st >= NO_MATCH)
    assert nan_min.sum() > 5 and np.all(st[nan_min] == NO_MATCH)
    r = RefCalls("test_edge_pins", "test_depth_seed_statuses_oracle_equals_reference")
    rr = r.depth_filter_update([c["ref_pyr"][0]], [c["T_ref_w"]], c["cur_pyr"][0], c["T_cur_w"], c["n_levels"], c["cam"],
                               c["ref_index"], c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"],
                               c["batch_id"], c["batch_counter"], c["seeds"])
    r.finish()
    assert np.array_equal(rr["status"], np.where(st == 6, 1, np.where((st == 1) | (st == 7), 2, 0)))
    untouched = (st != UPDATED) & (rr["status"] == 0)  # kept seeds that never reached updateSeed: bit for bit
    for k in SEED_KEYS:
        assert np.array_equal(_bits(g[k][untouched]), _bits(rr[k][untouched])), k


@pytest.mark.parametrize("limit", [25, 40, 60, 100])
def test_depth_filter_search_step_limit(ctx, oracle, limit):
    """max_epi_search_steps below the default: the seeds whose outcome the limit changes (against the same call at the
    default of 1000) are exactly skipped scans -- NO_MATCH with no score -- and there are some."""
    c = synth.make_depth_case(33, n_seeds=1500, baseline=0.3)
    g, o = _run_both(ctx, oracle, [c["ref_pyr"]], [c["T_ref_w"]], c, max_epi_search_steps=limit)
    _check_update(g, o, c, [c["T_ref_w"]], oracle_statement=False)
    gd, od = _run_both(ctx, oracle, [c["ref_pyr"]], [c["T_ref_w"]], c)
    _check_update(gd, od, c, [c["T_ref_w"]], oracle_statement=False)
    changed = (g["status"] != gd["status"]) | (g["n_zmssd"] != gd["n_zmssd"])
    assert changed.sum() > 0
    assert np.all(g["status"][changed] == NO_MATCH) and np.all(g["n_zmssd"][changed] == 0)
    assert np.all(gd["n_zmssd"][changed] > 0)  # at the default limit these seeds were scanned


# ---- 2b / 2c: the match-only API, branch by branch ------------------------------------------------------------------------
def _match_both(ctx, oracle, c, cur_pyr, T_cur_w, idx, d, **kw):
    """Kernel (one launch for the candidates idx) and oracle (one call per candidate) for the depth ranges d = (est, min, max)."""
    T_cur_ref = synth.se3_mul(T_cur_w, synth.se3_inv(c["T_ref_w"]))
    fr, fc = ctx.frame(c["ref_pyr"]), ctx.frame(cur_pyr)
    sel = lambda k: np.asarray(c[k])[idx]
    g = ctx.find_epipolar_match_direct([fr], [c["T_ref_w"]], fc, T_cur_w, c["cam"], np.zeros(len(idx), np.int32), sel("ftr_px"),
                                       sel("ftr_f"), sel("ftr_level"), sel("ftr_type"), sel("ftr_grad"), d[0], d[1], d[2], **kw)
    fr.destroy(); fc.destroy()
    os_ = [oracle.find_epipolar_match_direct(c["ref_pyr"], cur_pyr, c["cam"], T_cur_ref, c["ftr_px"][i], c["ftr_f"][i],
                                             int(c["ftr_level"][i]), int(c["ftr_type"][i]), c["ftr_grad"][i], d[0][j], d[1][j],
                                             d[2][j], kw.get("max_search_level", 2), kw.get("align_max_iter", 10),
                                             kw.get("max_epi_search_steps", 1000)) for j, i in enumerate(idx)]
    for j, o in enumerate(os_):
        assert g["success"][j] == o["success"] and g["reject"][j] == o["reject"], j
        assert g["search_level"][j] == o["search_level"] and g["n_zmssd"][j] == o["n_zmssd"], j
        assert np.isclose(g["epi_length"][j], o["epi_length"], rtol=1e-9, atol=1e-12), j
        assert np.allclose(g["A_cur_ref"][j], o["A_cur_ref"], rtol=1e-9, atol=1e-12), j
        # px_cur: the refined match, or the scan's start when the refinement failed, or (0, 0) when nothing started
        assert np.allclose(g["px_cur"][j], o["px_cur"], rtol=0, atol=1e-6), (j, g["px_cur"][j], o["px_cur"])
        if o["success"]:
            assert np.isclose(g["depth"][j], o["depth"], rtol=1e-6), j
    return g, os_


def _ranges(c, idx, rel):
    """Depth ranges around each candidate's true depth: d_min / d_max = depth / (1 +- rel)."""
    d = c["depth_gt"][idx]
    return d, d / (1 + rel), d / np.maximum(1 - rel, 1e-3)


def test_epipolar_match_every_branch(ctx, oracle):
    c = synth.make_depth_case(22, n_seeds=300, baseline=0.3)
    rng = np.random.default_rng(8)
    M = c["M"]
    c["ftr_type"] = (rng.uniform(size=M) < 0.4).astype(np.int32)
    c["ftr_grad"][::17] = 0.0                       # edgelets without a gradient: the angle test sees NaN and passes
    c["ftr_type"][::17] = 1
    branches = dict(reject=0, zero_gradient=0, short=0, level0=0, level1=0, level2=0, no_score=0, triangulation=0,
                    at_limit=0, over_limit=0)
    # (1) ordinary ranges (scan at the candidate's search level) and tight ranges (epipolar segment < 2 px)
    idx = np.arange(M)
    for rel in (0.3, 2e-4):
        g, os_ = _match_both(ctx, oracle, c, c["cur_pyr"], c["T_cur_w"], idx, _ranges(c, idx, rel))
        for j, o in enumerate(os_):
            if o["reject"]:
                branches["reject"] += 1
            elif c["ftr_type"][j] == 1 and not c["ftr_grad"][j].any():
                branches["zero_gradient"] += 1
            if not o["reject"] and o["epi_length"] < 2:
                branches["short"] += 1
            if o["n_zmssd"] > 0:
                branches[f"level{o['search_level']}"] += 1
    # (2) no ZMSSD under the threshold: the current image is noise, every score is ~64 * (var(ref) + var(noise))
    noise = np.random.default_rng(9).integers(0, 256, c["cur_pyr"][0].shape, dtype=np.uint8)
    noise_pyr = synth.build_pyramid(noise, len(c["cur_pyr"]))
    idx = np.flatnonzero(c["ftr_type"] == 0)[:60]
    g, os_ = _match_both(ctx, oracle, c, noise_pyr, c["T_cur_w"], idx, _ranges(c, idx, 0.3))
    for o in os_:
        if o["n_zmssd"] > 0 and not o["success"] and not np.any(o["px_cur"]):
            branches["no_score"] += 1
    # (3) triangulation failure: a current frame rotated but not moved; the segment collapses (< 2 px), the alignment
    # converges, and the two bearings are parallel (depthFromTriangulation's determinant < 1e-6)
    T_rot = synth.se3_mul(synth.se3_exp(np.array([0, 0, 0, 0.004, -0.003, 0.002])), c["T_ref_w"])
    rot_pyr = synth.build_pyramid(synth.render(c["cam"], T_rot, c["plane"], synth.make_texture(7)), len(c["cur_pyr"]))
    idx = np.flatnonzero(c["ftr_type"] == 0)[:60]
    g, os_ = _match_both(ctx, oracle, c, rot_pyr, T_rot, idx, _ranges(c, idx, 0.3))
    T_cur_ref = synth.se3_mul(T_rot, synth.se3_inv(c["T_ref_w"]))
    for j, o in enumerate(os_):
        i = idx[j]
        mid = np.mean([c["cam"].world2cam(T_cur_ref[:, :3] @ (c["ftr_f"][i] * dd) + T_cur_ref[:, 3]) for dd in _ranges(c, [i], 0.3)[1:]], axis=0)
        if not o["success"] and o["epi_length"] < 2 and np.linalg.norm(o["px_cur"] - mid.ravel()) > 1e-9:
            branches["triangulation"] += 1  # the refinement moved px_cur, yet no depth came out
    # (4) the step limit at its edge: n0 = floor(epi_length / 0.7) steps are allowed at max_epi_search_steps = n0, not at n0 - 1
    idx = np.flatnonzero(c["ftr_type"] == 0)[:16]
    d = _ranges(c, idx, 0.3)
    _, os_ = _match_both(ctx, oracle, c, c["cur_pyr"], c["T_cur_w"], idx, d)
    for j, o in enumerate(os_):
        n0 = int(o["epi_length"] / 0.7)
        if o["epi_length"] < 2 or n0 < 2 or o["n_zmssd"] == 0:  # only segments whose scan scores something
            continue
        one = [idx[j]]
        dj = tuple(x[j:j + 1] for x in d)
        _, (oa,) = _match_both(ctx, oracle, c, c["cur_pyr"], c["T_cur_w"], one, dj, max_epi_search_steps=n0)
        _, (ob,) = _match_both(ctx, oracle, c, c["cur_pyr"], c["T_cur_w"], one, dj, max_epi_search_steps=n0 - 1)
        assert oa["n_zmssd"] == o["n_zmssd"] and ob["n_zmssd"] == 0 and not ob["success"], j
        branches["at_limit"] += 1
        branches["over_limit"] += 1
    print("epipolar scan branches:", branches)
    for k, v in branches.items():
        assert v > 0, k


def test_epipolar_match_equal_scores_pick_the_first_step(ctx, oracle):
    """A low-contrast reference patch scanned across a constant current image: every 8x8 block the scan scores is the same
    array, so every ZMSSD is the same number (64 * var(patch), under the 2000 * 64 threshold).  The reference keeps the first
    strict minimum in step order; the start of the refinement (px_cur when it fails) shows which one won."""
    c = synth.make_depth_case(24, n_seeds=100, baseline=0.3)
    tex = synth.make_texture(7)
    low = (128 + (tex.astype(np.int32) - 128) // 6).astype(np.uint8)
    c["ref_pyr"] = synth.build_pyramid(synth.render(c["cam"], c["T_ref_w"], c["plane"], low), len(c["ref_pyr"]))
    flat = [np.full_like(im, 100) for im in c["cur_pyr"]]
    assert all(np.ptp(im) == 0 for im in flat)  # every block scored along any line is identical: a tie everywhere
    c["ftr_type"][:] = 0
    idx = np.arange(c["M"])
    g, os_ = _match_both(ctx, oracle, c, flat, c["T_cur_w"], idx, _ranges(c, idx, 0.3))
    ties = sum(1 for o in os_ if o["n_zmssd"] >= 2 and np.any(o["px_cur"]))
    print("equal-score scans:", ties)
    assert ties > 20
