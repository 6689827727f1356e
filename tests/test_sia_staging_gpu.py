"""GPU: the staging of the alignment batch (svo_b200_sia_batch_stage / _run / _fetch) and of the single-pair calls built on it.

The batch stages through a pinned / device buffer pair of its own, so any other entry point of the context may run between
its stage, run and fetch without changing a bit of what it fetches, and a fetch may be repeated.  svo_b200_sparse_img_align
and svo_b200_sparse_residuals add their trace or residual-pass regions to the batch's staging, leave nothing staged behind,
and copy back to the caller no more than the rows and trace entries it asked for.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from rpg_svo_b200 import capi, synth
from tests import klt_cases as kc
from tests import sia_cases as sc
from tests import sia_robust_cases as rc

pytestmark = pytest.mark.gpu

W, H, NFEAT, NLEVELS = 640, 480, 300, 5


@pytest.fixture(scope="module")
def gctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def others(gctx):
    """One call each of four other entry points of the context, each of which stages through the context's own buffers."""
    ctx = gctx
    po = [synth.make_pose_opt_case(s, n=600) for s in (3, 4)]
    po_off = np.array([0, 600, 1200], np.int32)
    cat = lambda k: np.concatenate([c[k] for c in po])  # noqa: E731
    dc = synth.make_depth_case(5, n_seeds=400)
    ref, cur = ctx.frame(dc["ref_pyr"]), ctx.frame(dc["cur_pyr"])
    k = kc.case("shift_640")
    fp, fc = ctx.frame_from_level0(k["prev"], 1), ctx.frame_from_level0(k["cur"], 1)
    pp, pc = ctx.klt_pyramid(fp, True), ctx.klt_pyramid(fc, False)

    def call():
        ctx.pose_optimize_batch(2.0, 10, [c["cam"].fx for c in po], np.stack([c["T_init"] for c in po]), po_off, cat("f"),
                                cat("pos"), cat("level"), cat("has_point"))
        ctx.depth_filter_update([ref], [dc["T_ref_w"]], cur, dc["T_cur_w"], dc["cam"], dc["ref_index"], dc["ftr_px"],
                                dc["ftr_f"], dc["ftr_level"], dc["ftr_type"], dc["ftr_grad"], dc["batch_id"],
                                dc["batch_counter"], dc["seeds"])
        ctx.fast_detect(ref, 30, 3, 20.0)
        ctx.klt_track(pp, pc, k["prev_pts"], k["next_pts"], k["max_level"], k["max_iter"], k["eps"])

    yield call
    for x in (pp, pc):
        x.destroy()
    for x in (fp, fc, ref, cur):
        x.destroy()


def _batch(ctx, B):
    st = synth.make_stream_fast(21, B + 1, W, H, NFEAT, NLEVELS, device="cuda")
    cat = lambda k: np.concatenate([st["feats"][b][k] for b in range(B)])  # noqa: E731
    pool = capi.FramePool(ctx, W, H, NLEVELS, B + 1)
    pool.upload_array(st["level0"].numpy())
    args = (pool.frames[:B], pool.frames[1:B + 1], st["cam"], np.tile(synth.se3_identity()[None], (B, 1, 1)),
            np.arange(B + 1, dtype=np.int32) * NFEAT, cat("px"), cat("f"), cat("pos"), cat("has_point"),
            np.stack([synth.se3_inv(st["poses"][b])[:, 3] for b in range(B)]), NLEVELS - 1, 0)
    return pool, args


def _fetch(ctx, B, weighted):
    r = ctx.sia_batch_fetch(want_H=True)
    if weighted:
        r["scales"] = ctx.sia_last_scales(B)
    return r


def _assert_same(a, b):
    for k in ("T", "H", "visible"):
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
    assert np.array_equal(a["stats"], b["stats"])
    if "scales" in b:
        assert rc.same_bits(a["scales"], b["scales"])


BATCHES = ["cluster-32", "throughput", "tukey-8"]


@pytest.mark.parametrize("kind", BATCHES)
def test_other_entry_points_between_stage_run_and_fetch(gctx, others, kind):
    """A batch with pose optimizer, depth filter, detector and KLT calls between its stage and run and between its run and
    fetch fetches, twice, bit for bit what the same batch fetches without them."""
    ctx = gctx
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    B = {"cluster-32": 32, "throughput": 3 * sm, "tukey-8": 8}[kind]
    weighted = kind.startswith("tukey")
    pool, args = _batch(ctx, B)
    try:
        if weighted:
            ctx.sia_robust(capi.SCALE_MAD, capi.WEIGHT_TUKEY)
        ctx.sia_batch_stage(*args)
        ctx.sia_batch_run()
        alone = _fetch(ctx, B, weighted)
        L = ctx.sia_last_launch()
        geo = {"cluster-32": L["ctas_per_pair"] > 1, "throughput": (L["threads"], L["features_per_thread"]) == (160, 2),
               "tukey-8": L["threads"] == 256}[kind]
        assert geo and L["n_pairs"] == B, L
        assert alone["stats"]["n_iters"].min() > 0
        ctx.sia_batch_stage(*args)
        others()
        ctx.sia_batch_run()
        others()
        first = _fetch(ctx, B, weighted)
        second = _fetch(ctx, B, weighted)
        _assert_same(first, alone)
        _assert_same(second, alone)
    finally:
        ctx.sia_robust(capi.SCALE_UNIT, capi.WEIGHT_UNIT)
        pool.destroy()


def _residual_case():
    d = sc.border_pair(5, W, H, NFEAT)
    return d, d["T_gt"], 2


def test_single_pair_calls_leave_nothing_staged(gctx):
    ctx = gctx
    d, T, level = _residual_case()
    ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
    args = (d["px"], d["f"], d["pos"], d["has_point"], d["ref_pos"])
    for call in (lambda: ctx.sparse_img_align(ref, cur, d["cam"], synth.se3_identity(), *args, NLEVELS - 1, 0, want_trace=True),
                 lambda: ctx.sparse_residuals(ref, cur, d["cam"], level, T, *args)):
        call()
        n = ctx.launch_count()
        with pytest.raises(capi.SvoB200Error, match="nothing staged"):
            ctx.sia_batch_run()
        with pytest.raises(capi.SvoB200Error, match="nothing staged"):
            ctx._check(ctx.lib.svo_b200_sia_batch_fetch(ctx.h, None, None, None, None))
        assert ctx.launch_count() == n
    ref.destroy(); cur.destroy()


def _align_raw(ctx, d, ref, cur, cap, extra):
    """svo_b200_sparse_img_align through the raw ABI with a trace array of cap + extra entries, the extra ones 0xa5 bytes:
    (T, trace bytes, n_trace)."""
    N = len(d["px"])
    T = synth.se3_identity().reshape(12).copy()
    px, f, pos, rpos = capi.c64(d["px"]), capi.c64(d["f"]), capi.c64(d["pos"]), capi.c64(d["ref_pos"])
    hp = np.ascontiguousarray(d["has_point"], np.uint8)
    trace = (capi.SiaIter * (cap + extra))()
    C.memset(trace, 0xA5, C.sizeof(trace))
    ntr = C.c_int(-1)
    cs, opt = capi.cam_struct(d["cam"]), capi.SiaOptions(NLEVELS - 1, 0, 30, 1e-6)
    vis, Hm, stats = np.zeros(N, np.uint8), np.zeros(36), capi.SiaStats()
    ctx._check(ctx.lib.svo_b200_sparse_img_align(
        ctx.h, ref.h, cur.h, C.byref(cs), C.byref(opt), capi._p(T), capi._p(px), capi._p(f), capi._p(pos), capi._p(hp),
        capi._p(rpos), N, capi._p(vis), capi._p(Hm), C.byref(stats), trace, cap, C.byref(ntr)))
    return T, bytes(trace), ntr.value


def test_trace_copy_back_stops_at_trace_cap(gctx):
    """With trace_cap below the iterations run, n_trace reports them all, the first trace_cap entries are those of a full
    trace and the caller's entry past trace_cap is untouched."""
    ctx = gctx
    d = sc.subset(sc.base_pair(), NFEAT)
    ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
    sz = C.sizeof(capi.SiaIter)
    T_full, full, n_full = _align_raw(ctx, d, ref, cur, NLEVELS * 30 + 8, 0)
    cap = 3
    assert n_full > cap
    T, tr, n = _align_raw(ctx, d, ref, cur, cap, 1)
    assert n == n_full
    assert tr[:cap * sz] == full[:cap * sz]
    assert tr[cap * sz:] == b"\xa5" * sz
    assert np.array_equal(T.view(np.uint64), T_full.view(np.uint64))
    ref.destroy(); cur.destroy()


OPTIONAL = ("ref_patch", "residuals", "in_image", "H", "Jres", "chi2", "n_meas")


def _residuals_raw(ctx, d, ref, cur, level, T, null=None):
    """svo_b200_sparse_residuals through the raw ABI with row arrays one row longer than N, the last row 0xa5 bytes, and
    the optional output `null` passed as NULL."""
    N = len(d["px"])
    o = dict(visible=np.zeros(N + 1, np.uint8), ref_patch=np.zeros((N + 1, 16), np.float32),
             residuals=np.zeros((N + 1, 16), np.float32), in_image=np.zeros(N + 1, np.uint8), H=np.zeros(36),
             Jres=np.zeros(6), chi2=np.zeros(1), n_meas=np.zeros(1, np.int64))
    for k in ("visible", "ref_patch", "residuals", "in_image"):
        o[k][N:].view(np.uint8)[...] = 0xA5
    cs = capi.cam_struct(d["cam"])
    Tp, px, f, pos, rpos = (capi.c64(x) for x in (np.asarray(T).reshape(12), d["px"], d["f"], d["pos"], d["ref_pos"]))
    hp = np.ascontiguousarray(d["has_point"], np.uint8)
    ptr = {k: None if k == null else capi._p(o[k]) for k in OPTIONAL}
    ctx._check(ctx.lib.svo_b200_sparse_residuals(
        ctx.h, ref.h, cur.h, C.byref(cs), level, capi._p(Tp), capi._p(px), capi._p(f), capi._p(pos), capi._p(hp),
        capi._p(rpos), N, capi._p(o["visible"]), *[ptr[k] for k in OPTIONAL]))
    return o


def test_residual_pass_copy_back_stays_inside_n_rows(gctx):
    """The residual pass writes the caller's first N rows, as the binding's call returns them, and never row N; each
    optional output may be NULL without changing the others."""
    ctx = gctx
    d, T, level = _residual_case()
    N = len(d["px"])
    ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
    g = ctx.sparse_residuals(ref, cur, d["cam"], level, T, d["px"], d["f"], d["pos"], d["has_point"], d["ref_pos"])
    v = g["visible"].astype(bool)
    assert 0 < v.sum() < N and 0 < g["in_image"].sum()
    for null in (None,) + OPTIONAL:
        o = _residuals_raw(ctx, d, ref, cur, level, T, null)
        for k in ("visible", "ref_patch", "residuals", "in_image"):
            assert np.all(o[k][N:].view(np.uint8) == 0xA5), (null, k)
        assert np.array_equal(o["visible"][:N], g["visible"]), null
        # the patch rows of invisible features are whatever the kernel's shared memory held (test_sia_gpu.py)
        if null != "ref_patch":
            assert np.array_equal(o["ref_patch"][:N][v].view(np.uint32), g["ref_patch"][v].view(np.uint32)), null
        if null != "residuals":
            assert np.array_equal(o["residuals"][:N].view(np.uint32), g["residuals"].view(np.uint32)), null
        if null != "in_image":
            assert np.array_equal(o["in_image"][:N], g["in_image"]), null
        if null != "H":
            assert np.array_equal(o["H"].view(np.uint64), g["H"].reshape(36).view(np.uint64)), null
        if null != "Jres":
            assert np.array_equal(o["Jres"].view(np.uint64), g["Jres"].view(np.uint64)), null
        if null != "chi2":
            assert o["chi2"][0] == g["chi2"], null
        if null != "n_meas":
            assert o["n_meas"][0] == g["n_meas"], null
    ref.destroy(); cur.destroy()
