"""GPU: align_batch_kernel (feature_alignment::align2D / align1D) and find_match_direct_kernel (Matcher::findMatchDirect) at
their border, degenerate, multi-reference and batch edges (cases in tests/align_cases.py), against the oracle bit for bit,
the compiled reference's recorded outputs (test_align_pins.py) and a float64 numpy statement of the warp; plus the ABI's
argument checks."""
import ctypes as C
from collections import Counter

import numpy as np
import pytest

from rpg_svo_b200 import capi
from tests import align_cases as ac
from tests.ref_golden import RefCalls
from tests.test_align_pins import ALIGN_NAMES, KNOWN_ALIGN_DIFFS, MATCH_NAMES, align_diffs

pytestmark = pytest.mark.gpu
EINVAL = -1


@pytest.fixture(scope="module")
def pool(ctx):
    imgs, _ = ac.pool_case()
    p = capi.FramePool(ctx, 640, 480, 5, len(imgs))
    p.upload_array(imgs)
    yield p
    p.destroy()


def _kernel_align(ctx, c, frame):
    conv2, px2 = ctx.align2d_batch(frame, c["level"], c["pwb"], c["patch"], c["n_iter"], c["px"])
    conv1, px1, h1 = ctx.align1d_batch(frame, c["level"], c["dir"], c["pwb"], c["patch"], c["n_iter"], c["px"])
    return conv2, px2, conv1, px1, h1


def _assert_equals_oracle(g, o, name):
    conv2, px2, conv1, px1, h1 = g
    assert np.array_equal(conv2, o["conv2"]), name
    assert ac.same_bits(px2, o["px2"]), name
    assert np.array_equal(conv1, o["conv1"]), name
    assert ac.same_bits(px1, o["px1"]), name
    assert ac.same_bits(h1, o["h1"]), name  # +inf included


@pytest.mark.parametrize("name", ALIGN_NAMES)
def test_align_case_bit_exact(ctx, oracle, pool, name):
    """px as bits (NaN = NaN), converged and h_inv against the oracle and the recorded reference.  The FramePool cases run
    on the pool's first and last frame, whose device-built pyramids must equal the host pyramids."""
    c = next(x for x in ac.align_cases() if x["name"] == name)
    if "pool_index" in c:
        frame = pool.frames[c["pool_index"]]
        for L in range(5):
            assert np.array_equal(frame.download_level(L), c["pyr"][L]), L
    else:
        frame = ctx.frame(c["pyr"])
    g = _kernel_align(ctx, c, frame)
    o = ac.run_oracle_align(oracle, c)
    _assert_equals_oracle(g, o, name)
    ref = RefCalls("test_align_pins", f"test_align_case_oracle_equals_reference[{name}]")
    r = ac.run_ref_align(ref, c)
    ref.finish()
    assert align_diffs(c, o, r) == {k for k in KNOWN_ALIGN_DIFFS if k[0] == name}
    if "pool_index" not in c:
        frame.destroy()


@pytest.mark.parametrize("M", list(ac.BATCH_SIZES) + [ac.BIG_BATCH])
def test_align_batch_shapes_equal_single_calls(ctx, oracle, M):
    """Every problem of one launch (levels mixed) equals the same problem launched alone, bit for bit; a sample covering
    the first and the last CTA equals the oracle (and, for the big batch, the recorded reference)."""
    c = ac.batch_problems(M)
    fr = ctx.frame(c["pyr"])
    g = _kernel_align(ctx, c, fr)
    single = [[], [], [], [], []]
    for i in range(M):
        s = ctx.align2d_batch(fr, c["level"][i:i + 1], c["pwb"][i:i + 1], c["patch"][i:i + 1], 10, c["px"][i:i + 1])
        s1 = ctx.align1d_batch(fr, c["level"][i:i + 1], c["dir"][i:i + 1], c["pwb"][i:i + 1], c["patch"][i:i + 1], 10,
                               c["px"][i:i + 1])
        for k, x in enumerate(s + s1):
            single[k].append(x[0])
    for k in range(5):
        assert np.array_equal(ac.bits(np.array(single[k], np.float64)), ac.bits(np.asarray(g[k], np.float64))), k  # NaNs too
    rows = ac.sample_rows(M)
    o = ac.run_oracle_align(oracle, c, rows)
    _assert_equals_oracle(tuple(x[rows] for x in g), o, M)
    if M == ac.BIG_BATCH:
        ref = RefCalls("test_align_pins", "test_align_big_batch_sample_oracle_equals_reference")
        assert not align_diffs(c, o, ac.run_ref_align(ref, c, rows))
        ref.finish()
    assert M < 4097 or np.unique(c["level"]).size == 5
    fr.destroy()


def test_align_exit_reasons_cover_every_branch(oracle):
    """How each run of the cases above ended (the oracle's exit reason; the kernels equal the oracle bit for bit on every
    one): both border breaks, convergence and the iteration limit in 2-D and 1-D, and the rollback in 1-D.  The NaN return
    after the border test is unreachable."""
    counts = {"2d": Counter(), "1d": Counter()}
    for c in ac.align_cases() + [ac.batch_problems(4097)]:
        o = ac.run_oracle_align(oracle, c)
        counts["2d"].update(o["exit2"].tolist())
        counts["1d"].update(o["exit1"].tolist())
    reasons = ("border_first", "border", "converged", "max_iter", "rollback", "nan")
    print("\nexit reason     2-D    1-D")
    for k in reasons:
        print(f"{k:<14} {counts['2d'][k]:>5} {counts['1d'][k]:>6}")
    for k in reasons[:4]:
        assert counts["2d"][k] > 0 and counts["1d"][k] > 0, k
    assert counts["1d"]["rollback"] > 0 and counts["2d"]["rollback"] == 0
    assert counts["2d"]["nan"] == counts["1d"]["nan"] == 0


# ---- find_match_direct ------------------------------------------------------------------------------------------------------
def _kernel_match(ctx, c, frames, cur, idx=None, ref_index=None):
    idx = np.arange(c["M"]) if idx is None else idx
    sel = lambda k: np.asarray(c[k])[idx]
    ri = sel("ref_index") if ref_index is None else ref_index
    return ctx.find_match_direct(frames, c["ref_T"] if ref_index is None else [c["ref_T"][int(c["ref_index"][idx[0]])]], cur,
                                 c["T_cur_w"], c["cam"], ri, sel("ref_px"), sel("ref_f"), sel("ref_level"), sel("ftr_type"),
                                 sel("ref_grad"), sel("point_pos"), sel("px_cur"), max_search_level=int(c["max_search_level"]),
                                 align_max_iter=int(c["align_max_iter"]))


def _check_vs_oracle(oracle, c, g, o, stats):
    name = c["name"]
    assert np.array_equal(g["success"], o["success"]), name
    assert np.array_equal(g["search_level"], o["search_level"]), name
    assert np.allclose(g["A_cur_ref"], o["A_cur_ref"], rtol=1e-9, atol=1e-12, equal_nan=True), name
    either = g["success"] | o["success"]
    assert np.max(np.abs(g["px_cur"][either] - o["px_cur"][either]), initial=0.0) <= 1e-4, name
    assert np.array_equal(np.isnan(g["px_cur"]), np.isnan(o["px_cur"])), name
    for i in range(c["M"]):
        if ac.in_frame(c, i):
            A, s = ac.numpy_warp(c, i)
            assert np.allclose(g["A_cur_ref"][i], A, rtol=1e-9, atol=1e-12), (name, i)
            assert g["search_level"][i] == s, (name, i)
        else:
            assert not g["A_cur_ref"][i].any() and g["search_level"][i] == 0 and not g["success"][i], (name, i)
    # h_inv of edgelets: equal unless an f64 rounding difference in A flips a uint8 truncation of a warped sample
    for i in np.flatnonzero((np.asarray(c["ftr_type"]) == 1) & np.array([ac.in_frame(c, i) for i in range(c["M"])])):
        stats["edgelets"] += 1
        if ac.same_bits(g["h_inv"][i], o["h_inv"][i]):
            stats["h_inv_identical"] += 1
            continue
        r, L = int(c["ref_index"][i]), int(c["ref_level"][i])
        img = c["ref_pyrs"][r][L]
        sl = int(o["search_level"][i])
        pg = oracle.warp_affine(g["A_cur_ref"][i], img, c["ref_px"][i], L, sl, 5)[1]
        po = oracle.warp_affine(o["A_cur_ref"][i], img, c["ref_px"][i], L, sl, 5)[1]
        assert not np.array_equal(pg, po), (name, i, g["h_inv"][i], o["h_inv"][i])


def _check_vs_ref(g, r, c):
    seen = ac.close_view(c)
    assert not r["success"][~seen].any()
    g, r = ({k: v[seen] for k, v in x.items()} for x in (g, r))
    assert np.array_equal(g["success"], r["success"])
    assert np.array_equal(g["search_level"], r["search_level"])
    assert np.allclose(g["A_cur_ref"], r["A_cur_ref"], rtol=1e-9, atol=1e-12, equal_nan=True)
    either = g["success"] | r["success"]
    assert np.max(np.abs(g["px_cur"][either] - r["px_cur"][either]), initial=0.0) <= 1e-4


H_INV_STATS = Counter()


@pytest.mark.parametrize("name", [c["name"] for c in ac.match_cases()])
def test_match_case_vs_oracle_numpy_and_reference(ctx, oracle, name):
    c = next(x for x in ac.match_cases() if x["name"] == name)
    frames, cur = [ctx.frame(p) for p in c["ref_pyrs"]], ctx.frame(c["cur_pyr"])
    g = _kernel_match(ctx, c, frames, cur)
    o = ac.run_oracle_match(oracle, c)
    _check_vs_oracle(oracle, c, g, o, H_INV_STATS)
    if name in MATCH_NAMES:
        ref = RefCalls("test_align_pins", f"test_match_case_oracle_equals_reference[{name}]")
        _check_vs_ref(g, ac.run_ref_match(ref, c), c)
        ref.finish()
    print(f"{name}: {int(g['success'].sum())}/{c['M']} matched; edgelet h_inv bit-identical so far "
          f"{H_INV_STATS['h_inv_identical']}/{H_INV_STATS['edgelets']}")
    for f in frames + [cur]:
        f.destroy()


def test_match_cases_reach_every_search_level_and_zero_fill(ctx, oracle):
    """Search levels 0-4 all occur (the cap binds for the 8x closer camera), a negative cap acts as 0, and the 180 degree
    roll case puts warp samples exactly on cols - 1 and rows - 1."""
    levels = set()
    for c in ac.search_level_cases():
        o = ac.run_oracle_match(oracle, c)
        levels |= set(o["search_level"].tolist())
        if c["max_search_level"] < 0:
            assert not o["search_level"].any()
        if "k8" in c["name"] and c["max_search_level"] in (1, 2):
            assert np.all(o["search_level"][[ac.in_frame(c, i) for i in range(c["M"])]] == c["max_search_level"])
    assert levels == {0, 1, 2, 3, 4}
    c = ac.warp_border_cases()[1]
    o = ac.run_oracle_match(oracle, c)
    f32 = np.float32
    hits = Counter()
    for i in range(c["M"]):  # the kernel's sample positions (warp_warp_affine), in float32 as it computes them
        a = o["A_cur_ref"][i].ravel()
        invdet = 1.0 / (a[0] * a[3] - a[2] * a[1])
        A00, A01, A10, A11 = f32(a[3] * invdet), f32(-a[1] * invdet), f32(-a[2] * invdet), f32(a[0] * invdet)
        sc = f32(1 << int(o["search_level"][i]))
        prx, pry = f32(c["ref_px"][i][0]), f32(c["ref_px"][i][1])
        for y in range(10):
            for x in range(10):
                ppx, ppy = f32(x - 5) * sc, f32(y - 5) * sc
                qx = f32(f32(float(A00) * float(ppx) + float(f32(A01 * ppy))) + prx)
                qy = f32(f32(float(A10) * float(ppx) + float(f32(A11 * ppy))) + pry)
                hits["cols-1"] += qx == 639
                hits["rows-1"] += qy == 479
                hits["outside"] += bool(qx < 0 or qy < 0 or qx >= 639 or qy >= 479)
    print("warp samples of the 180 degree roll case:", dict(hits))
    assert hits["cols-1"] > 0 and hits["rows-1"] > 0 and hits["outside"] > hits["cols-1"] + hits["rows-1"]


@pytest.mark.parametrize("n_ref", [3, 4])
def test_match_multi_ref_equals_single_frame_calls(ctx, oracle, n_ref):
    """Candidates of every reference frame (different poses, images and pyramid depths) in one launch, ref_index
    interleaved and unsorted: each equals a launch with its own frame alone (n_ref = 1) bit for bit, and the oracle."""
    c = ac.multi_ref_case(n_ref)
    frames, cur = [ctx.frame(p) for p in c["ref_pyrs"]], ctx.frame(c["cur_pyr"])
    g = _kernel_match(ctx, c, frames, cur)
    assert len(set(c["ref_index"][:8].tolist())) > 1 and not np.all(np.diff(c["ref_index"]) >= 0)
    for r in range(n_ref):
        idx = np.flatnonzero(c["ref_index"] == r)
        s = _kernel_match(ctx, c, [frames[r]], cur, idx, ref_index=np.zeros(len(idx), np.int32))
        for k in ("success", "search_level"):
            assert np.array_equal(g[k][idx], s[k]), (r, k)
        for k in ("px_cur", "A_cur_ref", "h_inv"):
            assert np.array_equal(ac.bits(g[k][idx]), ac.bits(s[k])), (r, k)
    _check_vs_oracle(oracle, c, g, ac.run_oracle_match(oracle, c), Counter())
    ref = RefCalls("test_align_pins", f"test_match_multi_ref_oracle_equals_reference[{n_ref}]")
    _check_vs_ref(g, ac.run_ref_match(ref, c), c)
    ref.finish()
    assert g["success"].sum() > 0.25 * c["M"]
    for f in frames + [cur]:
        f.destroy()


def test_h_inv_bit_identical_fraction():
    """Report of the edgelet h_inv comparison above (runs after the matcher cases)."""
    n, same = H_INV_STATS["edgelets"], H_INV_STATS["h_inv_identical"]
    print(f"\nedgelet h_inv bit-identical to the oracle: {same}/{n}" + (f" ({same / n:.4%})" if n else ""))


# ---- ABI: argument checks and optional outputs ------------------------------------------------------------------------------
def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class _Match:
    """Raw ctypes arguments of svo_b200_find_match_direct for a few candidates of one case."""

    def __init__(self, ctx, c, n=4):
        self.c, self.n = c, n
        self.frames = [ctx.frame(p) for p in c["ref_pyrs"]]
        self.cur = ctx.frame(c["cur_pyr"])
        g = lambda k, t: np.ascontiguousarray(np.asarray(c[k])[:n], t)
        self.ri, self.px, self.f = g("ref_index", np.int32), g("ref_px", np.float64), g("ref_f", np.float64)
        self.lv, self.ty, self.gr = g("ref_level", np.int32), g("ftr_type", np.int32), g("ref_grad", np.float64)
        self.pos, self.pc = g("point_pos", np.float64), g("px_cur", np.float64)
        self.refT = np.ascontiguousarray(np.asarray(c["ref_T"]).reshape(-1))
        self.curT = np.ascontiguousarray(np.asarray(c["T_cur_w"]).reshape(-1))
        self.cam = capi.cam_struct(c["cam"])

    def call(self, ctx, frames=None, n_ref=None, M=None, ri=None, lv=None, max_level=2, outs=True):
        frames = self.frames if frames is None else frames
        arr = (C.c_void_p * max(len(frames), 1))(*[None if f is None else f.h.value for f in frames])
        opt = capi.MatchOptions(max_level, 10)
        M = self.n if M is None else M
        px = self.pc.copy()
        succ = np.zeros(self.n, np.uint8)
        sl, A, h = np.zeros(self.n, np.int32), np.zeros((self.n, 4)), np.zeros(self.n)
        rc = ctx.lib.svo_b200_find_match_direct(
            ctx.h, arr, _p(self.refT), len(frames) if n_ref is None else n_ref, self.cur.h, _p(self.curT), C.byref(self.cam),
            C.byref(opt), M, _p(self.ri if ri is None else ri), _p(self.px), _p(self.f), _p(self.lv if lv is None else lv),
            _p(self.ty), _p(self.gr), _p(self.pos), _p(px), _p(succ), _p(sl) if outs else None, _p(A) if outs else None,
            _p(h) if outs else None)
        return rc, dict(px_cur=px, success=succ, search_level=sl, A=A, h_inv=h)

    def destroy(self):
        for f in self.frames + [self.cur]:
            f.destroy()


def _still_usable(ctx, fr):
    c = ac.batch_problems(5)
    a = ctx.align2d_batch(fr, c["level"], c["pwb"], c["patch"], 10, c["px"])
    b = ctx.align2d_batch(fr, c["level"], c["pwb"], c["patch"], 10, c["px"])
    assert np.array_equal(a[0], b[0]) and np.array_equal(ac.bits(a[1]), ac.bits(b[1]))


def test_abi_rejects_bad_arguments_and_stays_usable(ctx):
    c = ac.batch_problems(5)
    fr = ctx.frame(c["pyr"])
    L = ctx.lib
    px, conv, h = c["px"].copy(), np.zeros(5, np.uint8), np.zeros(5)
    d = np.ascontiguousarray(c["dir"])
    for bad in (-1, 5):  # level outside the pyramid
        lv = c["level"].copy()
        lv[3] = bad
        assert L.svo_b200_align2d_batch(ctx.h, fr.h, 5, _p(lv), _p(c["pwb"]), _p(c["patch"]), 10, _p(px), _p(conv)) == EINVAL
        assert L.svo_b200_align1d_batch(ctx.h, fr.h, 5, _p(lv), _p(d), _p(c["pwb"]), _p(c["patch"]), 10, _p(px), _p(conv),
                                        _p(h)) == EINVAL
        _still_usable(ctx, fr)
    assert L.svo_b200_align2d_batch(ctx.h, fr.h, -1, _p(c["level"]), _p(c["pwb"]), _p(c["patch"]), 10, _p(px), _p(conv)) == EINVAL
    assert L.svo_b200_align1d_batch(ctx.h, fr.h, 5, _p(c["level"]), None, _p(c["pwb"]), _p(c["patch"]), 10, _p(px), _p(conv),
                                    _p(h)) == EINVAL
    assert np.array_equal(px, c["px"])  # nothing written on a rejected call
    _still_usable(ctx, fr)
    m = _Match(ctx, ac.multi_ref_case(3))
    for bad in (-1, 3):  # ref_index outside [0, n_ref)
        ri = m.ri.copy()
        ri[1] = bad
        assert m.call(ctx, ri=ri)[0] == EINVAL
        _still_usable(ctx, fr)
    shallow = int(np.argmin([len(p) for p in m.c["ref_pyrs"]]))
    ri, lv = m.ri.copy(), m.lv.copy()
    ri[0], lv[0] = shallow, len(m.c["ref_pyrs"][shallow])  # ref_level == that frame's n_levels
    assert m.call(ctx, ri=ri, lv=lv)[0] == EINVAL
    assert m.call(ctx, max_level=5)[0] == EINVAL  # max_search_level == the current frame's n_levels
    assert m.call(ctx, frames=[m.frames[0], None, m.frames[2]])[0] == EINVAL  # a NULL reference frame
    assert m.call(ctx, frames=[None, None, None], ri=np.zeros(4, np.int32))[0] == EINVAL
    assert m.call(ctx, M=-1)[0] == EINVAL
    _still_usable(ctx, fr)
    rc, out = m.call(ctx)
    assert rc == 0 and out["success"].any()
    m.destroy()
    fr.destroy()


def test_abi_empty_match_batch_without_reference_frames(ctx):
    """M == 0 is a no-op whatever n_ref is, as align_batch's M == 0."""
    m = _Match(ctx, ac.multi_ref_case(3))
    assert m.call(ctx, frames=[], n_ref=0, M=0)[0] == 0
    assert m.call(ctx, frames=[None], n_ref=1, M=0)[0] == 0
    assert m.call(ctx, M=0)[0] == 0
    m.destroy()


def test_abi_optional_outputs_may_be_null(ctx):
    """align1d with h_inv_out = NULL and find_match_direct with NULL search_level / A / h_inv outputs write the other
    outputs exactly as with them."""
    c = ac.batch_problems(4097)
    fr = ctx.frame(c["pyr"])
    conv1, px1, _ = ctx.align1d_batch(fr, c["level"], c["dir"], c["pwb"], c["patch"], 10, c["px"])
    px, conv = c["px"].copy(), np.zeros(len(px1), np.uint8)
    assert ctx.lib.svo_b200_align1d_batch(ctx.h, fr.h, len(px), _p(c["level"]), _p(np.ascontiguousarray(c["dir"])), _p(c["pwb"]),
                                          _p(c["patch"]), 10, _p(px), _p(conv), None) == 0
    assert np.array_equal(conv.astype(bool), conv1) and np.array_equal(ac.bits(px), ac.bits(px1))
    fr.destroy()
    m = _Match(ctx, ac.multi_ref_case(4), n=40)
    rc, full = m.call(ctx)
    rc2, part = m.call(ctx, outs=False)
    assert rc == rc2 == 0 and full["success"].any()
    assert np.array_equal(full["success"], part["success"]) and np.array_equal(ac.bits(full["px_cur"]), ac.bits(part["px_cur"]))
    m.destroy()
