"""svo_b200_fast_detect at its edges: every FAST threshold b the ABI accepts from 0 to 254 in both non-maximum
suppression tie modes, detection thresholds at and around a winner's float32 score (and -0.0), a result cap below the
corner count, occupied grids, equal Shi-Tomasi scores in one cell and pyramid levels too small for a corner.  The kernel
must equal the oracle bit for bit, and both must equal the independent numpy statement in tests/fast_numpy.py wherever
float64 arithmetic decides the cell."""
import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import fast_numpy as fn

pytestmark = pytest.mark.gpu

B_SWEEP = (0, 1, 19, 20, 21, 60, 200, 254)


def _same(g, o):
    assert g["n"] == len(o["x"])
    for k in ("x", "y", "level"):
        assert np.array_equal(g[k], o[k]), k
    assert np.array_equal(g["score"].view(np.uint32), o["score"].view(np.uint32))


def _run(ctx, oracle, pyr, cell, levels, thr, occ=None, b=20, ties=0, cap=8192):
    fr = ctx.frame(pyr)
    try:
        g = ctx.fast_detect(fr, cell, levels, thr, occ, fast_threshold=b, nonmax_ties_suppress=ties, cap=cap)
    finally:
        fr.destroy()
    o = oracle.fast_detect(pyr, levels, cell, thr, occ, cap=max(cap, 8192), nonmax_ties_suppress=ties, fast_threshold=b)
    return g, o


@pytest.mark.parametrize("kind", ["render", "noise", "checker", "low_contrast"])
def test_fast_threshold_sweep(ctx, oracle, kind):
    """b in {0, 1, 19, 20, 21, 60, 200, 254} x both tie modes: kernel == oracle bit for bit on a 160x120 frame, and on a
    64x48 frame both equal the numpy statement on every cell float64 decides."""
    big, small = fn.images(3, 160, 120)[kind], fn.images(1)[kind]
    n_found = 0
    for b in B_SWEEP:
        for ties in (0, 1):
            g, o = _run(ctx, oracle, big, 8, 3, 0.0, b=b, ties=ties)
            _same(g, o)
            n_found += g["n"]
            g, o = _run(ctx, oracle, small, 8, 3, 0.0, b=b, ties=ties)
            _same(g, o)
            r = fn.detect(small, 3, 8, 0.0, b=b, ties_suppress=bool(ties))
            assert len(r["ambiguous"]) <= 2
            fn.agree(r, g, 64, 8)
    assert n_found > 0
    if kind == "checker":  # every corner scores 254 and touches an equal neighbour: the tie modes differ
        sc = fn.fast_scores(small[0], 20)
        assert (sc == 254).sum() == (sc >= 0).sum() > 100
        assert fn.nonmax(sc, True).sum() < fn.nonmax(sc, False).sum()


def test_fast_threshold_zero_keeps_score_zero_corners(ctx, oracle):
    """At b = 0 a corner whose best arc contrast is 1 scores 0.  It is still a corner (the library's scores lie in
    [b, 254]) and it still suppresses equal neighbours when ties suppress."""
    for seed in (1, 2):
        pyr = fn.images(seed)["low_contrast"]
        for ties in (0, 1):
            r = fn.detect(pyr, 3, 8, 0.0, b=0, ties_suppress=bool(ties))
            assert (r["fast_score"] == 0).sum() >= 20                       # surviving score-0 corners win their cells
            g, o = _run(ctx, oracle, pyr, 8, 3, 0.0, b=0, ties=ties)
            _same(g, o)
            assert fn.agree(r, g, 64, 8) >= 40


def test_detection_threshold_edges(ctx, oracle):
    pyr = synth.make_two_view(5, width=320, height=240, n_levels=3)["ref_pyr"]
    g0, o0 = _run(ctx, oracle, pyr, 30, 3, 0.0)
    _same(g0, o0)
    assert g0["n"] > 40
    g, o = _run(ctx, oracle, pyr, 30, 3, -0.0)                              # compares like +0.0
    _same(g, o)
    _same(g, o0)
    # a threshold equal to a winner's float32 score: that corner is no longer strictly better than the threshold
    i = int(np.argsort(g0["score"])[len(g0["score"]) // 2])
    s = float(g0["score"][i])
    above = g0["score"] > s
    for thr in (s, np.nextafter(s, np.inf)):                                # both round to the float32 s
        g, o = _run(ctx, oracle, pyr, 30, 3, thr)
        _same(g, o)
        for k in ("x", "y", "level", "score"):
            assert np.array_equal(g[k], g0[k][above]), k
    assert np.nextafter(s, np.inf) != s and np.float32(np.nextafter(s, np.inf)) == np.float32(s)
    # the double just below s also rounds to s, which is then above the threshold: every cell no corner beat keeps the
    # reference's initial Corner(0, 0, detection_threshold, 0) and emits it at (0, 0), level 0, with score s
    g, o = _run(ctx, oracle, pyr, 30, 3, np.nextafter(s, -np.inf))
    _same(g, o)
    placeholder = (g["x"] == 0) & (g["y"] == 0) & (g["score"] == np.float32(s))
    assert placeholder.sum() == 11 * 8 - above.sum() > 0
    for k in ("x", "y", "level", "score"):
        assert np.array_equal(g[k][~placeholder], g0[k][above]), k
    # no corner beats 1e30, and float32(1e30) > 1e30: every cell emits the placeholder; at exactly float32(1e30), none
    g, o = _run(ctx, oracle, pyr, 30, 3, 1e30)
    _same(g, o)
    assert g["n"] == 11 * 8 and not g["x"].any() and not g["y"].any() and np.all(g["score"] == np.float32(1e30))
    g, o = _run(ctx, oracle, pyr, 30, 3, float(np.float32(1e30)))
    _same(g, o)
    assert g["n"] == 0


def test_detect_cap_occupancy_and_levels(ctx, oracle):
    pyr = synth.make_two_view(6, width=320, height=240, n_levels=3)["ref_pyr"]
    n_cells = 11 * 8
    g_all, o_all = _run(ctx, oracle, pyr, 30, 3, 0.0)
    _same(g_all, o_all)
    for cap in (0, 1, 7):                                                   # the first cap corners in cell order, n = total
        g, _ = _run(ctx, oracle, pyr, 30, 3, 0.0, cap=cap)
        assert g["n"] == g_all["n"] > 7
        for k in ("x", "y", "level"):
            assert np.array_equal(g[k], g_all[k][:cap])
    g, o = _run(ctx, oracle, pyr, 30, 3, 0.0, occ=np.ones(n_cells, np.uint8))
    _same(g, o)
    assert g["n"] == 0
    # occupy the cells won by level-1/2 corners and every other level-0 winner's cell: the runners-up must take over
    cells = fn.cells_of(g_all["x"], g_all["y"], 320, 30)
    occ = np.zeros(n_cells, np.uint8)
    occ[cells[g_all["level"] > 0]] = 1
    occ[cells[g_all["level"] == 0][::2]] = 1
    assert (g_all["level"] > 0).sum() >= 3
    g, o = _run(ctx, oracle, pyr, 30, 3, 0.0, occ=occ)
    _same(g, o)
    assert not occ[fn.cells_of(g["x"], g["y"], 320, 30)].any()


def test_tiled_motif_equal_scores_first_in_scan_order(ctx, oracle):
    """A 16x16 motif tiled over the frame: every cell of 32 px holds several corners with exactly equal Shi-Tomasi
    scores, and the first in (level, row, column) order must win."""
    motif = np.random.default_rng(4).integers(0, 256, (16, 16), dtype=np.uint8)
    pyr = synth.build_pyramid(np.tile(motif, (6, 8)), 3)                    # 128 x 96
    for ties in (0, 1):
        r = fn.detect(pyr, 3, 32, 0.0, ties_suppress=bool(ties))
        g, o = _run(ctx, oracle, pyr, 32, 3, 0.0, ties=ties)
        _same(g, o)
        assert fn.agree(r, g, 128, 32) == 12
        # equal best scores inside one cell: the winner is the first of them
        st = {}
        for L in range(3):
            keep = fn.nonmax(fn.fast_scores(pyr[L], 20), bool(ties))
            for y, x in zip(*np.nonzero(keep)):
                st.setdefault((int(y) << L) // 32 * 4 + (int(x) << L) // 32, []).append(fn.shi_tomasi(pyr[L], int(x), int(y))[0])
        tied = [k for k, v in st.items() if v.count(max(v)) > 1]
        assert len(tied) >= 4


@pytest.mark.parametrize("w,h,levels", [(40, 28, 3), (192, 104, 5), (64, 40, 4)])
def test_small_top_levels(ctx, oracle, w, h, levels):
    """Top levels narrower or lower than 7 px (no pixel passes the 3-px border) and than 10 px (no Shi-Tomasi box)."""
    img = np.random.default_rng(w).integers(0, 256, (h, w), dtype=np.uint8)
    pyr = synth.build_pyramid(img, levels)
    assert min(pyr[-1].shape) < 10
    for ties in (0, 1):
        g, o = _run(ctx, oracle, pyr, 8, levels, 0.0, ties=ties)
        _same(g, o)
        assert g["n"] > 0
