"""GPU: depth_filter_kernel's computeTau + updateSeed against the exactly rounded statement of tests/depth_update_hp.py.

Every seed that reaches updateSeed must leave the kernel as one of the statement's candidate tuples (a, b, mu, sigma2,
status), bit for bit, from the depth z the kernel reports: x = (float)(1./z) exactly, tau2 among the floats of the
computeTau enclosure, exp(exponent) within CUDA's 2 ulp.  The oracle goes through the same check with exp pinned to
glibc's expf.  Seeds that never reach updateSeed stay bit-identical to the oracle.  The depth itself must lie within
depthFromTriangulation's bound, in the update and in the match-only mode."""
import math
import time

import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import depth_update_cases as cases
from tests import depth_update_hp as hp

pytestmark = pytest.mark.gpu

KEYS = ("a", "b", "mu", "sigma2")
UPDATED, NO_MATCH = 5, 4


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _same(x, y):
    """Bit for bit, NaNs by class (the device's float ops return the canonical NaN, the host's keep the payload)."""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    return bool(np.all((_bits(x) == _bits(y)) | (np.isnan(x) & np.isnan(y))))


def _args(c):
    return (c["ref_index"], c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"],
            c["batch_counter"], c["seeds"])


def _run(ctx, oracle, c, **kw):
    ref, cur = ctx.frame(c["ref_pyr"]), ctx.frame(c["cur_pyr"])
    g = ctx.depth_filter_update([ref], [c["T_ref_w"]], cur, c["T_cur_w"], c["cam"], *_args(c), **kw)
    ref.destroy(); cur.destroy()
    o = oracle.depth_filter_update([c["ref_pyr"]], [c["T_ref_w"]], c["cur_pyr"], c["T_cur_w"], c["cam"], *_args(c), **kw)
    return g, o


def _check(c, out, exp, oracle=None):
    return hp.check_launch(out, c["seeds"], [c["T_ref_w"]], c["ref_index"], c["T_cur_w"], c["ftr_f"], c["cam"].fx,
                           exp=exp, oracle=oracle)


def _merge(tot, rep):
    for k in ("n", "single", "ill"):
        tot[k] = tot.get(k, 0) + rep[k]
    for d in ("k", "rec"):
        for key, v in rep[d].items():
            tot.setdefault(d, {})[key] = tot.setdefault(d, {}).get(key, 0) + v


def _all_cases():
    out = [(f"small_parallax_{b}", cases.small_parallax(77, b)) for b in cases.SMALL_BASELINES]
    return out + [("evolved", cases.evolved()), ("degenerate", cases.degenerate()), ("no_match", cases.no_match())]


@pytest.fixture(scope="module")
def runs(ctx, oracle):
    return [(name, c) + _run(ctx, oracle, c) for name, c in _all_cases()]


def test_every_updated_seed_is_a_candidate(runs, oracle):
    t0 = time.time()
    tot_g, tot_o = {}, {}
    for name, c, g, o in runs:
        # the match is the same code on both sides: the same seeds reach updateSeed, the others are bit-identical
        assert np.array_equal(g["n_zmssd"], o["n_zmssd"]), name
        upd = o["status"] >= UPDATED
        assert np.array_equal(g["status"] >= UPDATED, upd), name
        assert np.array_equal(g["status"][~upd], o["status"][~upd]), name
        for k in KEYS:
            assert _same(g[k][~upd], o[k][~upd]), (name, k)
        rg, ro = _check(c, g, "device"), _check(c, o, "glibc", oracle)
        assert not rg["bad"], (name, rg["bad"][:3])
        assert not ro["bad"], (name, ro["bad"][:3])
        assert ro["single"] == ro["n"], name
        ill = np.asarray(rg["ill_idx"], int)  # a seed whose tau2 enclosure is too wide to list: also near the oracle's
        for k in KEYS:
            assert np.allclose(g[k][ill], o[k][ill], rtol=2e-5, atol=1e-7, equal_nan=True), (name, k)
        _merge(tot_g, rg)
        _merge(tot_o, ro)
    print(f"kernel: {tot_g['n']} updated seeds, {tot_g['single']} with a single tau2 candidate "
          f"({tot_g['single'] / tot_g['n']:.1%}), {tot_g['ill']} ill-conditioned; expf offset k: {dict(sorted(tot_g['k'].items()))}")
    print("kernel branches:", dict(sorted(tot_g["rec"].items())))
    print(f"oracle: {tot_o['n']} updated seeds, each bit for bit its single statement; check took {time.time() - t0:.1f} s")
    for br in ("gamma=pos", "gamma=neg", "clamp=yes", "clamp=no"):
        assert tot_g["rec"].get(br, 0) > 0, br
    assert tot_g["n"] > 1000
    assert tot_g["ill"] <= tot_g["n"] // 20


def test_degenerate_groups_reach_the_update(runs):
    """Each degenerate field (a or b zero, subnormal, negative, NaN, a + b overflowing or past 2^24, z_range 0, negative,
    subnormal, inf, NaN, sigma2 subnormal) reaches updateSeed on some seed, whose result the candidate check covered."""
    (c, g), = [(c, g) for name, c, g, _ in runs if name == "degenerate"]
    reached = {grp: int(np.sum((c["group"] == grp) & (g["status"] >= UPDATED))) for grp in cases.DEGENERATE}
    print("degenerate groups updated:", reached)
    assert all(v > 0 for v in reached.values()), reached


def test_no_match_increments_b(runs):
    """NO_MATCH's b + 1 in float: 2^24 + 1 is 2^24, inf and NaN stay; the other fields are untouched."""
    (c, g), = [(c, g) for name, c, g, _ in runs if name == "no_match"]
    nm = g["status"] == NO_MATCH
    b0 = c["seeds"]["b"][nm]
    assert _same(g["b"][nm], b0 + np.float32(1))
    for k in ("a", "mu", "sigma2"):
        assert _same(g[k][nm], c["seeds"][k][nm]), k
    seen = {float(v) for v in b0} | ({math.nan} if np.isnan(b0).any() else set())
    assert {2.0 ** 24, math.inf}.issubset(seen) and np.isnan(b0).any(), seen


def test_depth_within_the_triangulation_bound(ctx, oracle, runs):
    """z of every updated seed (update mode) and of every successful candidate (match-only mode, the same seeds' windows)
    lies within depthFromTriangulation's bound around the 40-digit depth from the kernel's own px_cur, and the det < 1e-6
    decision agrees wherever its margin is decisive."""
    sides = {"det>=1e-6": 0, "det<1e-6": 0, "not decisive": 0}
    worst = 0.0
    for name, c, g, _ in runs:
        if not name.startswith("small_parallax"):
            continue
        T_cur_ref = synth.se3_mul(c["T_cur_w"], synth.se3_inv(c["T_ref_w"]))
        s = c["seeds"]
        sq = np.sqrt(s["sigma2"])
        d = (1.0 / s["mu"].astype(np.float64), 1.0 / (s["mu"] + sq).astype(np.float64),
             1.0 / np.maximum(s["mu"] - sq, np.float32(1e-8)).astype(np.float64))
        ref, cur = ctx.frame(c["ref_pyr"]), ctx.frame(c["cur_pyr"])
        m = ctx.find_epipolar_match_direct([ref], [c["T_ref_w"]], cur, c["T_cur_w"], c["cam"], c["ref_index"], c["ftr_px"],
                                           c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"], *d)
        ref.destroy(); cur.destroy()
        for mode, ok, z, px in (("update", g["status"] >= UPDATED, g["z"], g["px_cur"]),
                                ("match", m["success"], m["depth"], m["px_cur"])):
            for i in np.flatnonzero(ok | ((mode == "match") & np.any(px != 0, axis=1))):
                f_cur = hp.pinhole_bearing(c["cam"], px[i][0], px[i][1])
                zh, det, bound, det_unc = hp.triangulation(T_cur_ref, c["ftr_f"][i], f_cur)
                decisive = abs(det - 1e-6) > det_unc
                if not decisive:
                    sides["not decisive"] += 1
                    continue
                if ok[i]:
                    assert det >= 1e-6, (name, mode, i, det)
                    sides["det>=1e-6"] += 1
                    assert abs(z[i] - zh) <= bound, (name, mode, i, z[i], zh, bound)
                    worst = max(worst, abs(z[i] - zh) / bound)
                elif det < 1e-6:
                    sides["det<1e-6"] += 1
        assert np.array_equal(m["success"], g["status"] >= UPDATED), name
        assert np.array_equal(m["depth"][m["success"]], g["z"][m["success"]]), name
    print("triangulation decisions:", sides, f"worst |z - z_exact| / bound {worst:.3g}")
    assert sides["det>=1e-6"] > 0 and sides["det<1e-6"] > 0


def _one_seed(c, i):
    d = dict(c)
    for k in ("ref_index", "ftr_px", "ftr_f", "ftr_level", "ftr_type", "ftr_grad", "batch_id"):
        d[k] = np.ascontiguousarray(c[k][i:i + 1])
    d["seeds"] = {k: v[i:i + 1].copy() for k, v in c["seeds"].items()}
    return d


def test_convergence_test_at_its_tie(ctx, oracle):
    """sigma2_thresh does not enter the update.  With (double)z_range / thresh equal to (double)sqrtf(sigma2_new) the
    strict `<` keeps the seed UPDATED; one ulp of thresh to either side converges it or keeps it."""
    c = cases.small_parallax(77, 0.05)
    g0, _ = _run(ctx, oracle, c)
    i = int(np.flatnonzero(g0["status"] == UPDATED)[0])
    one = _one_seed(c, i)
    s = hp.sqrt(float(g0["sigma2"][i]), "s")
    zr = float(c["seeds"]["z_range"][i])
    near = [zr / s]
    for direction in (0.0, np.inf):
        t = zr / s
        for _ in range(64):
            t = float(np.nextafter(t, direction))
            near.append(t)
    th = next(t for t in near if zr / t == s)
    lo, hi = float(np.nextafter(th, 0.0)), float(np.nextafter(th, np.inf))
    while zr / lo == s:
        lo = float(np.nextafter(lo, 0.0))
    while zr / hi == s:
        hi = float(np.nextafter(hi, np.inf))
    got = {}
    for name, t in (("tie", th), ("looser", lo), ("tighter", hi)):
        g, o = _run(ctx, oracle, one, sigma2_thresh=t)
        assert np.array_equal(_bits(g["sigma2"]), _bits(g0["sigma2"][i:i + 1])), name  # thresh does not enter the update
        got[name] = (int(g["status"][0]), int(o["status"][0]) if o["z"][0] == g0["z"][i] else None)
    print("convergence tie:", got)
    assert got["tie"][0] == UPDATED and got["tighter"][0] == UPDATED and got["looser"][0] == hp.CONVERGED
