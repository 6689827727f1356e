"""GPU: the level setup of the one-CTA alignment geometries -- reference patches, the level's H sum (one sweep over a thread's
features in the 160 x 2 geometry, the other warps not waiting for the warp that sums and factorises it) and the slow path's
H sum -- at the cases that reach its edges, in both one-CTA geometries:

  edge-159 ... edge-304  feature counts at the last warp's and the 304-slot edges of the 160 x 2 geometry (the warp that sums
                         H owns slots 128-159 and 288-303); has_point is cleared at sc.EDGE_SLOTS, so every level has visible
                         and invisible patches side by side
  border-only            only features 3-5 px from a border: no patch is visible at levels 4 ... 1 (n_meas == 0, x = 0)
  border-300             a quarter of the features at the borders and a motion that moves patches out of the current image:
                         slow-path passes, and visible / invisible patches at every level

Each case is compared with the oracle (tests/sia_cases.py tolerances) and bit for bit with a recording made before the H sum
was restructured (tests/golden/sia_level_setup_bits.npz).  Recorded on an H100 with the library of the commit before that
change:
    SVO_SIA_LEVEL_SETUP_RECORD=tests/golden/sia_level_setup_bits.npz SVO_B200_LIB=<that build's libsvo_b200.so> \\
        python -m pytest tests/test_sia_level_setup_gpu.py -k recorded
"""
import os

import numpy as np
import pytest

from tests import sia_cases as sc

pytestmark = pytest.mark.gpu

GEOMETRIES = {"cta-2fpt": ((1, 2), 2), "cta-1fpt": ((1, 1), 1)}  # sia_config(ctas, fpt), features per thread launched
EDGE_COUNTS = (159, 160, 161, 303, 304)
CASES = [f"edge-{n}" for n in EDGE_COUNTS] + ["border-only", "border-300"]
BITS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sia_level_setup_bits.npz")


def _border_only(d):
    """The features of a border_pair that sit 3-5 px from a border (its first quarter and the four corner ones)."""
    nb = len(d["px"]) // 4 + 4
    e = dict(d)
    for k in ("px", "f", "pos", "has_point"):
        e[k] = np.ascontiguousarray(d[k][:nb])
    return e


@pytest.fixture(scope="module")
def cases():
    base = sc.base_pair()
    out = {f"edge-{n}": sc.subset(base, n) for n in EDGE_COUNTS}
    border = sc.border_pair(10, 640, 480, 300)  # a seed whose decisions are far from a tie
    out["border-only"] = _border_only(border)
    out["border-300"] = border
    return out


@pytest.fixture(scope="module")
def frames(ctx, cases):
    made = {}
    for name, d in cases.items():
        key = id(d["ref_pyr"])
        if key not in made:
            made[key] = (ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"]))
    yield {name: made[id(d["ref_pyr"])] for name, d in cases.items()}
    for r, c in made.values():
        r.destroy(); c.destroy()


@pytest.fixture(autouse=True)
def _reset_config(ctx):
    yield
    ctx.sia_config(-1, 0)


def _run(ctx, d, fr, geometry):
    cfg, fpt = GEOMETRIES[geometry]
    ctx.sia_config(*cfg)
    g = sc.gpu_run(ctx, d, frames=fr)
    L = ctx.sia_last_launch()
    assert (L["ctas_per_pair"], L["features_per_thread"], L["upfront"]) == (1, fpt, 0), L
    return g


_oracle_cache = {}


def _without_nan_chi2(r):
    """A level without a visible patch has n_meas == 0 and chi2 = 0 / 0 (NaN) in the kernel and the oracle alike."""
    return dict(r, trace=[dict(t, chi2=0.0 if np.isnan(t["chi2"]) else t["chi2"]) for t in r["trace"]])


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
@pytest.mark.parametrize("case", CASES)
def test_level_setup_edges_match_the_oracle(ctx, oracle, cases, frames, case, geometry):
    d = cases[case]
    g = _run(ctx, d, frames[case], geometry)
    if case not in _oracle_cache:
        _oracle_cache[case] = sc.oracle_run(oracle, d)
    o = _oracle_cache[case]
    if case.startswith("border"):
        assert sc.decision_margin(o) > 2e-5  # no accept / roll-back / convergence decision is a rounding near-tie
    by_level = {}
    for t in o["trace"]:
        by_level.setdefault(t["level"], []).append(t)
    if case == "border-only":
        assert all(t["n_meas"] == 0 for lv in (4, 3, 2, 1) for t in by_level[lv]) and by_level[0][0]["n_meas"] > 0
    if case == "border-300":
        assert any(t["n_meas"] // 16 < int(o["visible"].sum()) for t in by_level[0])  # patches really left the image
    assert [np.isnan(t["chi2"]) for t in g["trace"]] == [np.isnan(t["chi2"]) for t in o["trace"]]
    sc.assert_parity(_without_nan_chi2(g), _without_nan_chi2(o), n_feat=len(d["px"]))


def _outputs(g):
    tr = g["trace"]
    return {"T": np.asarray(g["T"]), "H": np.asarray(g["H"]), "visible": np.asarray(g["visible"]),
            "n_tracked": np.array(g["n_tracked"]),
            "steps": np.array([(t["level"], t["iter"], t["accepted"], t["n_meas"]) for t in tr], dtype=np.int64).reshape(-1, 4),
            "chi2": np.array([t["chi2"] for t in tr]), "x": np.array([t["x"] for t in tr]).reshape(-1, 6)}


def test_level_setup_edges_are_bit_identical_to_the_recorded_ones(ctx, cases, frames):
    """Pose, H, mask, counters and the whole iteration trace of every case in both geometries, bit for bit.
    SVO_SIA_LEVEL_SETUP_RECORD=<file> records them instead."""
    from tests.golden.make_golden import digest

    got = {"input_sha256": np.array(digest(*[a for c in CASES for a in (*cases[c]["ref_pyr"], *cases[c]["cur_pyr"], cases[c]["px"],
                                                                        cases[c]["f"], cases[c]["pos"], cases[c]["has_point"],
                                                                        cases[c]["ref_pos"])]))}
    for geometry in GEOMETRIES:
        for case in CASES:
            for k, v in _outputs(_run(ctx, cases[case], frames[case], geometry)).items():
                got[f"{geometry}/{case}/{k}"] = v
    if os.environ.get("SVO_SIA_LEVEL_SETUP_RECORD"):
        np.savez(os.environ["SVO_SIA_LEVEL_SETUP_RECORD"], **got)
        return
    with np.load(BITS, allow_pickle=False) as z:
        want = {k: z[k] for k in z.files}
    assert str(got["input_sha256"]) == str(want["input_sha256"]), "the synthetic inputs differ from the recorded ones"
    assert set(got) == set(want)
    for k in sorted(set(got) - {"input_sha256"}):
        a, b = np.atleast_1d(got[k]), np.atleast_1d(want[k])
        assert a.shape == b.shape and a.dtype == b.dtype, k
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), k
