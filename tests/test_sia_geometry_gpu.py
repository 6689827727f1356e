"""GPU: every launch geometry of the alignment kernel at its capacity edges, and every staging path on odd-sized pyramids.

Each case forces a configuration (svo_b200_sia_config / svo_b200_sia_upfront), asserts through svo_b200_sia_last_launch
which instantiation actually ran -- a fallback inside the launch choice would otherwise turn a cluster test into a one-CTA
test with every assertion still passing -- and compares with the CPU oracle (tests/sia_cases.py: assert_parity).
"""
import os

import numpy as np
import pytest

from rpg_svo_b200 import capi, synth
from tests import sia_cases as sc

pytestmark = pytest.mark.gpu

# (ctas_per_pair, features_per_thread, upfront mode) as in test_sia_gpu.GEOMETRIES, plus the 2-CTA cluster
GEOMETRIES = {"auto": (-1, 0, -1), "cta-1fpt": (1, 1, -1), "cta-2fpt": (1, 2, -1), "cluster-2": (2, 0, -1),
              "cluster-4": (4, 0, -1), "cluster-4-per-level": (4, 0, 0), "cluster-8": (8, 0, -1)}


def _configure(ctx, cfg):
    ctx.sia_config(cfg[0], cfg[1])
    ctx.sia_upfront(cfg[2])


@pytest.fixture(autouse=True)
def _reset_config(ctx):
    yield
    ctx.sia_config(-1, 0)
    ctx.sia_upfront(-1)


def _geom(L):
    return (L["ctas_per_pair"], L["threads"], L["features_per_thread"], bool(L["upfront"]))


@pytest.fixture(scope="module")
def base():
    return sc.base_pair()


@pytest.fixture(scope="module")
def base_frames(ctx, base):
    fr = (ctx.frame(base["ref_pyr"]), ctx.frame(base["cur_pyr"]))
    yield fr
    for f in fr:
        f.destroy()


_oracle_cache = {}


def _oracle(oracle, key, d, **kw):
    if key not in _oracle_cache:
        _oracle_cache[key] = sc.oracle_run(oracle, d, **kw)
    return _oracle_cache[key]


# ---- 1. capacity edges: (config, N, expected (CTAs per pair, threads, features per thread, upfront)) ----------------------
UP4 = (4, 96, 1, True)
EDGE_ROWS = (
    [((-1, 0, -1), n, UP4) for n in (16, 95, 96, 97, 383, 384)]
    + [((-1, 0, -1), n, (1, 512, 1, False)) for n in (385, 512)]
    + [((-1, 0, -1), n, (1, 512, 2, False)) for n in (513, 1024)]
    + [((1, 1, -1), 320, (1, 320, 1, False)), ((1, 1, -1), 321, (1, 384, 1, False)), ((1, 1, -1), 384, (1, 384, 1, False)),
       ((1, 1, -1), 385, (1, 512, 1, False))]
    + [((1, 2, -1), n, (1, 160, 2, False)) for n in (159, 160, 161, 303, 304)]
    + [((1, 2, -1), 305, (1, 320, 1, False))]
    + [((2, 0, -1), n, (2, 96, 1, False)) for n in (1, 96, 97, 192)]
    + [((2, 0, -1), 193, (1, 160, 2, False))]  # more than 2 x 96 features: one CTA per pair (the automatic one-CTA choice)
    + [((8, 0, -1), n, (8, 96, 1, False)) for n in (1, 97, 767, 768)]
    + [((8, 0, -1), 769, (1, 512, 2, False))]
    + [((4, 0, 0), n, (4, 96, 1, False)) for n in (97, 384)]
)


@pytest.mark.parametrize("cfg,n,expect", EDGE_ROWS, ids=[f"{c[0]}.{c[1]}.{c[2]}-N{n}" for c, n, _ in EDGE_ROWS])
def test_capacity_edges(ctx, oracle, base, base_frames, cfg, n, expect):
    d = sc.subset(base, n)
    _configure(ctx, cfg)
    g = sc.gpu_run(ctx, d, frames=base_frames)
    L = ctx.sia_last_launch()
    assert _geom(L) == expect, L
    assert L["n_pairs"] == 1 and not L["residuals_only"]
    sc.assert_parity(g, _oracle(oracle, ("base", n), d), n_feat=n)


def test_more_than_1024_features_is_an_error_not_a_launch(ctx, base, base_frames):
    d = sc.subset(base, 1025)
    with pytest.raises(capi.SvoB200Error, match="1024"):
        sc.gpu_run(ctx, d, frames=base_frames)


# ---- distorted cameras through the general-camera instantiations of the main geometries ------------------------------------
CAM_ROWS = [("atan", (-1, 0, -1), UP4), ("atan", (1, 1, -1), (1, 320, 1, False)), ("atan", (1, 2, -1), (1, 160, 2, False)),
            ("atan", (4, 0, 0), (4, 96, 1, False)), ("pinhole_radtan", (-1, 0, -1), UP4),
            ("pinhole_radtan", (1, 2, -1), (1, 160, 2, False)), ("pinhole_radtan", (1, 1, -1), (1, 320, 1, False)),
            ("pinhole_radtan", (4, 0, 0), (4, 96, 1, False))]


@pytest.fixture(scope="module")
def cam_pairs():
    out = {}
    for kind in ("atan", "pinhole_radtan"):
        cam = synth.reference_param_camera(kind)
        out[kind] = synth.make_frame_pair(1000, width=cam.width, height=cam.height, n_feat=300, n_levels=5, cam=cam)
    return out


@pytest.mark.parametrize("kind,cfg,expect", CAM_ROWS, ids=[f"{k}-{c[0]}.{c[1]}.{c[2]}" for k, c, _ in CAM_ROWS])
def test_distorted_cameras_run_the_general_camera_instantiations(ctx, oracle, cam_pairs, kind, cfg, expect):
    d = cam_pairs[kind]
    _configure(ctx, cfg)
    g = sc.gpu_run(ctx, d)
    L = ctx.sia_last_launch()
    assert _geom(L) == expect and L["general_camera"] == 1, L
    sc.assert_parity(g, _oracle(oracle, ("cam", kind), d))


# ---- 2. batches -----------------------------------------------------------------------------------------------------------
def _batch(ctx, frames, parts, T0=None):
    """Stage / run / fetch one batch: parts = list of feature dicts, all on the same frame pair."""
    B = len(parts)
    off = np.concatenate([[0], np.cumsum([len(p["px"]) for p in parts])]).astype(np.int32)
    cat = lambda k, shape: np.concatenate([p[k] for p in parts]) if off[-1] else np.zeros(shape)  # noqa: E731
    T0 = np.tile(synth.se3_identity(), (B, 1, 1)) if T0 is None else T0
    ctx.sia_batch_stage([frames[0]] * B, [frames[1]] * B, parts[0]["cam"], T0, off, cat("px", (0, 2)), cat("f", (0, 3)),
                        cat("pos", (0, 3)), cat("has_point", (0,)).astype(np.uint8), np.stack([p["ref_pos"] for p in parts]), 4, 0)
    ctx.sia_batch_run()
    r = ctx.sia_batch_fetch(want_H=True)
    L = ctx.sia_last_launch()
    out = [dict(T=r["T"][k], H=r["H"][k], visible=r["visible"][off[k]:off[k + 1]], n_tracked=int(r["stats"]["n_tracked"][k]))
           for k in range(B)]
    return out, L


def _throughput_batches(base):
    """Two batches large enough for the automatic one-CTA choice: 36 pairs (4 B > 132 SMs) at the slot edges, with an empty
    pair and a pair without any 3D point, and 64 pairs with feature counts from 1 to 300."""
    edges = [sc.subset(base, n) for n in (0, 1, 17, 159, 160, 161, 303, 304)]
    no_pts = sc.subset(base, 200)
    no_pts["has_point"][:] = 0
    edges.append(no_pts)
    edges += [sc.subset(base, 250 + k) for k in range(36 - len(edges))]
    spread = [sc.subset(base, n) for n in [1, 17, 159, 160, 161, 299, 300] + [int(n) for n in np.linspace(20, 300, 57).astype(int)]]
    return {"edges-36": edges, "spread-64": spread}


def test_throughput_batch_with_edge_counts_equals_single_calls(ctx, oracle, base, base_frames):
    """Batches in the throughput geometry (160 x 2), pairs at its slot edges, an empty pair and a pair without any 3D point:
    every pair equals a single call forced onto the same geometry bit for bit, and the oracle."""
    for name, parts in _throughput_batches(base).items():
        ctx.sia_config(-1, 0)
        out, L = _batch(ctx, base_frames, parts)
        assert _geom(L) == (1, 160, 2, False) and L["n_pairs"] == len(parts), (name, L)
        ctx.sia_config(1, 2)
        for k, p in enumerate(parts):
            n = len(p["px"])
            if n == 0 or not p["has_point"].any():
                assert out[k]["n_tracked"] == 0 and np.array_equal(out[k]["T"], synth.se3_identity()), (name, k)
                assert not out[k]["visible"].any()
                continue
            s = sc.gpu_run(ctx, p, frames=base_frames)
            assert _geom(ctx.sia_last_launch()) == (1, 160, 2, False)
            assert np.array_equal(out[k]["T"], s["T"]) and np.array_equal(out[k]["H"], s["H"]), (name, k)
            assert np.array_equal(out[k]["visible"], s["visible"]) and out[k]["n_tracked"] == s["n_tracked"], (name, k)
            # The spread batch's counts are not chosen for a decision margin (sc.decision_margin): at N = 105 a near-tie ends
            # the iterations three iterations apart from the oracle's, so there the batch outputs (mask, n_tracked, pose) are
            # compared and the iteration trace is not.
            sc.assert_parity(s if name == "edges-36" else out[k], _oracle(oracle, ("base", n), p), n_feat=n)


def test_occupancy_fallback_upfront_then_per_level_then_one_cta(ctx, oracle, base, base_frames):
    """Small batches: the upfront 4-CTA cluster while all B clusters are resident at once (the device's
    cudaOccupancyMaxActiveClusters, reported by the launch), then the per-level cluster flow, then one CTA per pair once
    4 B exceeds the SM count."""
    d = sc.subset(base, 100)
    sc.gpu_run(ctx, d, frames=base_frames)
    L = ctx.sia_last_launch()
    n, sms = L["resident_clusters"], L["sm_count"]
    assert _geom(L) == UP4 and n >= 1, L
    sizes = sorted({n, n + 1, sms // 4, sms // 4 + 1})
    o = _oracle(oracle, ("base", 100), d)
    seen = []
    for B in sizes:
        out, L = _batch(ctx, base_frames, [d] * B)
        expect = UP4 if B <= n and 4 * B <= sms else (4, 96, 1, False) if 4 * B <= sms else (1, 160, 2, False)
        assert _geom(L) == expect, (B, n, sms, L)
        seen.append(expect)
        for k in (0, B - 1):
            sc.assert_parity(out[k], o)
    assert seen[0] == UP4 and seen[-1] == (1, 160, 2, False) and (4, 96, 1, False) in seen, seen


# ---- 3. odd pyramid shapes, every geometry ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def odd(ctx):
    out = {}
    for size in sc.ODD_SIZES:
        d = sc.odd_pair(size)
        out[size] = (d, ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"]))
    yield out
    for _, r, c in out.values():
        r.destroy(); c.destroy()


def _expected_stages(size, L):
    """The staging mode each odd shape is there to reach, per geometry (the throughput geometry has no windows and a
    staging region of ~6 KB, so it gathers those levels from global memory instead)."""
    tp = L["threads"] == 160
    if size == (644, 484):
        return {0: "global", 1: "global", 2: "global" if tp else "image"}
    if size == (648, 488):
        return {0: "global" if tp else "window", 1: "global"}
    if size == (160, 120):
        return {0: "global" if tp else "image", 1: "image"}
    return {0: "global" if tp else "window", 1: "global" if tp else "window"}


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
@pytest.mark.parametrize("size", sc.ODD_SIZES, ids=[f"{w}x{h}" for w, h in sc.ODD_SIZES])
def test_odd_pyramid_alignment(ctx, oracle, odd, size, geometry):
    d, ref, cur = odd[size]
    _configure(ctx, GEOMETRIES[geometry])
    g = sc.gpu_run(ctx, d, frames=(ref, cur))
    L = ctx.sia_last_launch()
    cfg = GEOMETRIES[geometry]
    if cfg[0] > 1:
        assert L["ctas_per_pair"] == cfg[0], L
    for lv, mode in _expected_stages(size, L).items():
        assert L["stages"][lv] == mode, (lv, L)
    o = _oracle(oracle, ("odd", size), d)
    assert any(t["n_meas"] // 16 < int(o["visible"].sum()) for t in o["trace"])  # patches really left the image
    assert sc.decision_margin(o) > 2e-5  # no accept / roll-back / convergence decision is a rounding near-tie
    sc.assert_parity(g, o)


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
@pytest.mark.parametrize("size", sc.ODD_SIZES, ids=[f"{w}x{h}" for w, h in sc.ODD_SIZES])
def test_odd_pyramid_residual_pass(ctx, oracle, odd, size, geometry):
    """At the motion (patches leave the image) and at the identity (the features 3-4 px from the right / bottom edge then
    sit on the last column / row whose footprint fits: the border test's edge case, in every staging mode)."""
    d, ref, cur = odd[size]
    _configure(ctx, GEOMETRIES[geometry])
    for pose, T in (("motion", d["T_gt"]), ("identity", synth.se3_identity())):
        for level in range(5):
            g = ctx.sparse_residuals(ref, cur, d["cam"], level, T, d["px"], d["f"], d["pos"], d["has_point"], d["ref_pos"])
            L = ctx.sia_last_launch()
            assert L["residuals_only"] == 1 and L["min_level"] == L["max_level"] == level
            if level in _expected_stages(size, L):
                assert L["stages"][level] == _expected_stages(size, L)[level], (level, L)
            key = ("odd-res", size, pose, level)
            if key not in _oracle_cache:
                _oracle_cache[key] = oracle.sparse_residuals(d["ref_pyr"][level], d["cur_pyr"][level], level, d["cam"], T,
                                                             d["px"], d["f"], d["pos"], d["has_point"], d["ref_pos"])
            sc.assert_residual_parity(g, _oracle_cache[key])


BITS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sia_geometry_bits.npz")


def test_results_are_bit_identical_to_the_recorded_ones(ctx, odd):
    """The oracle's tolerances cannot see a change of summation order (a reordered partial sum moves the result by an ulp),
    which every geometry fixes by construction and the data-movement changes planned for the kernel must keep.  So the exact
    outputs of every geometry on the 648x488 border case are pinned: pose, H and the trace's chi2 and steps, bit for bit.
    SVO_SIA_BITS_RECORD=<file> records them instead (after a deliberate change of arithmetic)."""
    from tests.golden.make_golden import digest

    d, ref, cur = odd[(648, 488)]
    got = {"input_sha256": np.array(digest(*d["ref_pyr"], *d["cur_pyr"], d["px"], d["f"], d["pos"], d["has_point"], d["ref_pos"]))}
    for name, cfg in GEOMETRIES.items():
        _configure(ctx, cfg)
        g = sc.gpu_run(ctx, d, frames=(ref, cur))
        got[f"{name}/T"], got[f"{name}/H"] = g["T"], g["H"]
        got[f"{name}/chi2"] = np.array([t["chi2"] for t in g["trace"]])
        got[f"{name}/x"] = np.array([t["x"] for t in g["trace"]])
    if os.environ.get("SVO_SIA_BITS_RECORD"):
        np.savez(os.environ["SVO_SIA_BITS_RECORD"], **got)
        return
    with np.load(BITS, allow_pickle=False) as z:
        want = {k: z[k] for k in z.files}
    assert str(got["input_sha256"]) == str(want["input_sha256"]), "the synthetic inputs differ from the recorded ones"
    assert set(got) == set(want)
    for k in got:
        if k != "input_sha256":
            assert got[k].shape == want[k].shape and np.array_equal(got[k].view(np.uint64), want[k].view(np.uint64)), k


@pytest.mark.parametrize("geometry", ["auto", "cta-1fpt", "cta-2fpt"])
def test_last_frame_of_an_odd_sized_pool_as_current_frame(ctx, oracle, geometry):
    """Frames of a pool share one slab per level with no per-frame slack: only the slab's trailing 256 bytes are there for
    the aligned-word fetches past the last pixel.  The last frame, at 644x484, is the current frame of a two-pair batch
    whose features include the bottom-right corner."""
    d = sc.odd_pair((644, 484))
    pool = capi.FramePool(ctx, 644, 484, 5, 3)
    try:
        pool.upload_array(np.stack([d["ref_pyr"][0], d["ref_pyr"][0], d["cur_pyr"][0]]))
        ref, cur = pool.frames[0], pool.frames[2]
        # the pool builds its own pyramids: the oracle runs on exactly those levels
        e = dict(d, ref_pyr=[ref.download_level(l) for l in range(5)], cur_pyr=[cur.download_level(l) for l in range(5)])
        _configure(ctx, GEOMETRIES[geometry])
        out, L = _batch(ctx, (ref, cur), [e, e])
        assert L["n_pairs"] == 2 and L["stages"][0] == "global", L
        o = _oracle(oracle, ("pool", 644), e)
        br = (d["px"][:, 0] > 644 - 6) & (d["px"][:, 1] > 484 - 6)
        assert br.sum() >= 4 and o["visible"][br].any()  # the corner features are really tracked at level 0
        for k in range(2):
            sc.assert_parity(out[k], o)
    finally:
        pool.destroy()


# ---- 4. every instantiation and every staging mode is reached -------------------------------------------------------------
def _inst(r):
    return (r["residuals_only"], r["ctas_per_pair"], r["threads"], r["features_per_thread"], r["min_blocks"], r["general_camera"],
            r["upfront"])


# (residuals pass, CTAs per pair, threads, features per thread, MINB, general camera, upfront): the branches of launch_sia
ALIGN_INSTANTIATIONS = [(0, 2, 96, 1, 2, 1, 0), (0, 4, 96, 1, 1, 0, 1), (0, 4, 96, 1, 1, 1, 1), (0, 4, 96, 1, 2, 0, 0),
                        (0, 4, 96, 1, 2, 1, 0), (0, 8, 96, 1, 2, 1, 0), (0, 1, 320, 1, 2, 0, 0), (0, 1, 320, 1, 2, 1, 0),
                        (0, 1, 384, 1, 2, 1, 0), (0, 1, 512, 1, 1, 1, 0), (0, 1, 160, 2, 3, 0, 0), (0, 1, 160, 2, 3, 1, 0),
                        (0, 1, 512, 2, 1, 1, 0)]
RESIDUAL_INSTANTIATIONS = [(1, 2, 96, 1, 2, 1, 0), (1, 4, 96, 1, 2, 1, 0), (1, 8, 96, 1, 2, 1, 0), (1, 1, 320, 1, 2, 1, 0),
                           (1, 1, 384, 1, 2, 1, 0), (1, 1, 512, 1, 1, 1, 0), (1, 1, 160, 2, 3, 1, 0), (1, 1, 512, 2, 1, 1, 0)]
# launches that reach all of them, each followed by a residual pass at level 1: (config, features, camera).  On the 640x480
# pyramid the 320 x 1 geometry stages levels 0-1 in windows and level 2 whole; the 160 x 2 one gathers levels 0-2 from global
# memory.
SWEEP = [((-1, 0, -1), 100, "pinhole"), ((-1, 0, -1), 100, "atan"), ((4, 0, 0), 100, "pinhole"), ((4, 0, 0), 100, "atan"),
         ((2, 0, -1), 100, "pinhole"), ((8, 0, -1), 100, "pinhole"), ((1, 1, -1), 300, "pinhole"), ((1, 1, -1), 300, "atan"),
         ((1, 1, -1), 350, "pinhole"), ((1, 1, -1), 450, "pinhole"), ((1, 2, -1), 300, "pinhole"), ((1, 2, -1), 300, "atan"),
         ((-1, 0, -1), 700, "pinhole")]


def test_every_instantiation_and_staging_mode_is_reached(ctx, base, base_frames, cam_pairs):
    """Every instantiation launch_sia can dispatch to runs, nothing else does, and the three staging modes all occur."""
    atan = cam_pairs["atan"]
    atan_frames = (ctx.frame(atan["ref_pyr"]), ctx.frame(atan["cur_pyr"]))
    frames = {"pinhole": base_frames, "atan": atan_frames}
    records = []
    try:
        for cfg, n, kind in SWEEP:
            _configure(ctx, cfg)
            d = sc.subset(base if kind == "pinhole" else atan, n)
            sc.gpu_run(ctx, d, frames=frames[kind])
            records.append(ctx.sia_last_launch())
            ctx.sparse_residuals(*frames[kind], d["cam"], 1, synth.se3_identity(), d["px"], d["f"], d["pos"], d["has_point"],
                                 d["ref_pos"])
            records.append(ctx.sia_last_launch())
    finally:
        for f in atan_frames:
            f.destroy()
    reached = {}
    for r in records:
        reached.setdefault(_inst(r), set()).update(str(m) for m in r["stages"].values())
    print("\nresiduals CTAs threads FPT MINB general-camera upfront | staging modes reached")
    for inst in ALIGN_INSTANTIATIONS + RESIDUAL_INSTANTIATIONS:
        print(" ".join(f"{v:>4}" for v in inst), "|", ", ".join(sorted(reached.get(inst, {"NOT REACHED"}))))
    missing = [i for i in ALIGN_INSTANTIATIONS + RESIDUAL_INSTANTIATIONS if i not in reached]
    assert not missing, missing
    assert set(reached) <= set(ALIGN_INSTANTIATIONS + RESIDUAL_INSTANTIATIONS), set(reached) - set(ALIGN_INSTANTIATIONS + RESIDUAL_INSTANTIATIONS)
    modes = set().union(*reached.values())
    assert {"global", "image", "window"} <= modes, modes
