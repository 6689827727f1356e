"""Edge cases of the robust alignment kernel (sia_robust_kernel), shared by test_sia_robust_edge_pins.py (oracle vs the
compiled reference, and the MAD scale vs an exact numpy median) and test_sia_robust_edges_gpu.py (kernel vs oracle).

The kernel deals feature i to thread i % 256, slot i // 256 (up to four slots), tests the reference and the current patch
against the border itself, keeps a set-only visibility mask across levels and selects the MAD median with a four-sweep
radix select.  The cases aim at each of those:
  slots_<N>_<w>          N in SLOT_COUNTS features of sc.base_pair() (or of another scene, see SEEDS), has_point cleared
                         at the robust slot edges (ROBUST_EDGES)
  slots_1024_live_tukey  1024 features with those slots live
  odd_<W>x<H>            sc.odd_pair's border case at sc.ODD_SIZES: odd level sizes, motion that carries patches out of the
                         current image
  border_640             sc.border_pair at 640x480, 400 features
  admissible_<w>         features on the first / last admissible column and row of the coarsest level (ui - 3 == 0,
                         ui + 3 == W_l - 1) and one pixel beyond
  levels_<max>_<min>     level ranges of a five-level pyramid; depth3_2_0 / depth6_5_0 pyramids of three and six levels
  t0_perturbed           a start 2 mm / 0.1 degree off the ground-truth pose; t0_converged a start from the oracle's own result
  coarse_empty_iters_<n> every feature 24-47 px from the border: level 4 has no patch, levels 3..0 do (n_iter 0 and 30)
  ties_<k>_<w>           hand-built pyramids whose every level holds k grey values: the |res| have many ties, and with two
                         values more than half of them are exactly 0 (the MAD scale is 0)"""
import functools

import numpy as np

from oracle import binding_robust
from rpg_svo_b200 import synth
from tests import sia_cases as sc
from tests import sia_robust_cases as rc

SLOT_COUNTS = (255, 256, 257, 511, 512, 513, 767, 768, 769, 1023, 1024)
ROBUST_EDGES = (0, 255, 256, 511, 512, 767, 768, 1023)  # first / last feature of each of the kernel's four slots
LEVEL_RANGES = ((4, 2), (3, 1), (2, 0), (0, 0), (2, 2))

# The compiled reference builds its own pyramid from level 0; these cases upload hand-built levels, so they are compared
# with the oracle and numpy only.  coarse_empty_*: the reference takes the median of no errors at level 4 (undefined in
# vk::getMedian), as in sia_robust_cases.NO_REF.
NO_REF = {"coarse_empty_iters_0", "coarse_empty_iters_30", "ties_2_tukey", "ties_2_huber", "ties_4_tukey", "ties_4_huber"}
# n_iter 0: the loop never writes H_, whose content the reference leaves undefined
NO_H = {"coarse_empty_iters_0"}


def robust_subset(d, n, clear_edges=True, order=0):
    """n features of `d` with has_point cleared at ROBUST_EDGES: the first n, or (order > 0) the first n of a permutation
    drawn with that seed."""
    if order:
        d = dict(d)
        perm = np.random.default_rng(order).permutation(len(d["px"]))
        for key in ("px", "f", "pos", "has_point"):
            d[key] = np.ascontiguousarray(d[key][perm])
    s = sc.subset(d, n, clear_edges=False)
    if clear_edges:
        s["has_point"][[e for e in ROBUST_EDGES if e < n]] = 0
    return s


def with_features(d, px):
    """`d` with the features at `px`, their bearings and 3D points recomputed on the scene's plane."""
    q = dict(d)
    q["px"] = np.ascontiguousarray(px, np.float64)
    q["f"] = np.ascontiguousarray(d["cam"].cam2world(q["px"]))
    q["pos"] = np.ascontiguousarray(synth.intersect(synth.Plane.tilted(), d["T_ref_w"], q["f"]))
    q["has_point"] = np.ones(len(px), np.uint8)
    return q


def admissible_pair(seed, level=4):
    """150 interior features plus 48 on the first and last admissible column and row of `level` (floor(u_l) - 3 == 0,
    floor(u_l) + 3 == W_l - 1, rows alike) and 48 one pixel of that level beyond them."""
    d = synth.make_frame_pair(seed, n_feat=150)
    rng = np.random.default_rng(seed)
    W, H, s = d["cam"].width >> level, d["cam"].height >> level, float(1 << level)
    extra = []
    for cols, rows in (((3, W - 4), None), (None, (3, H - 4)), ((2, W - 3), None), (None, (2, H - 3))):
        for k in range(24):
            frac = rng.uniform(0.05, 0.95, 2)
            if cols is not None:
                u = cols[k % 2] + frac[0]
                v = rng.uniform(4.0, H - 5.0)
            else:
                u = rng.uniform(4.0, W - 5.0)
                v = rows[k % 2] + frac[1]
            extra.append((u * s, v * s))
    return with_features(d, np.concatenate([d["px"], np.array(extra)]))


def strip_pair(seed, n=240):
    """Every feature 24-47 px from the nearest border (and at least 48 px from the others): at level 4 (1/16) no reference
    patch fits, at level 3 (1/8) every one does."""
    d = synth.make_frame_pair(seed, n_feat=10)
    rng = np.random.default_rng(seed)
    W, H = d["cam"].width, d["cam"].height
    side = rng.integers(0, 4, n)
    dist = rng.uniform(24.0, 47.0, n)
    along_x, along_y = rng.uniform(48.0, W - 49.0, n), rng.uniform(48.0, H - 49.0, n)
    x = np.where(side == 0, dist, np.where(side == 1, W - 1 - dist, along_x))
    y = np.where(side == 2, dist, np.where(side == 3, H - 1 - dist, along_y))
    return with_features(d, np.stack([x, y], axis=1))


def quantised(d, k):
    """Both pyramids of `d` with every level mapped to k grey values (at the level's own quantiles), uploaded as they are:
    not what halfSample would build from level 0."""
    vals = np.linspace(40, 215, k).round().astype(np.uint8)
    q = dict(d)
    for key in ("ref_pyr", "cur_pyr"):
        out = []
        for img in d[key]:
            edges = np.quantile(img, np.linspace(0, 1, k + 1)[1:-1])
            out.append(np.ascontiguousarray(vals[np.digitize(img, edges)]))
        q[key] = out
    return q


# The seed of each case: (scene, feature order) for the slot, level-range and tie cases (_scene, robust_subset's `order`),
# the scene for the others.  Chosen so that no Gauss-Newton decision of the oracle's run is
# within MARGIN of flipping (sc.decision_margin), which test_sia_robust_edge_pins.py asserts.
SEEDS = {"slots_511_tukey": (0, 9), "slots_511_huber": (0, 9), "slots_512_tukey": (0, 9), "slots_512_huber": (0, 9),
         "slots_513_tukey": (0, 9), "slots_513_huber": (0, 9), "slots_767_tukey": (0, 10), "slots_767_huber": (0, 10),
         "slots_768_tukey": (0, 10), "slots_768_huber": (0, 10), "slots_769_tukey": (0, 10),
         "slots_769_huber": (0, 10), "slots_1023_tukey": (2, 0), "slots_1023_huber": (0, 12),
         "slots_1024_tukey": (2, 0), "slots_1024_huber": (0, 12), "slots_1024_live_tukey": (2, 0), "odd_644x484": 9,
         "odd_160x120": 5, "levels_2_0": (0, 1), "levels_2_2": (0, 1), "depth3_2_0": 1, "depth6_5_0": 7,
         "t0_perturbed": 12, "t0_converged": 2, "coarse_empty_iters_30": 1}
# sc.decision_margin of every case is at least this: about 9x the largest relative chi2 difference between the kernel's and the
# oracle's trace (5.8e-6, NVIDIA H100 80GB HBM3), so that the kernel's trace can be compared with the oracle's exactly.
MARGIN = 5e-5


@functools.lru_cache(maxsize=None)
def _scene(seed):
    """sc.base_pair() (seed 0), or a 640x480 scene of 1100 features drawn with `seed`, every feature with a 3D point."""
    if seed == 0:
        return sc.base_pair()
    d = synth.make_frame_pair(seed, n_feat=1100)
    d["has_point"][:] = 1
    return d


def build(name, seed):
    """Case `name` built with `seed` (see SEEDS)."""
    def case(p, weight, n_iter=30, max_level=4, min_level=0, T0=None):
        return dict(name=name, p=p, weight=rc.WEIGHTS[weight], n_iter=n_iter, max_level=max_level, min_level=min_level,
                    T0=synth.se3_identity() if T0 is None else T0)

    parts = name.split("_")
    if parts[0] == "slots":
        live = parts[2] == "live"
        return case(robust_subset(_scene(seed[0]), int(parts[1]), clear_edges=not live, order=seed[1]), parts[-1])
    if parts[0] == "odd":
        w, h = (int(v) for v in parts[1].split("x"))
        return case(sc.border_pair(seed, w, h, 180), "tukey")  # sc.odd_pair with a seed of its own
    if name == "border_640":
        return case(sc.border_pair(seed, 640, 480, 400), "huber")
    if parts[0] == "admissible":
        return case(admissible_pair(seed), parts[1])
    if parts[0] == "levels":
        return case(robust_subset(_scene(seed[0]), 300, order=seed[1]), "tukey", max_level=int(parts[1]), min_level=int(parts[2]))
    if name == "depth3_2_0":
        return case(synth.make_frame_pair(seed, n_feat=300, n_levels=3), "tukey", max_level=2)
    if name == "depth6_5_0":
        return case(synth.make_frame_pair(seed, n_feat=300, n_levels=6), "huber", max_level=5)
    if name == "t0_perturbed":
        gt = synth.make_frame_pair(seed, n_feat=250)
        return case(gt, "tukey", T0=synth.se3_mul(synth.se3_exp(np.array([2e-3, -1e-3, 1.5e-3, 1.7e-3, -1e-3, 1e-3])),
                                                  gt["T_cur_ref_gt"]))
    if name == "t0_converged":
        gt = synth.make_frame_pair(seed, n_feat=250)
        return case(gt, "tukey", T0=oracle_run(case(gt, "tukey"))["T"])
    if parts[0] == "coarse":
        return case(strip_pair(seed), "tukey", n_iter=int(parts[3]))
    if parts[0] == "ties":
        # Huber on four grey values takes many tiny steps: five iterations per level end it before they near a tie
        return case(quantised(robust_subset(_scene(seed[0]), 400, order=seed[1]), int(parts[1])), parts[2],
                    n_iter=5 if name == "ties_4_huber" else 30)
    raise KeyError(name)


NAMES = ([f"slots_{n}_{w}" for n in SLOT_COUNTS for w in ("tukey", "huber")] + ["slots_1024_live_tukey"] +
         [f"odd_{w}x{h}" for w, h in sc.ODD_SIZES] + ["border_640", "admissible_tukey", "admissible_huber"] +
         [f"levels_{mx}_{mn}" for mx, mn in LEVEL_RANGES] + ["depth3_2_0", "depth6_5_0", "t0_perturbed", "t0_converged"] +
         [f"coarse_empty_iters_{n}" for n in (0, 30)] + [f"ties_{v}_{w}" for v in (2, 4) for w in ("tukey", "huber")])
DEFAULT_SEEDS = {"border_640": 5, "admissible_tukey": 57, "admissible_huber": 57, "depth3_2_0": 37, "depth6_5_0": 38,
                 "t0_perturbed": 11, "t0_converged": 11, "coarse_empty_iters_0": 73, "coarse_empty_iters_30": 73}


def cases():
    return [build(n, seed_of(n)) for n in NAMES]


def seed_of(name):
    if name in SEEDS or name in DEFAULT_SEEDS:
        return SEEDS.get(name, DEFAULT_SEEDS.get(name))
    if name.startswith("odd_"):
        return sc.ODD_SEEDS[tuple(int(v) for v in name[4:].split("x"))]
    return (0, 0)


_CASES = None


def all_cases():
    global _CASES
    if _CASES is None:
        _CASES = cases()
    return _CASES


def case(name):
    return next(k for k in all_cases() if k["name"] == name)


def names():
    return [k["name"] for k in all_cases()]


def oracle_run(k, n_iter=None):
    p = k["p"]
    return binding_robust.sparse_img_align_robust(p["ref_pyr"], p["cur_pyr"], p["cam"], k["T0"], p["px"], p["f"], p["pos"],
                                                  p["has_point"], p["ref_pos"], k["max_level"], k["min_level"], k["weight"],
                                                  k["n_iter"] if n_iter is None else n_iter)


def ref_run(ref, k):
    """The compiled reference on case k through the `ref` fixture, started at T0 (T_cur_w = T0 T_ref_w)."""
    p = k["p"]
    if ref.record_dir:
        ref.oracle = binding_robust
    return ref.call("sparse_img_align_robust", p["ref_pyr"][0], p["cur_pyr"][0], p["n_levels"], p["cam"], p["T_ref_w"],
                    synth.se3_mul(k["T0"], p["T_ref_w"]), p["px"], p["f"], p["pos"], p["has_point"], k["max_level"],
                    k["min_level"], k["weight"], k["n_iter"])


def median_levels(k):
    """The levels whose scale is computed at the initial pose T0: the first level, and every level when n_iter is 0."""
    return list(range(k["max_level"], k["min_level"] - 1, -1)) if k["n_iter"] == 0 else [k["max_level"]]


def numpy_scales(oracle, k):
    """{level: 1.48 * the upper median of |res|} for median_levels(k), from the oracle's residual pass at T0 with the
    visibility the coarser levels left (vk::getMedian: nth_element at floor(n / 2)); None where no patch is in the image."""
    p = k["p"]
    want = set(median_levels(k))
    vis = np.zeros(len(p["px"]), np.uint8)
    out = {}
    for level in range(k["max_level"], min(want) - 1, -1):
        r = oracle.sparse_residuals(p["ref_pyr"][level], p["cur_pyr"][level], level, p["cam"], k["T0"], p["px"], p["f"],
                                    p["pos"], p["has_point"], p["ref_pos"], visible_in=vis)
        vis = r["visible"]
        if level in want:
            a = np.abs(r["residuals"][r["in_image"].astype(bool)].astype(np.float32)).ravel()
            out[level] = np.float32(1.48) * np.partition(a, a.size // 2)[a.size // 2] if a.size else None
    return out
