"""Edge cases of the two-view initialisation's KLT tracking (svo_b200_klt_*), shared by test_klt_edge_pins.py (the oracle
against OpenCV's own calcOpticalFlowPyrLK / buildOpticalFlowPyramid, recorded) and test_klt_edges_gpu.py (the kernels
against both).  Images come from tests/klt_cases.py's integer texture and warp, so the recorded outputs replay everywhere.

What the cases exercise (branch -> case; the tests assert that each branch occurs):
  non-finite coordinates        nonfinite: NaN, +-inf, +-3e9 and 1e9 in x alone or y alone of prev_pts or of the initial
                                guess, at warp positions 0, 3 and 4 of every 8 (first and last warp of a CTA, first of the
                                next) among ordinary points; each is lost out of bounds at every level, as OpenCV loses it
  images below the window       tiny_1x1, tiny_2x3 (every point lost on the eigenvalue: no gradient in x), tiny_17x29,
                                tiny_30x30, tiny_31x31: one level, bordered windows that reflect more than once
  coarsest level 31 / 32 wide   tiny_61x62, tiny_62x62 (2 levels, the last 31 x 31), tiny_63x63 (the last 32 x 32)
  odd sizes at every level      tiny_645x485 (5 levels: 645 x 485 ... 41 x 31)
  derivatives at full scale     binary: a 0/255 texture shifted by a fraction of a pixel (Scharr values reach +-4080)
  max_iter clamps               iter_0 and iter_neg3 (no step at any level), iter_1x (one step), iter_150 (klt_cases'
                                far_flow construction at 150: about 100 level runs end at exactly 100 steps)
  eps clamp                     eps_10 and eps_1e6 (both clamped to 10: identical)
  max_level vs levels built     level_0 .. level_3, level_7 (a 4-level pyramid: 7 runs the 4 levels that exist)
  pyramids of different depth   mixed_levels (prev built to max_level 4, next to 2: the tracker runs 3 levels),
                                same_handle (one pyramid as prev and next)
  level capacity                capacity (3968 x 3968: 8 levels, the last 31 x 31; tracked at max_level 7); CAPACITY_PYRAMIDS
                                (3968 x 3968 at max_level 7 and 10, 7936 x 7936 at 7: OpenCV's first 8 of 9 levels)
No decision of the oracle lies within klt_cases.MARGINS of flipping on these seeds (test_klt_edge_pins.py checks it)."""
from __future__ import annotations

import numpy as np

from oracle import binding_klt
from tests import klt_cases as kc

TINY = [(1, 1), (2, 3), (17, 29), (30, 30), (31, 31), (61, 62), (62, 62), (63, 63), (645, 485)]
NONFINITE = np.float32([np.nan, np.inf, -np.inf, 3e9, -3e9, 1e9])

SEEDS = {"nonfinite": 21, **{f"tiny_{w}x{h}": 30 + i for i, (w, h) in enumerate(TINY)}, "binary": 41, "iter_0": 1, "iter_neg3": 1,
         "iter_1x": 1, "iter_150": 15,"eps_10": 1, "eps_1e6": 1, **{f"level_{m}": 1 for m in (0, 1, 2, 3, 7)}, "mixed_levels": 1,
         "same_handle": 1, "capacity": 51}
NAMES = list(SEEDS)

# pyramids pinned bit for bit beside the tracked cases: (w, h, max_level)
EDGE_PYRAMIDS = [(w, h, 4) for w, h in TINY] + [(3968, 3968, 7), (3968, 3968, 10), (7936, 7936, 7)]


def _pair(rng, w, h, sx256, sy256, shear256):
    t = kc.texture(rng, w, h)
    return kc.warp(t, w, h, 0, 0, 0), kc.warp(t, w, h, sx256, sy256, shear256)


def _edge_pts(rng, w, h, n):
    """n points in [-10, size + 10], plus points on the first and last column and row."""
    p = kc._pts(rng, n, w, h, 10.0)
    ys, xs = rng.random(4) * h, rng.random(4) * w
    edge = [(0, y) for y in ys] + [(w - 1, y) for y in ys] + [(x, 0) for x in xs] + [(x, h - 1) for x in xs]
    return np.concatenate([p, np.float32(edge)]).astype(np.float32)


def nonfinite_rows():
    """(prev_pts row, guess row) pairs with one non-finite or huge coordinate, over an ordinary point (100.25, 200.75)."""
    rows = []
    for v in NONFINITE:
        for where in range(4):  # prev x, prev y, guess x, guess y
            p, g = np.float32([100.25, 200.75]), np.float32([100.25, 200.75])
            (p if where < 2 else g)[where % 2] = v
            rows.append((p, g))
    return rows


def special_slots(n_special):
    """Indices of the special rows: positions 0, 3 and 4 of every group of 8 points (4 warps per CTA)."""
    return np.array([8 * (i // 3) + (0, 3, 4)[i % 3] for i in range(n_special)])


def case(name, seed=None):
    rng = np.random.default_rng(SEEDS[name] if seed is None else seed)
    k = dict(name=name, max_level=4, max_iter=30, eps=0.001, exact_bounds=False, levels=None, same_handle=False)
    if name == "nonfinite":
        prev, cur = _pair(rng, 640, 480, 1869, -1075, 3)
        rows = nonfinite_rows()
        slots = special_slots(len(rows))
        n = int(slots[-1]) + 4
        plain = kc._pts(rng, n - len(rows), 640, 480, 0.0)
        p0, p1 = np.zeros((n, 2), np.float32), np.zeros((n, 2), np.float32)
        ordinary = np.setdiff1d(np.arange(n), slots)
        p0[ordinary], p1[ordinary] = plain, plain
        p0[slots], p1[slots] = [r[0] for r in rows], [r[1] for r in rows]
        k.update(prev=prev, cur=cur, prev_pts=p0, next_pts=p1, special=slots, ordinary=ordinary)
    elif name.startswith("tiny_"):
        w, h = (int(v) for v in name[5:].split("x"))
        prev, cur = _pair(rng, w, h, 333, -205, 2)
        p0 = _edge_pts(rng, w, h, 48)
        k.update(prev=prev, cur=cur, prev_pts=p0, next_pts=p0.copy())
    elif name == "binary":
        t = (kc.texture(rng, 640, 480) > 127).astype(np.int64) * 255
        prev, cur = kc.warp(t, 640, 480, 0, 0, 0), kc.warp(t, 640, 480, 141, -77, 0)
        p0 = kc._pts(rng, 200, 640, 480, 0.0)
        k.update(prev=prev, cur=cur, prev_pts=p0, next_pts=p0.copy())
    elif name == "iter_150":
        k = kc.case("far_flow", SEEDS[name] if seed is None else seed)
        if seed is None:  # three points whose decisions at 150 steps lie within MARGINS of flipping
            keep = np.setdiff1d(np.arange(len(k["prev_pts"])), [236, 258, 277])
            k.update(prev_pts=k["prev_pts"][keep], next_pts=k["next_pts"][keep])
        k.update(name=name, max_iter=150, levels=None, same_handle=False)
    elif name in ("iter_0", "iter_neg3", "iter_1x", "eps_10", "eps_1e6") or name.startswith("level_") or name in ("mixed_levels", "same_handle"):
        b = kc.case("shift_640", seed)
        k.update(prev=b["prev"], cur=b["cur"], prev_pts=b["prev_pts"][:120], next_pts=b["next_pts"][:120])
        if name.startswith("iter_"):
            k["max_iter"] = {"iter_0": 0, "iter_neg3": -3, "iter_1x": 1}[name]
        elif name.startswith("eps_"):
            k["eps"] = {"eps_10": 10.0, "eps_1e6": 1e6}[name]
        elif name.startswith("level_"):
            k["max_level"] = int(name[6:])
        elif name == "mixed_levels":
            k.update(max_level=2, levels=(4, 2))  # the kernel: prev built to 4, next to 2, option max_level 4
        else:
            k.update(cur=b["prev"], same_handle=True)
    elif name == "capacity":
        prev, cur = _pair(rng, 3968, 3968, 1587, 1203, 1)
        p0 = kc._pts(rng, 48, 3968, 3968, 0.0)
        k.update(prev=prev, cur=cur, prev_pts=p0, next_pts=p0.copy(), max_level=7)
    else:
        raise KeyError(name)
    return k


def pyramid_image(w, h):
    """The image of a pinned pyramid: klt_cases.pyr_image, and for 7936 x 7936 the 3968 x 3968 one mirrored into 2 x 2."""
    if (w, h) == (7936, 7936):
        t = kc.pyr_image(3968, 3968)
        return np.block([[t, t[:, ::-1]], [t[::-1], t[::-1, ::-1]]])
    return kc.pyr_image(w, h)


def ref_pyramid(ref, img, max_level):
    """buildOpticalFlowPyramid(img, (30, 30), max_level, withDerivatives=True) through the `ref` fixture, kept as the level
    count and SHA-256 digests of every level and its derivatives."""
    from tests.ref_golden import sha256_u8

    if ref.record_dir:
        ref.oracle = binding_klt
    return ref.call("klt_pyramid", img, max_level, keep=lambda r: dict(n_levels=r["n_levels"], images=[sha256_u8(a) for a in r["images"]],
                                                                       derivs=[sha256_u8(a) for a in r["derivs"]]))


def same_nonfinite(a, b):
    """Where b is not finite, a holds the same value (NaN for NaN, the same infinity)."""
    m = ~np.isfinite(b)
    return bool(np.all(np.isnan(a[m]) == np.isnan(b[m])) and np.all((a[m] == b[m]) | np.isnan(b[m])))


def bits_equal(a, b):
    """Bit for bit, NaN compared as 'both NaN' (any payload)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a) & np.isnan(b)
    return a.shape == b.shape and bool(np.all(nan | (a.view(np.uint32) == b.view(np.uint32))))
