"""Cases of the two-view initialisation's KLT tracking (svo_b200_klt_*), shared by test_klt_pins.py (the oracle against
OpenCV's own calcOpticalFlowPyrLK, recorded) and test_klt_gpu.py (the kernel against both).

Images are built with integer arithmetic only (uniform noise, two box blurs, a fixed-point bilinear warp), so that every
machine builds the same bytes and the recorded reference outputs replay everywhere.  The current image samples the
previous one's texture at (x, y) + shift + shear * (y, x), shift and shear in 1/256 px.

What the cases exercise (branch -> case; the tests assert that each branch occurs):
  converged on eps, half-step   shift_640 / shift_752 / shift_644 (4, 4 and 5 levels), 350-400 points
  lost out of bounds at level 0 shift_640 (points seeded up to 10 px outside the image)
  iteration limit               iter_1 (max_iter 1: every level ends on it); far_flow (30 steps at level 0)
  eps 0                         iter_30_tight (only the half-step rule and the limit stop a level)
  out of bounds at a coarse     far_flow (an initial flow of (-90, 70) px: the coarsest window walks out and the finer
  level, an initial flow far off levels go on)
  lost on the eigenvalue        flat (a constant block, and a block of vertical stripes: no vertical gradient)
  first / last admissible       border (one level, next == prev: corner floor(x - 14.5) at exactly -30 and just below the
  column and row                level size, and one step beyond each)
A level-0 decision is never within MARGINS of flipping (test_klt_pins.py checks it on every case): the seeds below are
ones for which it holds."""
from __future__ import annotations

import numpy as np

from oracle import binding_klt

# seed of every case (chosen so that no decision is within MARGINS of flipping)
SEEDS = {"shift_640": 1, "shift_752": 2, "shift_644": 3, "iter_1": 4, "iter_30_tight": 5, "far_flow": 9, "flat": 8, "border": 8}
# |eps^2 - delta.delta|, |max(|sum_x|, |sum_y|) - 0.01|, |minEig - 1e-4|, |det - FLT_EPSILON|, |distance to a bound| (px)
MARGINS = (1e-10, 1e-6, 1e-6, 1e-3, 1e-3)
TOL_PX = 1e-3  # tracked points, oracle against OpenCV (observed: see the test's printout)


def texture(rng, w, h):
    """Smooth uint8 texture: uniform noise, two 7 x 7 box blurs, contrast stretched by integer arithmetic."""
    t = rng.integers(0, 256, (h + 16, w + 16), dtype=np.int64)
    for _ in range(2):
        c = np.cumsum(np.pad(t, ((1, 0), (1, 0))), 0).cumsum(1)
        t = (c[7:, 7:] - c[:-7, 7:] - c[7:, :-7] + c[:-7, :-7]) // 49
    t = t[: h + 4, : w + 4]
    lo, hi = int(t.min()), int(t.max())
    return ((t - lo) * 255 // max(hi - lo, 1)).astype(np.int64)


def warp(t, w, h, sx256, sy256, shear256):
    """cur(x, y) = t(x + 2 + sx + shear * y, y + 2 + sy - shear * x) in 1/256 px, bilinear in fixed point, edge-clamped."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.int64)
    X = (xx + 2) * 256 + sx256 + (shear256 * yy) // 256
    Y = (yy + 2) * 256 + sy256 - (shear256 * xx) // 256
    ix, iy = X >> 8, Y >> 8
    fx, fy = X & 255, Y & 255
    H, W = t.shape
    ix0, iy0 = np.clip(ix, 0, W - 1), np.clip(iy, 0, H - 1)
    ix1, iy1 = np.clip(ix + 1, 0, W - 1), np.clip(iy + 1, 0, H - 1)
    v = (t[iy0, ix0] * (256 - fx) * (256 - fy) + t[iy0, ix1] * fx * (256 - fy) + t[iy1, ix0] * (256 - fx) * fy
         + t[iy1, ix1] * fx * fy + 32768) >> 16
    return v.astype(np.uint8)


def _pair(rng, w, h, sx=7.3, sy=-4.2, shear=0.01):
    t = texture(rng, w, h)
    prev = warp(t, w, h, 0, 0, 0)
    cur = warp(t, w, h, int(round(sx * 256)), int(round(sy * 256)), int(round(shear * 256)))
    return prev, cur


def _pts(rng, n, w, h, outside=10.0):
    return (rng.random((n, 2)) * [w + 2 * outside, h + 2 * outside] - outside).astype(np.float32)


def case(name, seed=None):
    rng = np.random.default_rng(SEEDS[name] if seed is None else seed)
    k = dict(name=name, max_level=4, max_iter=30, eps=0.001, exact_bounds=False)
    if name in ("shift_640", "shift_752", "shift_644"):
        w, h = {"shift_640": (640, 480), "shift_752": (752, 480), "shift_644": (644, 484)}[name]
        prev, cur = _pair(rng, w, h)
        p0 = _pts(rng, 400 if name == "shift_640" else 350, w, h, 10.0 if name == "shift_640" else 0.0)
        k.update(prev=prev, cur=cur, prev_pts=p0, next_pts=p0.copy())
    elif name in ("iter_1", "iter_30_tight"):
        prev, cur = _pair(rng, 640, 480)
        p0 = _pts(rng, 200, 640, 480, 0.0)
        k.update(prev=prev, cur=cur, prev_pts=p0, next_pts=p0.copy())
        if name == "iter_1":
            k["max_iter"] = 1
        else:
            k["eps"] = 0.0
    elif name == "far_flow":
        prev, cur = _pair(rng, 640, 480, 3.0, -2.0, 0.0)
        p0 = _pts(rng, 300, 640, 480, 0.0)
        k.update(prev=prev, cur=cur, prev_pts=p0, next_pts=(p0 + np.float32([-90.0, 70.0])).astype(np.float32))
    elif name == "flat":
        prev, cur = _pair(rng, 640, 480, 1.5, 0.5, 0.0)
        prev = prev.copy()
        cur = cur.copy()
        for img in (prev, cur):
            img[40:240, 40:300] = 117                                                       # flat
            img[260:460, 340:600] = (60 + 40 * ((np.arange(260) // 6) % 2)).astype(np.uint8)  # vertical stripes: d/dy = 0
        p0 = np.concatenate([rng.random((60, 2)) * [160, 100] + [90, 90],     # flat block interior
                             rng.random((60, 2)) * [160, 100] + [390, 310],   # stripes interior
                             _pts(rng, 80, 640, 480, 0.0)]).astype(np.float32)
        k.update(prev=prev, cur=cur, prev_pts=p0, next_pts=p0.copy())
    elif name == "border":
        prev, _ = _pair(rng, 640, 480)
        w, h = 640, 480
        lo, hi = np.float32(-15.5), np.float32(w + 14.5)
        below = lo - np.float32(2.0 ** -19)  # two float32 steps: the corner -30 - 2^-19 floors to -31
        last_x = np.nextafter(hi, np.float32(-np.inf))
        last_y = np.nextafter(np.float32(h + 14.5), np.float32(-np.inf))
        ys = (rng.random(8) * h).astype(np.float32)
        xs = (rng.random(8) * w).astype(np.float32)
        p = [(lo, y) for y in ys] + [(last_x, y) for y in ys] + [(below, y) for y in ys[:2]] + [(hi, y) for y in ys[:2]]
        p += [(x, lo) for x in xs] + [(x, last_y) for x in xs] + [(x, below) for x in xs[:2]] + [(x, np.float32(h + 14.5)) for x in xs[:2]]
        p0 = np.array(p, np.float32)
        k.update(prev=prev, cur=prev, prev_pts=p0, next_pts=p0.copy(), max_level=0, exact_bounds=True)
    else:
        raise KeyError(name)
    return k


NAMES = list(SEEDS)


def oracle_run(k):
    return binding_klt.track(k["prev"], k["cur"], k["prev_pts"], k["next_pts"], k["max_level"], k["max_iter"], k["eps"])


def ref_run(ref, k):
    """OpenCV's calcOpticalFlowPyrLK on case k through the `ref` fixture (tests/ref_golden.py): its recorded outputs, or --
    when recording -- cv2 itself through oracle/binding_klt.py."""
    if ref.record_dir:
        ref.oracle = binding_klt
    return ref.call("klt_track", k["prev"], k["cur"], k["prev_pts"], k["next_pts"], k["max_level"], k["max_iter"], k["eps"])


# pyramid sizes pinned bit for bit: 4 levels, 4, 5 (the last level 41 x 31), 5 with odd sizes, 1 (cut at once)
PYR_SIZES = [(640, 480), (752, 480), (644, 484), (645, 485), (60, 40)]


def pyr_image(w, h, seed=11):
    return texture(np.random.default_rng(seed), w, h)[:h, :w].astype(np.uint8)


def ref_pyramid(ref, img):
    """buildOpticalFlowPyramid(img, (30, 30), 4, withDerivatives=True) through the `ref` fixture, kept as the level count and
    SHA-256 digests of every level and its derivatives."""
    from tests.ref_golden import sha256_u8

    if ref.record_dir:
        ref.oracle = binding_klt
    return ref.call("klt_pyramid", img, 4, keep=lambda r: dict(n_levels=r["n_levels"], images=[sha256_u8(a) for a in r["images"]],
                                                               derivs=[sha256_u8(a) for a in r["derivs"]]))


def margins_ok(k, o):
    """Level-0 decisions (and every decision feeding them) far enough from flipping: the mask of points that satisfy
    MARGINS at every level run.  Bounds margins are skipped on cases whose bounds tests see exact inputs only.  A window
    corner cannot leave a coarse level without leaving level 0 (levels halve, bounds and border scale with them), so an
    out-of-bounds coarse level always ends in a loss at level 0."""
    m = np.abs(o["margins"])  # N x levels x 5 (inf where a test did not run, NaN for levels not built)
    ok = np.ones(len(m), bool)
    for j, tol in enumerate(MARGINS):
        if j == 4 and k["exact_bounds"]:
            continue
        v = m[:, : o["n_levels"], j]
        if j == 3:  # the determinant test decides only where the eigenvalue test passes
            v = np.where(o["margins"][:, : o["n_levels"], 2] < -MARGINS[2], np.inf, v)
        ok &= np.all(v > tol, axis=1)
    return ok
