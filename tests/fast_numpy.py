"""An independent numpy statement of FastDetector::detect (svo/src/feature_detection.cpp:66-115) for small images.

Written from the definitions, not from the oracle or the kernel:
- the FAST-10 segment test on the 16-pixel Bresenham ring of radius 3: at least 10 contiguous ring pixels all brighter
  than centre + b, or all darker than centre - b, with a 3-pixel border;
- the corner score as the `fast` library computes it: a bisection of the threshold over [b, 255] that keeps bmin a
  threshold the pixel passes and returns bmin once bmax - bmin <= 1;
- 3x3 non-maximum suppression on the dense score map (a detected 8-neighbour with a larger score suppresses, or with a
  larger-or-equal one when ties suppress);
- vk::shiTomasiScore in float64 (8x8 box of central differences, smaller eigenvalue);
- the per-cell arg-max over (level, row, column) scan order with a strictly-greater update.

Because the Shi-Tomasi score is computed in float64 here and in float32 by the implementations under test, a cell whose
two best scores (or whose best score and the threshold) are within float32 rounding of each other cannot be decided;
`detect` reports those cells as ambiguous."""
from __future__ import annotations

import numpy as np

RING = [(0, -3), (1, -3), (2, -2), (3, -1), (3, 0), (3, 1), (2, 2), (1, 3),
        (0, 3), (-1, 3), (-2, 2), (-3, 1), (-3, 0), (-3, -1), (-2, -2), (-1, -3)]


def _ring(img: np.ndarray, ys: np.ndarray, xs: np.ndarray) -> np.ndarray:
    """(16, n) ring intensities of the pixels (ys, xs), as int."""
    return np.stack([img[ys + dy, xs + dx].astype(np.int64) for dx, dy in RING])


def _passes(ring: np.ndarray, c: np.ndarray, t) -> np.ndarray:
    """Segment test at threshold t (scalar or per pixel): 10 contiguous ring pixels > c + t or < c - t."""
    out = np.zeros(ring.shape[1], bool)
    for hit in (ring > c + t, ring < c - t):
        for s in range(16):
            arc = np.ones(ring.shape[1], bool)
            for j in range(10):
                arc &= hit[(s + j) % 16]
            out |= arc
    return out


def fast_scores(img: np.ndarray, b: int) -> np.ndarray:
    """Dense map of FAST-10 corner scores at threshold b; -1 where the pixel is not a corner."""
    h, w = img.shape
    score = np.full((h, w), -1, np.int64)
    if h < 7 or w < 7:
        return score
    ys, xs = np.mgrid[3:h - 3, 3:w - 3]
    ys, xs = ys.ravel(), xs.ravel()
    ring, c = _ring(img, ys, xs), img[ys, xs].astype(np.int64)
    det = _passes(ring, c, b)
    ys, xs, ring, c = ys[det], xs[det], ring[:, det], c[det]
    bmin, bmax = np.full(len(ys), b), np.full(len(ys), 255)
    t = (bmin + bmax) // 2
    done = np.zeros(len(ys), bool)
    while not done.all():
        ok = _passes(ring, c, t)
        bmin = np.where(~done & ok, t, bmin)
        bmax = np.where(~done & ~ok, t, bmax)
        done |= (bmin == bmax - 1) | (bmin == bmax)
        t = (bmin + bmax) // 2
    score[ys, xs] = bmin
    return score


def nonmax(score: np.ndarray, ties_suppress: bool) -> np.ndarray:
    """Boolean map of the corners that survive 3x3 non-maximum suppression."""
    h, w = score.shape
    pad = np.full((h + 2, w + 2), -1, np.int64)
    pad[1:-1, 1:-1] = score
    keep = score >= 0
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dx == 0 and dy == 0:
                continue
            n = pad[1 + dy:1 + dy + h, 1 + dx:1 + dx + w]
            keep &= ~((n >= 0) & ((n >= score) if ties_suppress else (n > score)))
    return keep


def shi_tomasi(img: np.ndarray, u: int, v: int) -> tuple[float, float]:
    """(score, trace of the structure tensor); float32 arithmetic can move the score by a few ulps of the trace."""
    h, w = img.shape
    if u - 4 < 1 or u + 4 >= w - 1 or v - 4 < 1 or v + 4 >= h - 1:
        return 0.0, 0.0
    I = img.astype(np.float64)
    dx = I[v - 4:v + 4, u - 3:u + 5] - I[v - 4:v + 4, u - 5:u + 3]
    dy = I[v - 3:v + 5, u - 4:u + 4] - I[v - 5:v + 3, u - 4:u + 4]
    xx, yy, xy = (dx * dx).sum() / 128.0, (dy * dy).sum() / 128.0, (dx * dy).sum() / 128.0
    return 0.5 * (xx + yy - np.sqrt((xx + yy) ** 2 - 4.0 * (xx * yy - xy * xy))), xx + yy


def detect(pyr, n_pyr_levels: int, cell_size: int, detection_threshold: float, b: int = 20, ties_suppress: bool = False,
           grid_occupancy=None, rtol: float = 2e-6) -> dict:
    """Corners in cell order: dict(x, y, level, score (float64), fast_score, trace, cell) and `ambiguous`, the cells whose
    outcome float32 rounding can decide either way: two values closer than rtol * (|best| + largest trace)."""
    h0, w0 = pyr[0].shape
    ncols, nrows = -(-w0 // cell_size), -(-h0 // cell_size)
    thr = float(np.float32(detection_threshold))
    cands: dict[int, list] = {}
    for L in range(n_pyr_levels):
        img = pyr[L]
        sc = fast_scores(img, b)
        keep = nonmax(sc, ties_suppress)
        for y, x in zip(*np.nonzero(keep)):  # row-major: the scan order
            k = (int(y) << L) // cell_size * ncols + (int(x) << L) // cell_size
            if grid_occupancy is not None and grid_occupancy[k]:
                continue
            st, tr = shi_tomasi(img, int(x), int(y))
            cands.setdefault(k, []).append((st, int(x) << L, int(y) << L, L, int(sc[y, x]), tr))
    out = dict(x=[], y=[], level=[], score=[], fast_score=[], trace=[], cell=[])
    ambiguous = []
    for k in range(ncols * nrows):
        best, top = None, thr  # Corner(0, 0, detection_threshold, 0, 0.0f), then the first strictly greater score wins
        for c in cands.get(k, []):
            if c[0] > top:
                best, top = c, c[0]
        tol = rtol * (abs(top) + max([c[5] for c in cands.get(k, [])], default=0.0))
        if any(v != top and abs(v - top) <= tol for v in [thr] + [c[0] for c in cands.get(k, [])]):
            ambiguous.append(k)
        if best is not None and best[0] > detection_threshold:
            for key, v in zip(("score", "x", "y", "level", "fast_score", "trace"), best):
                out[key].append(v)
            out["cell"].append(k)
    res = {k: np.array(v) for k, v in out.items()}
    res["ambiguous"] = np.array(ambiguous, np.int64)
    res["n_cells"] = ncols * nrows
    return res


def cells_of(x, y, w0: int, cell_size: int) -> np.ndarray:
    return (np.asarray(y) // cell_size) * (-(-w0 // cell_size)) + np.asarray(x) // cell_size


def agree(ref: dict, got: dict, w0: int, cell_size: int) -> int:
    """Assert that `got` (oracle or kernel output) equals the numpy reference on every cell that is not ambiguous;
    returns the number of cells compared."""
    amb = set(ref["ambiguous"].tolist())
    gc = cells_of(got["x"], got["y"], w0, cell_size)
    g = {int(k): (int(a), int(b_), int(c)) for k, a, b_, c in zip(gc, got["x"], got["y"], got["level"])}
    r = {int(k): (int(a), int(b_), int(c)) for k, a, b_, c in zip(ref["cell"], ref["x"], ref["y"], ref["level"])}
    n = 0
    for k in range(ref["n_cells"]):
        if k in amb:
            continue
        assert g.get(k) == r.get(k), (k, g.get(k), r.get(k))
        n += 1
    gs = {int(k): float(s) for k, s in zip(gc, got["score"])} if "score" in got else {}
    for k, s, tr in zip(ref["cell"], ref["score"], ref["trace"]):
        if int(k) in gs and int(k) not in amb:
            assert abs(gs[int(k)] - s) <= 2e-6 * (s + tr), (k, gs[int(k)], s)
    return n


def images(seed: int = 1, w: int = 64, h: int = 48, n_levels: int = 3) -> dict:
    """Small test frames: a rendered view, uniform noise, a 0/255 checkerboard of 5-px squares (every corner scores 254,
    so the suppression meets ties everywhere) and low-contrast noise in 100..102 (most corners score 0 at b = 0)."""
    from rpg_svo_b200 import synth

    rng = np.random.default_rng(seed)
    cb = (((np.indices((h, w)) // 5).sum(0) % 2) * 255).astype(np.uint8)
    return dict(render=synth.make_two_view(seed + 2, width=w, height=h, n_levels=n_levels)["ref_pyr"],
                noise=synth.build_pyramid(rng.integers(0, 256, (h, w), dtype=np.uint8), n_levels),
                checker=synth.build_pyramid(cb, n_levels),
                low_contrast=synth.build_pyramid(rng.integers(100, 103, (h, w), dtype=np.uint8), n_levels))
