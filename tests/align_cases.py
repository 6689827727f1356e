"""Feature-aligner (align2D / align1D) and direct-matcher (Matcher::findMatchDirect) cases at their border, degenerate,
multi-reference and batch edges, shared by the GPU edge tests (test_align_edges_gpu.py) and the CPU pins of the same cases
against the compiled reference (test_align_pins.py)."""
from functools import lru_cache

import numpy as np

from rpg_svo_b200 import synth

F32 = np.float32


def f32_below(x) -> float:
    """The float32 value just below float32(x), as a double."""
    return float(np.nextafter(F32(x), F32(-np.inf)))


def f32_above(x) -> float:
    return float(np.nextafter(F32(x), F32(np.inf)))


@lru_cache(maxsize=16)
def rendered_pyramid(width: int, height: int, n_levels: int, tex_seed: int = 7) -> tuple:
    """A frame of the tilted textured plane seen from synth.base_pose()."""
    cam = synth.camera_for(width, height)
    img = synth.render(cam, synth.base_pose(), synth.Plane.tilted(), synth.make_texture(tex_seed))
    return tuple(synth.build_pyramid(img, n_levels))


def template(img: np.ndarray, u: float, v: float):
    """(patch_with_border[100], patch[64]) of img around the sub-pixel position (u, v), which must lie >= 5 px inside."""
    p = synth.patch_with_border(img, np.array([u, v]))
    return p.ravel(), p[1:9, 1:9].ravel()


def _problem_set(name, pyr, rows, n_iter, **extra):
    """rows: (level, pwb, patch, (u, v), (dir_x, dir_y))."""
    return dict(name=name, pyr=list(pyr), n_iter=n_iter, level=np.array([r[0] for r in rows], np.int32),
                pwb=np.stack([r[1] for r in rows]).astype(np.uint8), patch=np.stack([r[2] for r in rows]).astype(np.uint8),
                px=np.array([r[3] for r in rows], np.float64), dir=np.array([r[4] for r in rows], np.float32), **extra)


def _interior_template(rng, pyr, level, u, v, spread=1.5):
    """A template taken near (u, v) (clamped 6 px inside the level; from level 0 if the level is too small), so the
    alignment starting at (u, v) has something to pull towards."""
    img = pyr[level]
    h, w = img.shape
    if w < 13 or h < 13:
        img = pyr[0]
        h, w = img.shape
    tu = float(np.clip(u + rng.uniform(-spread, spread), 6, w - 7)) if np.isfinite(u) else w / 2 + 0.3
    tv = float(np.clip(v + rng.uniform(-spread, spread), 6, h - 7)) if np.isfinite(v) else h / 2 + 0.3
    return template(img, tu, tv)


def _unit(rng):
    d = rng.normal(size=2)
    return d / np.linalg.norm(d)


def _well_posed(rng, pyr, n, levels=None, margin=8.0, off=1.5):
    """n ordinary problems: the true position uniformly inside `margin`, the start within `off` px of it."""
    rows = []
    levels = range(len(pyr)) if levels is None else levels
    levels = [l for l in levels if min(pyr[l].shape) > 2 * margin + 2]
    for i in range(n):
        L = levels[i % len(levels)]
        h, w = pyr[L].shape
        t = np.array([rng.uniform(margin, w - margin), rng.uniform(margin, h - margin)])
        pwb, patch = template(pyr[L], *t)
        rows.append((L, pwb, patch, tuple(t - rng.uniform(-off, off, 2)), tuple(_unit(rng))))
    return rows


# ---- align2D / align1D ------------------------------------------------------------------------------------------------------
def border_case(n_iter):
    """Starts on the border test's float edges at every level of a 5-level pyramid: 4, the float32 just below 4, cols-4 and
    rows-4, the float32 just below those, and doubles just below 4 / cols-4 that round up to them in float32.  u = 4 gives
    the first admissible footprint (column 0), u = float32 below cols-4 the last (column cols-1); likewise for rows."""
    rng = np.random.default_rng(100 + n_iter)
    pyr = rendered_pyramid(640, 480, 5)
    rows = []
    for L, img in enumerate(pyr):
        h, w = img.shape
        edges = lambda n: [4.0, f32_below(4), 4.0 - 1e-12, float(n - 4), f32_below(n - 4), (n - 4) - 1e-12, 4.5, n - 4.5]
        mid_u, mid_v = w / 2 + 0.37, h / 2 + 0.61
        for u in edges(w):
            rows.append((L, *_interior_template(rng, pyr, L, u, mid_v), (u, mid_v), tuple(_unit(rng))))
        for v in edges(h):
            rows.append((L, *_interior_template(rng, pyr, L, mid_u, v), (mid_u, v), tuple(_unit(rng))))
        for u in (4.0, f32_below(w - 4)):  # the two extreme footprints in both coordinates at once
            for v in (4.0, f32_below(h - 4)):
                rows.append((L, *_interior_template(rng, pyr, L, u, v), (u, v), tuple(_unit(rng))))
    return _problem_set(f"border_n{n_iter}", pyr, rows, n_iter)


NEVER_ITERATE = [np.nan, np.inf, -np.inf, 1e9, -1e9, f32_below(1e9), f32_above(1e9), f32_below(-1e9), 3e9, -3e9, -0.5, -3.0,
                 -1e-30, -4.5, -2.1e9]


def never_iterate_case():
    """Starts the border test rejects before any step: NaN, +-inf, +-1e9 and the float32 values beside it, +-3e9 (beyond
    int32: x86's conversion gives INT_MIN, the kernel's |u| < 1e9 guard a negative index) and negative pixels; in u, in v
    and in both.  The output is (double)(float)px."""
    rng = np.random.default_rng(5)
    pyr = rendered_pyramid(640, 480, 5)
    rows = []
    for k, bad in enumerate(NEVER_ITERATE):
        L = k % 5
        h, w = pyr[L].shape
        good_u, good_v = w / 2 + 0.25, h / 2 + 0.75
        for px in ((bad, good_v), (good_u, bad), (bad, bad)):
            rows.append((L, *_interior_template(rng, pyr, L, good_u, good_v), px, tuple(_unit(rng))))
    return _problem_set("never_iterate", pyr, rows, 10)


def n_iter_case(n_iter):
    rng = np.random.default_rng(200)  # the same problems for every n_iter
    pyr = rendered_pyramid(640, 480, 5)
    return _problem_set(f"n_iter_{n_iter}", pyr, _well_posed(rng, pyr, 150), n_iter)


def drift_case():
    """Starts 1-2 px inside the border with the true position outside it, so the border test breaks after >= 1 step.  The
    current image is the interior of a larger render, which supplies the templates of positions outside the image."""
    o0 = 32
    cam = synth.camera_for(640, 480)
    big_cam = synth.Camera(cam.fx, cam.fy, cam.cx + o0, cam.cy + o0, 640 + 2 * o0, 480 + 2 * o0)
    big = synth.build_pyramid(synth.render(big_cam, synth.base_pose(), synth.Plane.tilted(), synth.make_texture(7)), 4)
    pyr = [np.ascontiguousarray(b[o0 >> L:(o0 >> L) + (480 >> L), o0 >> L:(o0 >> L) + (640 >> L)]) for L, b in enumerate(big)]
    rng = np.random.default_rng(7)
    rows = []
    for L in range(4):
        h, w = pyr[L].shape
        o = o0 >> L
        for side in range(4):
            for _ in range(6):
                out, start = rng.uniform(1.0, 2.5), 4 + rng.uniform(1.0, 2.0)
                a = rng.uniform(10, (h if side < 2 else w) - 10)  # along the side
                if side == 0:
                    t, s = (out, a), (start, a)
                elif side == 1:
                    t, s = (w - 1 - out, a), (w - 1 - start, a)
                elif side == 2:
                    t, s = (a, out), (a, start)
                else:
                    t, s = (a, h - 1 - out), (a, h - 1 - start)
                pwb, patch = template(big[L], t[0] + o, t[1] + o)
                d = np.subtract(t, s)
                rows.append((L, pwb, patch, s, tuple(d / np.linalg.norm(d))))
    return _problem_set("drift_out", pyr, rows, 10)


def _patch(kind):
    y, x = np.mgrid[0:10, 0:10]
    if kind == "constant":
        p = np.full((10, 10), 128)
    elif kind == "const_along_y":  # varies in x only: d/dy = 0
        p = 20 * x + 7
    elif kind == "bright_pixel":
        p = np.zeros((10, 10)); p[5, 5] = 255
    elif kind == "checker1":  # period 2: the central differences are all 0
        p = 255 * ((x + y) % 2)
    elif kind == "checker2":  # 2-px squares
        p = 255 * ((x // 2 + y // 2) % 2)
    else:
        raise ValueError(kind)
    p = p.astype(np.uint8)
    return p.ravel(), p[1:9, 1:9].ravel()


def singular_case():
    """Templates whose H is singular or extreme: a constant patch (rank 1: px becomes NaN, converged 0), a patch constant
    along y (2-D singular; 1-D with dir (0, 1) gives h_inv = +inf), a single bright pixel, 0/255 checkerboards."""
    rng = np.random.default_rng(9)
    pyr = rendered_pyramid(640, 480, 5)
    rows = []
    for kind in ("constant", "const_along_y", "bright_pixel", "checker1", "checker2"):
        pwb, patch = _patch(kind)
        for k in range(8):
            L = k % 4
            h, w = pyr[L].shape
            px = (rng.uniform(10, w - 10), rng.uniform(10, h - 10))
            d = (0.0, 1.0) if k % 2 == 0 else tuple(_unit(rng))
            rows.append((L, pwb, patch, px, d))
    return _problem_set("singular", pyr, rows, 10)


DIRECTIONS = [(0.0, 0.0), (3.0, 4.0), (0.3, -0.1), (np.nan, 1.0), (1.0, np.nan), (1.0, 0.0), (0.0, 1.0), (-1.0, 0.0),
              (0.0, -1.0)]


def directions_case():
    """1-D directions (0, 0), non-unit, with a NaN component and along each axis, on ordinary problems (2-D runs on the
    same problems ignore them)."""
    rng = np.random.default_rng(11)
    pyr = rendered_pyramid(640, 480, 5)
    base = _well_posed(rng, pyr, 30 * len(DIRECTIONS), off=2.5)
    rows = [(L, pwb, patch, px, DIRECTIONS[i % len(DIRECTIONS)]) for i, (L, pwb, patch, px, _) in enumerate(base)]
    return _problem_set("directions", pyr, rows, 10)


def geometry_cases():
    """Odd sizes (644x484: a 161-px level 2; a 645-px width), a pyramid whose top level is narrower than 9 px (no start
    passes the border test there), and a 1-level frame."""
    out = []
    for (w, h, nl) in ((644, 484, 5), (645, 485, 4), (96, 72, 5), (640, 480, 1)):
        rng = np.random.default_rng(w + h + nl)
        cam = synth.camera_for(w, h)
        pyr = synth.build_pyramid(synth.render(cam, synth.base_pose(), synth.Plane.tilted(), synth.make_texture(7)), nl)
        rows = _well_posed(rng, pyr, 80, margin=7.0)
        for L in range(nl):  # the level edges and the middle of every level, small ones included
            lh, lw = pyr[L].shape
            for px in ((f32_below(lw - 4), lh / 2), (lw / 2, f32_below(lh - 4)), (4.0, 4.0), (lw / 2 + 0.3, lh / 2 + 0.3)):
                rows.append((L, *_interior_template(rng, pyr, L, *px), px, tuple(_unit(rng))))
        out.append(_problem_set(f"geometry_{w}x{h}x{nl}", pyr, rows, 10))
    return out


def pool_case():
    """Three frames of one geometry for a FramePool; problems on the first and the last (the pool builds the pyramids)."""
    cam = synth.camera_for(640, 480)
    imgs = []
    for k in range(3):
        T = synth.se3_mul(synth.se3_exp(np.array([0.05 * k, -0.03 * k, 0.02 * k, 0.01 * k, 0, -0.01 * k])), synth.base_pose())
        imgs.append(synth.render(cam, T, synth.Plane.tilted(), synth.make_texture(7)))
    out = []
    for k in (0, 2):
        pyr = synth.build_pyramid(imgs[k], 5)
        rng = np.random.default_rng(300 + k)
        out.append(_problem_set(f"pool_frame{k}", pyr, _well_posed(rng, pyr, 120), 10, pool_index=k))
    return np.stack(imgs), out


def align_cases():
    """Every problem set of the align2D / align1D edge tests except the batch shapes, in a fixed order."""
    return ([border_case(1), border_case(10), never_iterate_case()] + [n_iter_case(n) for n in (-1, 0, 1, 2, 10, 100)]
            + [drift_case(), singular_case(), directions_case()] + geometry_cases() + pool_case()[1])


def batch_problems(M, seed=400):
    """M well-posed problems over every level of one 5-level frame (mixed in the launch order), templates at integer
    positions (a plain 10x10 crop)."""
    rng = np.random.default_rng(seed + M)
    pyr = rendered_pyramid(640, 480, 5)
    level = rng.integers(0, 5, M).astype(np.int32)
    pwb = np.zeros((M, 100), np.uint8)
    px = np.zeros((M, 2))
    for L in range(5):
        idx = np.flatnonzero(level == L)
        h, w = pyr[L].shape
        tu, tv = rng.integers(8, w - 8, len(idx)), rng.integers(8, h - 8, len(idx))
        y, x = np.mgrid[-5:5, -5:5]
        pwb[idx] = pyr[L][tv[:, None, None] + y, tu[:, None, None] + x].reshape(len(idx), 100)
        px[idx] = np.stack([tu, tv], 1) + rng.uniform(-1.5, 1.5, (len(idx), 2))
    patch = pwb.reshape(M, 10, 10)[:, 1:9, 1:9].reshape(M, 64).copy()
    d = rng.normal(size=(M, 2))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return dict(name=f"batch{M}", pyr=list(pyr), n_iter=10, level=level, pwb=pwb, patch=patch, px=px, dir=d.astype(np.float32))


BATCH_SIZES = (1, 3, 4, 5, 4097)
BIG_BATCH = 65537


def sample_rows(M, n=96, warps_per_cta=4):
    """Indices covering the first and the last CTA of a launch of M problems (4 warps each) and a spread between."""
    first = np.arange(min(M, 2 * warps_per_cta))
    last = np.arange(max(0, M - 2 * warps_per_cta - 1), M)
    mid = np.linspace(0, M - 1, n).astype(int)
    return np.unique(np.concatenate([first, mid, last]))


def run_ref_align(ref, c, rows=None):
    """The compiled reference's align2D and align1D on the problems `rows` of c (all by default), in a fixed call order
    (recorded by test_align_pins.py, replayed by the GPU tests).  Returns (conv2, px2, conv1, px1, h1)."""
    rows = range(len(c["level"])) if rows is None else rows
    out = [[], [], [], [], []]
    for i in rows:
        img = c["pyr"][int(c["level"][i])]
        ok, p = ref.align2d(img, c["pwb"][i], c["patch"][i], int(c["n_iter"]), c["px"][i])
        ok1, p1, h = ref.align1d(img, c["dir"][i], c["pwb"][i], c["patch"][i], int(c["n_iter"]), c["px"][i])
        for k, x in enumerate((ok, p, ok1, p1, h)):
            out[k].append(x)
    return (np.array(out[0], bool), np.array(out[1]).reshape(-1, 2), np.array(out[2], bool), np.array(out[3]).reshape(-1, 2),
            np.array(out[4], np.float64))


def run_oracle_align(oracle, c, rows=None):
    """The oracle on the problems `rows` of c: dict of conv2, px2, exit2, it2, conv1, px1, h1, exit1, it1."""
    rows = range(len(c["level"])) if rows is None else rows
    o = {k: [] for k in ("conv2", "px2", "exit2", "it2", "conv1", "px1", "h1", "exit1", "it1")}
    for i in rows:
        img = c["pyr"][int(c["level"][i])]
        ok, p, ex, it = oracle.align2d(img, c["pwb"][i], c["patch"][i], int(c["n_iter"]), c["px"][i], want_exit=True)
        ok1, p1, h, ex1, it1 = oracle.align1d(img, c["dir"][i], c["pwb"][i], c["patch"][i], int(c["n_iter"]), c["px"][i],
                                              want_exit=True)
        for k, x in zip(o, (ok, p, ex, it, ok1, p1, h, ex1, it1)):
            o[k].append(x)
    o = {k: np.array(v) for k, v in o.items()}
    o["px2"], o["px1"] = o["px2"].reshape(-1, 2), o["px1"].reshape(-1, 2)
    return o


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def same_bits(a, b) -> bool:
    """Bit for bit, except that any NaN equals any NaN: the GPU's canonical NaN (0x7fffffff as a float) and x86's default
    NaN (0xffc00000) differ in sign and payload, and neither carries information."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all((bits(a) == bits(b)) | (np.isnan(a) & np.isnan(b))))


# ---- Matcher::findMatchDirect ------------------------------------------------------------------------------------------------
FRONTO = synth.Plane(np.array([0.0, 0.0, 1.0]), 2.0, np.array([1.0, 0.0, 0.0]), np.array([0.0, 1.0, 0.0]))


def rot_z(deg):
    a = np.deg2rad(deg)
    T = np.zeros((3, 4))
    T[:, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
    return T


def _pose(R=None, t=(0, 0, 0)):
    T = np.zeros((3, 4))
    T[:, :3] = np.eye(3) if R is None else R
    T[:, 3] = t
    return T


def _render_pyr(cam, T, n_levels, plane=FRONTO):
    return synth.build_pyramid(synth.render(cam, T, plane, synth.make_texture(7)), n_levels)


def _cands(cam, T_ref_w, T_cur_w, px, level, plane=FRONTO, ftr_type=None, grad=None, rng=None, off=1.0, ref_index=None):
    """Candidate arrays for reference pixels px (level-0) observing the plane; the guess is the true reprojection +- off."""
    rng = np.random.default_rng(0) if rng is None else rng
    n = len(px)
    f = cam.cam2world(px)
    pos = synth.intersect(plane, T_ref_w, f)
    pc = pos @ T_cur_w[:, :3].T + T_cur_w[:, 3]
    guess = cam.world2cam(pc) + rng.uniform(-off, off, (n, 2))
    if ftr_type is None:
        ftr_type = (np.arange(n) % 3 == 2).astype(np.int32)
    if grad is None:
        a = rng.uniform(0, 2 * np.pi, n)
        grad = np.stack([np.cos(a), np.sin(a)], 1)
    return dict(ref_index=np.zeros(n, np.int32) if ref_index is None else np.asarray(ref_index, np.int32), ref_px=np.asarray(px, float),
                ref_f=f, ref_level=np.asarray(level, np.int32), ftr_type=np.asarray(ftr_type, np.int32), ref_grad=np.asarray(grad, float),
                point_pos=pos, px_cur=guess)


def _match_case(name, cam, ref_pyrs, ref_T, cur_pyr, T_cur_w, cands, max_search_level=2, align_max_iter=10):
    return dict(name=name, cam=cam, ref_pyrs=ref_pyrs, ref_T=ref_T, cur_pyr=cur_pyr, T_cur_w=T_cur_w,
                max_search_level=max_search_level, align_max_iter=align_max_iter, M=len(cands["ref_index"]), **cands)


def _cat(parts):
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def multi_ref_case(n_ref):
    """n_ref reference frames with different poses, images and pyramid depths; candidates of every frame in one launch,
    ref_index interleaved and unsorted."""
    cam = synth.camera_for(752, 480)
    rng = np.random.default_rng(40 + n_ref)
    plane = synth.Plane.tilted()
    depths = [5, 3, 4, 5][:n_ref]
    T0 = synth.base_pose()
    ref_T, ref_pyrs, parts = [], [], []
    T_cur_w = synth.se3_mul(synth.se3_exp(np.array([0.05, -0.04, 0.02, 0.01, -0.01, 0.02])), T0)
    for r in range(n_ref):
        T = synth.se3_mul(synth.se3_exp(np.concatenate([rng.uniform(-0.12, 0.12, 3), np.deg2rad(rng.uniform(-3, 3, 3))])), T0)
        ref_T.append(T)
        ref_pyrs.append(synth.build_pyramid(synth.render(cam, T, plane, synth.make_texture(7 + r)), depths[r]))
        n = 40
        level = rng.integers(0, min(3, depths[r]), n)
        px = np.stack([rng.uniform(60, 692, n), rng.uniform(60, 420, n)], 1)
        px = np.round(px / (1 << level)[:, None]) * (1 << level)[:, None]
        parts.append(_cands(cam, T, T_cur_w, px, level, plane=plane, rng=rng, ref_index=np.full(n, r)))
    c = _cat(parts)
    perm = rng.permutation(len(c["ref_index"]))
    c = {k: v[perm] for k, v in c.items()}
    cur_pyr = synth.build_pyramid(synth.render(cam, T_cur_w, plane, synth.make_texture(7)), 5)
    return _match_case(f"multi_ref{n_ref}", cam, ref_pyrs, ref_T, cur_pyr, T_cur_w, c)


def in_frame_case(cam=None, name="in_frame"):
    """Reference pixels whose (int)px / (1 << level) is 5, 6, w_L - 7 and w_L - 6 (and the same in y) at levels 0-4, on a
    644-px-wide camera (not a multiple of 16), plus px in (-1, 0), which truncates to 0."""
    cam = synth.camera_for(644, 484) if cam is None else cam
    rng = np.random.default_rng(50)
    T_ref_w = _pose()
    T_cur_w = synth.se3_mul(synth.se3_exp(np.array([0.01, -0.01, 0.0, 0.0, 0.0, 0.003])), T_ref_w)
    px, lv = [], []
    for L in range(5):
        s = 1 << L
        wL, hL = cam.width // s, cam.height // s
        for xi in (5, 6, wL - 7, wL - 6):
            px.append((xi * s + rng.uniform(0, s), hL // 2 * s + 0.5)); lv.append(L)
        for yi in (5, 6, hL - 7, hL - 6):
            px.append((wL // 2 * s + 0.5, yi * s + rng.uniform(0, s))); lv.append(L)
        px.append((-rng.uniform(0.01, 0.99), hL // 2 * s)); lv.append(L)
        px.append((wL // 2 * s, -0.5)); lv.append(L)
    px = np.array(px)
    c = _cands(cam, T_ref_w, T_cur_w, px, lv, rng=rng)
    return _match_case(name, cam, [_render_pyr(cam, T_ref_w, 5)], [T_ref_w], _render_pyr(cam, T_cur_w, 5), T_cur_w, c,
                       max_search_level=4)


def warp_border_cases():
    """Reference features 6-10 level pixels from the reference border whose warped 10x10 samples leave the image:
    (a) a 20 degree roll about the optical axis (a pure rotation, zoom 1) at reference levels 1-3, so search levels 1-3;
    (b) a 180 degree roll with the current camera 1.25x farther (A = -0.8 I, inverse -1.25 I exactly in float32) at level 0,
    where features at x = cols - 7.25 put a sample exactly on qx = cols - 1 (zero-filled: the test is qx >= cols - 1), and
    likewise for rows."""
    cam = synth.camera_for(640, 480)
    rng = np.random.default_rng(60)
    T_ref_w = _pose()
    ref_pyr = _render_pyr(cam, T_ref_w, 5)
    out = []
    T_cur_w = rot_z(20)
    px, lv = [], []
    for L in (1, 2, 3):
        s = 1 << L
        wL, hL = 640 // s, 480 // s
        for d in (6, 7, 8, 10):
            for side in range(4):
                a = rng.uniform(0.3, 0.7)
                x, y = [(d, a * hL), (wL - 1 - d, a * hL), (a * wL, d), (a * wL, hL - 1 - d)][side]
                px.append((x * s + rng.uniform(0, s), y * s + rng.uniform(0, s))); lv.append(L)
    c = _cands(cam, T_ref_w, T_cur_w, np.array(px), lv, rng=rng)
    out.append(_match_case("warp_border_roll20", cam, [ref_pyr], [T_ref_w], _render_pyr(cam, T_cur_w, 5), T_cur_w, c,
                           max_search_level=4))
    T_cur_w = _pose(np.diag([-1.0, -1.0, 1.0]), (0, 0, 0.5))
    px = [(640 - 7.25, y) for y in (100.5, 240.25, 380.75)] + [(x, 480 - 7.25) for x in (100.5, 320.25, 540.75)]
    px += [(6.0 + k / 8, 200.5) for k in range(8)] + [(300.5, 6.0 + k / 8) for k in range(8)]
    px += [(640 - 7.0 - k / 8, 150.5) for k in range(8)]
    c = _cands(cam, T_ref_w, T_cur_w, np.array(px), np.zeros(len(px), int), rng=rng)
    out.append(_match_case("warp_border_roll180", cam, [ref_pyr], [T_ref_w], _render_pyr(cam, T_cur_w, 5), T_cur_w, c,
                           max_search_level=2))
    return out


def search_level_cases(cam=None, tag=""):
    """The current camera 1x, 2x, 4x and 8x closer to a fronto-parallel plane than the reference (D = k^2 4^level), with
    max_search_level 0, 1, 2, 4 and negative values (which act as 0); corners and edgelets, some with a zero gradient."""
    cam = synth.camera_for(640, 480) if cam is None else cam
    T_ref_w = _pose()
    ref_pyr = _render_pyr(cam, T_ref_w, 5)
    out = []
    for k in (1, 2, 4, 8):
        T_cur_w = _pose(t=(0, 0, -(2.0 - 2.0 / k)))
        cur_pyr = _render_pyr(cam, T_cur_w, 5)
        rng = np.random.default_rng(70 + k)
        n = 24
        level = np.arange(n) % 3
        r = 0.35 * min(cam.width, cam.height) / k
        px = np.stack([cam.cx + rng.uniform(-r, r, n), cam.cy + rng.uniform(-r, r, n)], 1)
        px = np.round(px / (1 << level)[:, None]) * (1 << level)[:, None]
        ftr_type = (np.arange(n) % 2).astype(np.int32)
        c = _cands(cam, T_ref_w, T_cur_w, px, level, ftr_type=ftr_type, rng=rng)
        c["ref_grad"][::5] = 0.0  # edgelets (odd rows) among these have no gradient: dir = 0/0
        for ms in (0, 1, 2, 4, -1, -3):
            out.append(_match_case(f"search_level{tag}_k{k}_max{ms}", cam, [ref_pyr], [T_ref_w], cur_pyr, T_cur_w, c,
                                   max_search_level=ms))
    return out


def degenerate_cases(cam=None, tag=""):
    """A point at the reference camera centre (depth 0: A = 0, the warp is skipped, the zero patch gives NaN), a point
    behind the current camera, guesses outside the current image and NaN guesses, a pure rotation, and align_max_iter
    0 and 1."""
    cam = synth.camera_for(640, 480) if cam is None else cam
    T_ref_w = _pose()
    ref_pyr = _render_pyr(cam, T_ref_w, 5)
    rng = np.random.default_rng(80)
    T_fwd = _pose(t=(0.02, -0.01, -0.5))  # 0.5 m forward
    cur_pyr = _render_pyr(cam, T_fwd, 5)
    n = 30
    px = np.stack([rng.uniform(150, cam.width - 150, n), rng.uniform(120, cam.height - 120, n)], 1)
    level = np.arange(n) % 3
    px = np.round(px / (1 << level)[:, None]) * (1 << level)[:, None]
    c = _cands(cam, T_ref_w, T_fwd, px, level, rng=rng)
    c["point_pos"][0:6] = 0.0                                     # the reference camera centre
    c["point_pos"][6:12] = c["ref_f"][6:12] * 0.2                 # 0.2 m ahead of the reference, 0.3 m behind the current
    c["px_cur"][12:15] = [(-40.0, 100.0), (cam.width + 30.0, 50.0), (200.0, -1e6)]
    c["px_cur"][15:17] = [(np.nan, 100.0), (np.nan, np.nan)]
    out = [_match_case(f"degenerate{tag}", cam, [ref_pyr], [T_ref_w], cur_pyr, T_fwd, c)]
    T_rot = synth.se3_exp(np.array([0, 0, 0, 0.03, -0.02, 0.05]))
    c = _cands(cam, T_ref_w, T_rot, px, level, rng=rng)
    out.append(_match_case(f"pure_rotation{tag}", cam, [ref_pyr], [T_ref_w], _render_pyr(cam, T_rot, 5), T_rot, c))
    T_cur = _pose(t=(0.03, -0.02, -0.1))
    c = _cands(cam, T_ref_w, T_cur, px, level, rng=rng, off=1.5)
    cur_pyr = _render_pyr(cam, T_cur, 5)
    for it in (0, 1):
        out.append(_match_case(f"max_iter{it}{tag}", cam, [ref_pyr], [T_ref_w], cur_pyr, T_cur, c, align_max_iter=it))
    return out


def atan_camera():
    return synth.atan_camera(640, 480, 0.509326, 0.796651, 0.5, 0.5, 0.9320)


def match_cases():
    """Every single-reference matcher case in a fixed order (the multi-reference ones are separate)."""
    cam = atan_camera()
    return ([in_frame_case()] + warp_border_cases() + search_level_cases() + degenerate_cases()
            + [in_frame_case(cam, "in_frame_atan")] + search_level_cases(cam, "_atan")[:12] + degenerate_cases(cam, "_atan"))


def ref_pose_pair(c, r=0):
    T_cur_ref = synth.se3_mul(c["T_cur_w"], synth.se3_inv(c["ref_T"][r]))
    return T_cur_ref, synth.se3_inv(c["ref_T"][r])[:, 3]


def run_oracle_match(oracle, c, rows=None):
    """The oracle per candidate: dict of success, search_level, px_cur, A_cur_ref [n, 2, 2], h_inv."""
    rows = range(c["M"]) if rows is None else rows
    out = {k: [] for k in ("success", "search_level", "px_cur", "A_cur_ref", "h_inv")}
    for i in rows:
        r = int(c["ref_index"][i])
        T_cur_ref, ref_pos = ref_pose_pair(c, r)
        depth = float(np.linalg.norm(ref_pos - c["point_pos"][i]))
        o = oracle.find_match_direct(c["ref_pyrs"][r], c["cur_pyr"], c["cam"], T_cur_ref, c["ref_px"][i], c["ref_f"][i],
                                     int(c["ref_level"][i]), int(c["ftr_type"][i]), c["ref_grad"][i], depth,
                                     int(c["max_search_level"]), int(c["align_max_iter"]), c["px_cur"][i])
        for k in out:
            out[k].append(o[k])
    return {k: np.array(v) for k, v in out.items()}


def run_ref_match(ref, c, rows=None):
    """The compiled reference's Matcher::findMatchDirect per candidate (its own frames and pyramids from level 0; the
    search-level cap is Config::nPyrLevels() - 1)."""
    rows = range(c["M"]) if rows is None else rows
    out = {k: [] for k in ("success", "search_level", "px_cur", "A_cur_ref", "h_inv")}
    nl = len(c["cur_pyr"])
    for i in rows:
        r = int(c["ref_index"][i])
        o = ref.matcher(0, c["ref_pyrs"][r][0], c["cur_pyr"][0], nl, c["cam"], c["ref_T"][r], c["T_cur_w"], c["ref_px"][i],
                        c["ref_f"][i], int(c["ref_level"][i]), int(c["ftr_type"][i]), c["ref_grad"][i], c["point_pos"][i],
                        px_cur=c["px_cur"][i], n_pyr_levels=int(c["max_search_level"]) + 1)
        for k in out:
            out[k].append(o[k])
    return {k: np.array(v) for k, v in out.items()}


def close_view(c):
    """Point::getCloseViewObs's test (point.cpp: the cosine between the directions from the point to the current and to
    the reference camera >= 0.5): the reference's findMatchDirect returns false before the matcher where it fails (the
    kernel's caller makes that choice on the host)."""
    cur_pos = synth.se3_inv(c["T_cur_w"])[:, 3]
    ok = np.zeros(c["M"], bool)
    for i in range(c["M"]):
        a = cur_pos - c["point_pos"][i]
        b = synth.se3_inv(c["ref_T"][int(c["ref_index"][i])])[:, 3] - c["point_pos"][i]
        na, nb = np.linalg.norm(a), np.linalg.norm(b)
        ok[i] = na > 0 and nb > 0 and a @ b / (na * nb) >= 0.5
    return ok


def in_frame(c, i):
    """isInFrame(px.cast<int>() / (1 << level), halfpatch + 2, level) (matcher.cpp:143-145), with C's truncating casts."""
    L, w, h = int(c["ref_level"][i]), c["cam"].width, c["cam"].height
    xi, yi = (int(np.trunc(x)) // (1 << L) if x >= 0 else -(int(np.trunc(-x)) // (1 << L)) for x in c["ref_px"][i])
    return 6 <= xi < w // (1 << L) - 6 and 6 <= yi < h // (1 << L) - 6


def numpy_warp(c, i):
    """float64 numpy statement of warp::getWarpMatrixAffine (matcher.cpp:33-55) and warp::getBestSearchLevel (:57-70)
    with synth.Camera, independent of the oracle.  Returns (A [2, 2], search_level)."""
    cam, r = c["cam"], int(c["ref_index"][i])
    T_cur_ref, ref_pos = ref_pose_pair(c, r)
    depth = np.linalg.norm(ref_pos - c["point_pos"][i])
    L = int(c["ref_level"][i])
    px = c["ref_px"][i]
    xyz = c["ref_f"][i] * depth
    du = cam.cam2world(px + [5.0 * (1 << L), 0.0])
    dv = cam.cam2world(px + [0.0, 5.0 * (1 << L)])
    du, dv = du * (xyz[2] / du[2]), dv * (xyz[2] / dv[2])
    proj = lambda p: cam.world2cam(T_cur_ref[:, :3] @ p + T_cur_ref[:, 3])
    p0, pu, pv = proj(xyz), proj(du), proj(dv)
    A = np.array([[pu[0] - p0[0], pv[0] - p0[0]], [pu[1] - p0[1], pv[1] - p0[1]]]) / 5.0
    D, s = A[0, 0] * A[1, 1] - A[1, 0] * A[0, 1], 0
    while D > 3.0 and s < int(c["max_search_level"]):
        s, D = s + 1, D * 0.25
    return A, s
