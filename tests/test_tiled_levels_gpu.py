"""GPU: every way of filling a frame leaves a block-tiled copy of each pyramid level that equals the row-major level byte
for byte (zero outside the level), and the throughput geometry, which gathers its footprints from that copy, computes the
same residuals as the one-feature-per-thread geometry, which gathers them row by row, with features on the first and last
admissible column and row of levels whose sizes are not multiples of 4."""
import numpy as np
import pytest
import torch

from rpg_svo_b200 import capi, synth
from tests import sia_cases as sc

pytestmark = pytest.mark.gpu

# (width, height, levels): multiples of 16 (the pool's streaming level-0 kernel), of 4 only, of neither, widths that are
# multiples of 16 over an odd height and a height of 4k + 2 (the streaming kernel's lone last row, partial last block-row),
# one-level frames, top levels under 4 px wide, pyramids deeper than the fused pool kernel's five levels, a two-level pool
SIZES = [(640, 480, 5), (644, 484, 5), (645, 485, 5), (640, 481, 5), (640, 482, 5), (640, 480, 1), (645, 485, 1), (70, 50, 6),
         (640, 480, 7), (640, 480, 2), (13, 9, 2)]


def _untile(t, w, h):
    """[ceil(h/4), ceil(w/4), 4, 4] blocks -> the padded image and the level as stored in it"""
    full = t.transpose(0, 2, 1, 3).reshape(t.shape[0] * 4, t.shape[1] * 4)
    return full, full[:h, :w]


def _check(fr, w0, h0, levels):
    for l in range(levels):
        w, h = w0 >> l, h0 >> l
        full, lvl = _untile(fr.download_level_tiled(l), w, h)
        assert np.array_equal(lvl, fr.download_level(l)), f"level {l}"
        assert not full[h:].any() and not full[:, w:].any(), f"padding of level {l}"


def _images(w, h, n, seed):
    return np.random.default_rng(seed).integers(1, 256, (n, h, w), dtype=np.uint8)  # no zero pixel: padding stays visible


@pytest.mark.parametrize("w,h,levels", SIZES, ids=[f"{w}x{h}x{l}" for w, h, l in SIZES])
def test_frame_upload_all_levels_and_level0_only(ctx, w, h, levels):
    img = _images(w, h, 1, w * h)[0]
    a = ctx.frame(synth.build_pyramid(img, levels))
    b = ctx.frame_from_level0(img, levels)
    try:
        _check(a, w, h, levels)
        _check(b, w, h, levels)
    finally:
        a.destroy(); b.destroy()


@pytest.mark.parametrize("w,h,levels", SIZES, ids=[f"{w}x{h}x{l}" for w, h, l in SIZES])
def test_upload_device(ctx, w, h, levels):
    img = _images(w, h, 1, w + h)[0]
    dev = torch.from_numpy(img).cuda(ctx.device)
    torch.cuda.synchronize(ctx.device)
    fr = capi.Frame(ctx, w, h, levels)
    try:
        fr.upload_device(dev.data_ptr())
        ctx.synchronize()
        assert np.array_equal(fr.download_level(0), img)
        _check(fr, w, h, levels)
    finally:
        fr.destroy()


@pytest.mark.parametrize("w,h,levels", SIZES, ids=[f"{w}x{h}x{l}" for w, h, l in SIZES])
def test_pool_upload_first_and_last_frame_and_a_window(ctx, w, h, levels):
    imgs = _images(w, h, 5, 3 * w + h)
    pool = capi.FramePool(ctx, w, h, levels, 5)
    try:
        pool.upload_array(imgs)
        for i in (0, 4):
            assert np.array_equal(pool.frames[i].download_level(0), imgs[i])
            _check(pool.frames[i], w, h, levels)
        pool.upload_array(imgs[3:0:-1], first=1)  # a window inside the pool
        for i in (1, 2, 3):
            assert np.array_equal(pool.frames[i].download_level(0), imgs[4 - i])
            _check(pool.frames[i], w, h, levels)
    finally:
        pool.destroy()


def _edge_case(w, h, seed):
    """The border case of sia_cases at w x h, plus features exactly on the first and last column and row whose 7x7 reference
    footprint fits at level 0 (integer and half-pixel positions)."""
    d = sc.border_pair(seed, w, h, 160)
    px = d["px"].copy()
    edge = []
    for lo_x, hi_x in ((3.0, w - 4.0), (3.5, w - 3.5)):
        for lo_y, hi_y in ((3.0, h - 4.0), (3.5, h - 3.5)):
            edge += [(lo_x, lo_y), (hi_x, lo_y), (lo_x, hi_y), (hi_x, hi_y), (lo_x, h / 2), (hi_x, h / 2), (w / 2, lo_y),
                     (w / 2, hi_y)]
    px[-len(edge):] = edge
    f = d["cam"].cam2world(px)
    pos = synth.intersect(synth.Plane.tilted(), d["T_ref_w"], f)
    hp = d["has_point"].copy()
    hp[-len(edge):] = 1
    return dict(d, px=np.ascontiguousarray(px), f=np.ascontiguousarray(f), pos=np.ascontiguousarray(pos), has_point=hp), len(edge)


@pytest.mark.parametrize("size", [(645, 485), (643, 482), (646, 487)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_throughput_geometry_gathers_edge_footprints_like_the_row_major_path(ctx, oracle, size):
    w, h = size
    d, n_edge = _edge_case(w, h, w + 7 * h)
    ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
    try:
        for pose, T in (("identity", synth.se3_identity()), ("motion", d["T_gt"])):
            for level in range(5):
                out = {}
                for fpt in (2, 1):
                    ctx.sia_config(1, fpt)
                    out[fpt] = ctx.sparse_residuals(ref, cur, d["cam"], level, T, d["px"], d["f"], d["pos"], d["has_point"],
                                                    d["ref_pos"])
                    L = ctx.sia_last_launch()
                    assert (L["threads"], L["features_per_thread"]) == ((160, 2) if fpt == 2 else (320, 1)), L
                    if fpt == 2 and level <= 2:  # the levels the throughput geometry gathers from the tiled copy
                        assert L["stages"][level] == "global", (level, L)
                o = oracle.sparse_residuals(d["ref_pyr"][level], d["cur_pyr"][level], level, d["cam"], T, d["px"], d["f"],
                                            d["pos"], d["has_point"], d["ref_pos"])
                sc.assert_residual_parity(out[2], o)
                v = o["visible"].astype(bool)  # the patch cache of invisible features is not written
                for k in ("visible", "in_image"):
                    assert np.array_equal(out[2][k], out[1][k]), (pose, level, k)
                # the same pixel values, the same arithmetic: bit-equal patches and residuals (NaN where not evaluated)
                assert np.array_equal(out[2]["ref_patch"][v], out[1]["ref_patch"][v]), (pose, level)
                assert np.array_equal(out[2]["residuals"], out[1]["residuals"], equal_nan=True), (pose, level)
                if pose == "identity" and level == 0:
                    assert o["visible"][-n_edge:].all() and o["in_image"][-n_edge:].sum() >= n_edge // 2
        ctx.sia_config(1, 2)
        g = sc.gpu_run(ctx, d, frames=(ref, cur))
        assert ctx.sia_last_launch()["threads"] == 160
        o = sc.oracle_run(oracle, d)
        assert np.array_equal(g["visible"], o["visible"]) and g["n_tracked"] == o["n_tracked"]
        assert synth.pose_error(g["T"], o["T"])[0] < 1e-4
    finally:
        ctx.sia_config(-1, 0)
        ref.destroy(); cur.destroy()
