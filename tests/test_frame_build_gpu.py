"""GPU: a single frame is a frame pool of one, and every way of filling a frame -- host levels 0..n_given-1 of a single
frame or of a pool's frame, level 0 from device memory, a window of a pool -- builds the same pyramid with the same kernels:
row-major levels equal to vk::halfSample's (both rounding rules) and block-tiled copies equal to those levels, zero outside
them.  Pyramids deeper than the fused kernel's five levels are built by further passes of it over the whole window, so the
number of launches of an upload does not depend on the number of frames."""
import numpy as np
import pytest
import torch

from rpg_svo_b200 import capi, synth

pytestmark = pytest.mark.gpu

# widths that are multiples of 16 (the streaming level-0 kernel) and that are not, odd heights, top levels under 4 px,
# pyramids of 6, 7 and 8 levels (two fused passes), a two-level pyramid whose level 1 the streaming kernel builds alone
SIZES = [(640, 480, 8), (1920, 1080, 8), (70, 50, 6), (752, 480, 5), (645, 485, 7), (640, 481, 6), (96, 48, 2), (13, 9, 2)]
IDS = [f"{w}x{h}x{l}" for w, h, l in SIZES]


@pytest.fixture(params=[synth.PYR_X86, synth.PYR_SCALAR], ids=["x86-sse2-rule", "scalar-rule"])
def rule(request, ctx):
    ctx.set_pyramid_rule(request.param)
    yield request.param
    ctx.set_pyramid_rule(synth.PYR_X86)


def _images(w, h, n, seed):
    return np.random.default_rng(seed).integers(1, 256, (n, h, w), dtype=np.uint8)  # no zero pixel: padding stays visible


def _check(fr, pyr):
    for l, ref in enumerate(pyr):
        h, w = ref.shape
        assert np.array_equal(fr.download_level(l), ref), f"level {l}"
        t = fr.download_level_tiled(l)
        full = t.transpose(0, 2, 1, 3).reshape(t.shape[0] * 4, t.shape[1] * 4)
        assert np.array_equal(full[:h, :w], ref), f"tiled level {l}"
        assert not full[h:].any() and not full[:, w:].any(), f"padding of tiled level {l}"


@pytest.mark.parametrize("w,h,levels", SIZES, ids=IDS)
def test_frame_upload_any_number_of_given_levels(ctx, rule, w, h, levels):
    pyr = synth.build_pyramid(_images(w, h, 1, w * h)[0], levels, rule)
    for n_given in range(1, levels + 1):
        fr = capi.Frame(ctx, w, h, levels)
        try:
            fr.upload(pyr[:n_given])
            _check(fr, pyr)
        finally:
            fr.destroy()


@pytest.mark.parametrize("w,h,levels", SIZES, ids=IDS)
def test_frame_upload_device(ctx, rule, w, h, levels):
    img = _images(w, h, 1, w + h)[0]
    dev = torch.from_numpy(img).cuda(ctx.device)
    torch.cuda.synchronize(ctx.device)
    fr = capi.Frame(ctx, w, h, levels)
    try:
        fr.upload_device(dev.data_ptr())
        ctx.synchronize()
        _check(fr, synth.build_pyramid(img, levels, rule))
    finally:
        fr.destroy()


@pytest.mark.parametrize("w,h,levels", SIZES, ids=IDS)
def test_pool_window(ctx, rule, w, h, levels):
    imgs = _images(w, h, 3, 3 * w + h)
    pool = capi.FramePool(ctx, w, h, levels, 5)
    try:
        pool.upload_array(imgs, first=1)
        for i in range(3):
            _check(pool.frames[1 + i], synth.build_pyramid(imgs[i], levels, rule))
    finally:
        pool.destroy()


@pytest.mark.parametrize("w,h,levels", SIZES, ids=IDS)
def test_frame_upload_on_a_pool_frame(ctx, rule, w, h, levels):
    """builds the pyramid of that frame of the pool and of no other"""
    pyr = synth.build_pyramid(_images(w, h, 1, w ^ h)[0], levels, rule)
    zero = [np.zeros_like(p) for p in pyr]
    for n_given in range(1, levels + 1):
        pool = capi.FramePool(ctx, w, h, levels, 3)
        try:
            pool.frames[1].upload(pyr[:n_given])
            _check(pool.frames[1], pyr)
            _check(pool.frames[0], zero)
            _check(pool.frames[2], zero)
        finally:
            pool.destroy()


@pytest.mark.parametrize("w,h,levels", [(752, 480, 5), (645, 485, 7), (640, 480, 8), (96, 48, 2)],
                         ids=lambda v: str(v))
def test_single_frame_upload_launches_like_a_one_frame_pool(ctx, w, h, levels):
    img = _images(w, h, 1, 5)
    fr = capi.Frame(ctx, w, h, levels)
    pool = capi.FramePool(ctx, w, h, levels, 1)
    try:
        n0 = ctx.launch_count()
        fr.upload([img[0]])
        n1 = ctx.launch_count()
        pool.upload_array(img)
        n2 = ctx.launch_count()
        assert n1 - n0 == n2 - n1, (n1 - n0, n2 - n1)
        _check(fr, synth.build_pyramid(img[0], levels))
        _check(pool.frames[0], synth.build_pyramid(img[0], levels))
    finally:
        fr.destroy()
        pool.destroy()


@pytest.mark.parametrize("w,h", [(640, 480), (645, 485)], ids=lambda v: str(v))
def test_pool_upload_launches_do_not_depend_on_the_window(ctx, w, h):
    imgs = _images(w, h, 40, w - h)
    pool = capi.FramePool(ctx, w, h, 7, 40)
    try:
        n0 = ctx.launch_count()
        pool.upload_array(imgs[:1])
        n1 = ctx.launch_count()
        pool.upload_array(imgs)
        n2 = ctx.launch_count()
        assert n1 - n0 == n2 - n1, (n1 - n0, n2 - n1)
        for i in (0, 39):
            _check(pool.frames[i], synth.build_pyramid(imgs[i], 7))
    finally:
        pool.destroy()


def test_destroying_a_pool_frame_handle_leaves_the_pool_usable(ctx):
    w, h, levels = 640, 480, 5
    imgs = _images(w, h, 2, 11)
    pool = capi.FramePool(ctx, w, h, levels, 2)
    try:
        pool.upload_array(imgs)
        ctx.lib.svo_b200_frame_destroy(ctx.h, pool.frames[0].h)  # a borrowed handle: nothing happens
        for i in range(2):
            _check(pool.frames[i], synth.build_pyramid(imgs[i], levels))
        pool.upload_array(imgs[::-1])
        for i in range(2):
            _check(pool.frames[i], synth.build_pyramid(imgs[1 - i], levels))
    finally:
        pool.destroy()
