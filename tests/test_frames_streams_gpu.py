"""GPU: svo_b200_frame_upload_streams -- S frames' level-0 uploads and pyramid builds with one launch per stage -- against
single svo_b200_frame_upload calls (every level and every block-tiled copy, byte for byte) and vk::halfSample's pyramid
(synth.build_pyramid), under both rounding rules; launch counts over shapes up to 257 frames; every refusal, which must
launch and write nothing; the end of a staged alignment batch's run chain; and the C++ host mirror svo::streams::newFrames
against the svo::Frame constructor."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

from rpg_svo_b200 import capi, synth

pytestmark = pytest.mark.gpu
EINVAL = -1

# sizes x levels: widths that are multiples of 16 (the streaming level-0 kernel) and that are not (644, 645, 17), second
# fused passes (645 x 485 x 7, 640 x 480 x 8), the tiling kernel's level 1 (96 x 48 x 2) and a frame the tiling kernel alone
# fills (17 x 9 x 1)
MIXED = [(752, 480, 5), (640, 480, 5), (644, 484, 4), (656, 490, 5), (1920, 1080, 6), (645, 485, 7), (640, 480, 8), (96, 48, 2),
         (17, 9, 1)]
POOL = (640, 480, 5, 4)  # a pool whose frames 0 and 2 join the mixed batch


@pytest.fixture(params=[synth.PYR_X86, synth.PYR_SCALAR], ids=["x86-sse2-rule", "scalar-rule"])
def rule(request, ctx):
    ctx.set_pyramid_rule(request.param)
    yield request.param
    ctx.set_pyramid_rule(synth.PYR_X86)


def _image(w, h, seed):
    return np.random.default_rng(seed).integers(1, 256, (h, w), dtype=np.uint8)  # no zero pixel: padding stays visible


def _plan(w, levels):
    """(streaming launch, tiling launch, fused passes) of one frame's level-0 upload."""
    stream = levels > 1 and w % 16 == 0
    top = 1 if stream else 0
    tiles = (levels == 1) or (stream and levels == 2)
    return stream, tiles, len(range(top, levels - 1, 4))


def stage_launches(shapes):
    """One streaming launch if any frame has it, one tiling launch if any needs it, and the most fused passes of any."""
    plans = [_plan(w, l) for w, _, l in shapes]
    return int(any(p[0] for p in plans)) + int(any(p[1] for p in plans)) + max((p[2] for p in plans), default=0)


def _state(fr):
    return [(fr.download_level(l), fr.download_level_tiled(l)) for l in range(fr.n_levels)]


def _same_state(a, b):
    return len(a) == len(b) and all(np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) for x, y in zip(a, b))


def _single(ctx, w, h, levels, img):
    fr = capi.Frame(ctx, w, h, levels)
    fr.upload([img])
    s = _state(fr)
    fr.destroy()
    return s


def test_mixed_batch_equals_single_uploads_and_half_sample(ctx, rule):
    """Every size of MIXED as a single frame plus two non-adjacent frames of one pool, listed apart: every level and tiled
    copy equals a single upload of the same image, every level equals synth.build_pyramid, and the call makes the stage
    formula's launches (four: streaming, tiling, two fused passes)."""
    frames = [capi.Frame(ctx, w, h, l) for w, h, l in MIXED]
    pool = capi.FramePool(ctx, *POOL)
    frames = frames[:3] + [pool.frames[2]] + frames[3:7] + [pool.frames[0]] + frames[7:]
    imgs = [_image(f.width, f.height, 100 + i) for i, f in enumerate(frames)]
    n0 = ctx.launch_count()
    assert ctx.frames_upload(list(zip(frames, imgs))) == frames
    shapes = [(f.width, f.height, f.n_levels) for f in frames]
    assert ctx.launch_count() - n0 == stage_launches(shapes) == 4
    assert ctx.last_kernel_ms() > 0
    for f, img in zip(frames, imgs):
        got = _state(f)
        assert _same_state(got, _single(ctx, f.width, f.height, f.n_levels, img)), (f.width, f.height, f.n_levels)
        for l, ref in enumerate(synth.build_pyramid(img, f.n_levels, rule)):
            assert np.array_equal(got[l][0], ref), (f.width, f.height, f.n_levels, l)
    for f in frames:
        f.destroy()
    pool.destroy()


SHAPE_MIX = [(645, 485, 7), (96, 48, 2)]  # two fused passes; streaming and tiling launches from the second shape


@pytest.mark.parametrize("S", [0, 1, 2, 33, 132, 257])
def test_shapes(ctx, rule, S):
    """S frames cycling through SHAPE_MIX: the launch count is the stage formula's (the same for S = 2 and 257; none for
    S == 0), and every frame (all up to 33, a sample above) equals its single upload."""
    shapes = [SHAPE_MIX[s % 2] for s in range(S)]
    frames = [capi.Frame(ctx, w, h, l) for w, h, l in shapes]
    imgs = [_image(w, h, 1000 * S + s) for s, (w, h, _) in enumerate(shapes)]
    n0 = ctx.launch_count()
    ctx.frames_upload(list(zip(frames, imgs)))
    n = ctx.launch_count() - n0
    assert n == stage_launches(shapes) == {0: 0, 1: 2}.get(S, 4)
    rng = np.random.default_rng(S)
    for s in (range(S) if S <= 33 else rng.choice(S, 12, replace=False)):
        w, h, l = shapes[s]
        assert _same_state(_state(frames[s]), _single(ctx, w, h, l, imgs[s])), s
    for f in frames:
        f.destroy()


def test_refusals_write_nothing(ctx, rule):
    """After known content is uploaded, each refusal returns SVO_B200_EINVAL with no launch, and every frame keeps its levels
    and tiled copies: S < 0, a NULL table, a NULL frame, a NULL image, a frame listed twice (the bad entry last, after
    entries that would change their frames)."""
    lib = ctx.lib
    pool = capi.FramePool(ctx, 644, 484, 4, 3)
    frames = [capi.Frame(ctx, 752, 480, 5), pool.frames[1], capi.Frame(ctx, 17, 9, 1)]
    ctx.frames_upload([(f, _image(f.width, f.height, 7 + i)) for i, f in enumerate(frames)])
    before = [_state(f) for f in frames]
    other = [np.ascontiguousarray(_image(f.width, f.height, 70 + i)) for i, f in enumerate(frames)]

    def table(rows):
        return (capi.FrameUploadEntry * len(rows))(*[capi.FrameUploadEntry(f, p) for f, p in rows])

    good = [(f.h.value, im.ctypes.data) for f, im in zip(frames, other)]
    bad = [("S < 0", -1, table(good)), ("NULL table", 3, None),
           ("NULL frame", 4, table(good + [(None, other[0].ctypes.data)])),
           ("NULL image", 4, table(good + [(frames[0].h.value, None)])),
           ("frame twice", 4, table(good + [(frames[1].h.value, other[1].ctypes.data)])),
           ("pool frame twice", 4, table(good + [(C.c_void_p(lib.svo_b200_frame_pool_get(pool.h, 1)).value, other[1].ctypes.data)]))]
    for name, S, arr in bad:
        n0 = ctx.launch_count()
        assert lib.svo_b200_frame_upload_streams(ctx.h, S, arr) == EINVAL, name
        assert ctx.launch_count() == n0, name
        ctx.synchronize()
        for f, b in zip(frames, before):
            assert _same_state(_state(f), b), name
    n0 = ctx.launch_count()
    assert lib.svo_b200_frame_upload_streams(ctx.h, 0, None) == 0 and ctx.launch_count() == n0   # S == 0: no launch
    for f in frames:
        f.destroy()
    pool.destroy()


def test_upload_ends_an_alignment_run_chain(rule):
    """A staged alignment batch runs, its frames are re-uploaded with other images through one batched call, and the batch
    runs again: it fetches, bit for bit, what a fresh stage and run on the new images (uploaded window by window) fetches."""
    from tests.test_sia_chain_gpu import NLEVELS, H, W, _assert_same, _inputs, _stage

    B = 48
    d, level0_b = _inputs(21, B), _inputs(22, B)["level0"]

    def run(reupload):
        c = capi.Context(0)
        c.set_pyramid_rule(rule)
        pool = capi.FramePool(c, W, H, NLEVELS, B + 1)
        pool.upload_array(level0_b if not reupload else d["level0"])
        _stage(c, pool, B, d)
        c.sia_batch_run()
        c.sia_batch_run()
        if reupload:
            c.frames_upload(list(zip(pool.frames, level0_b)))
            c.sia_batch_run()
        r = c.sia_batch_fetch(want_H=True)
        pool.destroy()
        c.close()
        return r

    got, want = run(True), run(False)
    _assert_same(got, want)


def test_host_new_frames_equal_the_constructor():
    """host_frames_streams_demo: svo::streams::newFrames gives every frame the levels and tiled copies the svo::Frame
    constructor gives it (five and three streams of mixed sizes, 5 and 2 levels, both rules), and its refusals throw."""
    from tests.test_host_cpp_gpu import build_demo

    out = subprocess.run([build_demo("host_frames_streams_demo")], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr)
    rows = re.findall(r"constructor ([0-9a-f]{16}) batched ([0-9a-f]{16})$", out.stdout, re.M)
    assert len(rows) == 16 and all(a == b for a, b in rows)
    assert "frames 16 equal 16" in out.stdout
    assert "refusals thrown 4 of 4" in out.stdout
    assert "empty batch 0 frames" in out.stdout
    assert out.returncode == 0
