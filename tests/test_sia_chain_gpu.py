"""GPU: back-to-back runs of a staged full batch, which overlap on the device.

Consecutive svo_b200_sia_batch_run calls of one staged batch in the throughput geometry (160 threads x 2 features, three
CTAs per SM) launch each run as a programmatic dependent of the previous one: its CTAs start while the previous run's last
wave drains, and store the outputs only once that run has completed.  Any other work the library enqueues ends the chain.
Checked here: a chain of runs of a batch of more than three waves fetches exactly what one run does, and a chain broken by a
re-upload of the batch's images computes, bit for bit, what a fresh stage and run on the new images does.
"""
import numpy as np
import pytest
import torch

from rpg_svo_b200 import capi, synth

pytestmark = pytest.mark.gpu

W, H, NFEAT, NLEVELS = 640, 480, 300, 5


def _inputs(seed, B):
    st = synth.make_stream_fast(seed, B + 1, W, H, NFEAT, NLEVELS, device="cuda")
    cat = lambda k: np.concatenate([st["feats"][b][k] for b in range(B)])  # noqa: E731
    return dict(cam=st["cam"], level0=st["level0"].numpy(), px=cat("px"), f=cat("f"), pos=cat("pos"), hp=cat("has_point"),
                off=np.arange(B + 1, dtype=np.int32) * NFEAT, T0=np.tile(synth.se3_identity()[None], (B, 1, 1)),
                ref_pos=np.stack([synth.se3_inv(st["poses"][b])[:, 3] for b in range(B)]))


@pytest.fixture(scope="module")
def batch():
    """A batch of three full waves and part of a fourth on this device, and the level-0 images of a second stream."""
    B = 3 * 3 * torch.cuda.get_device_properties(0).multi_processor_count + 7
    return B, _inputs(11, B), _inputs(12, B)["level0"]


def _stage(ctx, pool, B, d):
    ctx.sia_batch_stage(pool.frames[:B], pool.frames[1:B + 1], d["cam"], d["T0"], d["off"], d["px"], d["f"], d["pos"], d["hp"],
                        d["ref_pos"], NLEVELS - 1, 0)


def _assert_same(a, b):
    for k in ("T", "H", "visible"):
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
    assert np.array_equal(a["stats"], b["stats"])


def _fresh(B, d, level0):
    """Stage and run the batch once on `level0` in a context of its own."""
    ctx = capi.Context(0)
    pool = capi.FramePool(ctx, W, H, NLEVELS, B + 1)
    pool.upload_array(level0)
    _stage(ctx, pool, B, d)
    ctx.sia_batch_run()
    r = ctx.sia_batch_fetch(want_H=True)
    pool.destroy()
    ctx.close()
    return r


def test_back_to_back_runs_fetch_what_one_run_computes(batch):
    B, d, _ = batch
    ctx = capi.Context(0)
    pool = capi.FramePool(ctx, W, H, NLEVELS, B + 1)
    pool.upload_array(d["level0"])
    _stage(ctx, pool, B, d)
    ctx.sia_batch_run()
    one = ctx.sia_batch_fetch(want_H=True)
    L = ctx.sia_last_launch()
    assert (L["threads"], L["features_per_thread"], L["ctas_per_pair"]) == (160, 2, 1), L
    assert one["stats"]["n_iters"].min() > 0
    for _ in range(12):
        ctx.sia_batch_run()
    _assert_same(ctx.sia_batch_fetch(want_H=True), one)
    pool.destroy()
    ctx.close()


def test_a_chain_broken_by_an_upload_runs_on_the_new_images(batch):
    B, d, level0_b = batch
    ctx = capi.Context(0)
    pool = capi.FramePool(ctx, W, H, NLEVELS, B + 1)
    pool.upload_array(d["level0"])
    _stage(ctx, pool, B, d)
    for _ in range(3):
        ctx.sia_batch_run()
    pool.upload_array(level0_b)  # the same pool frames, other images: the runs after it must see them
    for _ in range(3):
        ctx.sia_batch_run()
    got = ctx.sia_batch_fetch(want_H=True)
    pool.destroy()
    ctx.close()
    want = _fresh(B, d, level0_b)
    _assert_same(got, want)
    assert not np.array_equal(want["T"], _fresh(B, d, d["level0"])["T"])  # the upload changed what the batch computes
