"""GPU: the KLT kernels (svo_b200_klt_*) on the edge cases of tests/klt_edge_cases.py, against the oracle (decisions exact,
points bit for bit) and against OpenCV's own buildOpticalFlowPyramid / calcOpticalFlowPyrLK (recorded in
tests/golden/ref/test_klt_edges_gpu.npz; OpenCV is not needed here); rebuilding one pyramid handle at other sizes; pool
frames as the source image; the ABI's rejections and aliasing."""
import ctypes as C

import numpy as np
import pytest

from rpg_svo_b200 import capi
from tests import klt_cases as kc
from tests import klt_edge_cases as ke
from tests.ref_golden import ref, sha256_u8  # noqa: F401 (ref: fixture)

pytestmark = pytest.mark.gpu
_ctx = []


def gpu():
    """The module's context, created at first use (after a test's recorded reference calls)."""
    if not _ctx:
        _ctx.append(capi.Context(0))
    return _ctx[0]


def track(k, pts=None, want_exit=True):
    """Case k on the device: prev built with derivatives, next without, to max(max_level, 4) unless the case names the two
    build depths (then the tracker's option is the deeper one); one handle for both where the case asks for it."""
    c = gpu()
    lp, ln = k["levels"] or (max(k["max_level"], 4),) * 2
    fp = c.frame_from_level0(k["prev"], 1)
    pp = c.klt_pyramid(fp, True, lp)
    if k["same_handle"]:
        assert k["cur"] is k["prev"]
        fc, pc = None, pp
    else:
        fc = c.frame_from_level0(k["cur"], 1)
        pc = c.klt_pyramid(fc, False, ln)
    p0, p1 = (k["prev_pts"], k["next_pts"]) if pts is None else pts
    g = c.klt_track(pp, pc, p0, p1, max(lp, ln) if k["levels"] else k["max_level"], k["max_iter"], k["eps"], want_exit=want_exit)
    for x in {id(pp): pp, id(pc): pc}.values():
        x.destroy()
    for f in (fp, fc):
        if f is not None:
            f.destroy()
    return g


def digests(p, derivs):
    return [(sha256_u8(im).tobytes(), None if d is None else sha256_u8(d).tobytes())
            for im, d in (p.download(l, derivs) for l in range(p.n_levels))]


@pytest.mark.parametrize("spec", ke.EDGE_PYRAMIDS, ids=[f"{w}x{h}_max{m}" for w, h, m in ke.EDGE_PYRAMIDS])
def test_device_edge_pyramid_equals_opencv(spec, ref):
    """The device's level count, levels and derivatives have OpenCV's digests below the window, at a 31- or 32-pixel
    coarsest level and at the 8-level capacity."""
    w, h, max_level = spec
    img = ke.pyramid_image(w, h)
    r = ke.ref_pyramid(ref, img, max_level)
    c = gpu()
    f = c.frame_from_level0(img, 1)
    p = c.klt_pyramid(f, True, max_level)
    assert p.n_levels == r["n_levels"]
    for l in range(p.n_levels):
        im, der = p.download(l, True)
        assert np.array_equal(sha256_u8(im), r["images"][l]), l
        assert np.array_equal(sha256_u8(der), r["derivs"][l]), l
    p.destroy(); f.destroy()


@pytest.mark.parametrize("name", ke.NAMES)
def test_kernel_equals_oracle_and_opencv(name, ref):
    """Against the oracle: status, exit reasons of every level and step counts exact, points bit for bit (NaN as 'both
    NaN').  Against OpenCV: statuses exact, tracked points within TOL_PX, non-finite coordinates the same."""
    k = ke.case(name)
    r = kc.ref_run(ref, k)
    o = kc.oracle_run(k)
    g = track(k)
    if name == "nonfinite":
        sp = k["special"]
        print(f"nonfinite rows: status {g['status'][sp].tolist()}, reason {g['reason'][sp].tolist()}")
        for i in sp:
            print(f"  prev {k['prev_pts'][i]} guess {k['next_pts'][i]} -> status {g['status'][i]} {g['next_pts'][i]} "
                  f"levels {g['level_reason'][i, :4].tolist()} iters {g['iters'][i, :4].tolist()}")
    m = r["status"] == 1
    d_o = float(np.nanmax(np.abs(g["next_pts"] - o["next_pts"]))) if np.isfinite(o["next_pts"]).any() else 0.0
    d_r = float(np.abs(g["next_pts"][m] - r["next_pts"][m]).max()) if m.any() else 0.0
    print(f"{name}: {int(m.sum())}/{len(m)} tracked, max |kernel - oracle| = {d_o:.3g} px, max |kernel - OpenCV| = {d_r:.3g} px")
    assert np.array_equal(g["status"], o["status"]) and np.array_equal(g["status"], r["status"])
    assert np.array_equal(g["reason"], o["reason"])
    assert np.array_equal(g["level_reason"], o["level_reason"])
    assert np.array_equal(g["iters"], o["iters"])
    assert ke.bits_equal(g["next_pts"], o["next_pts"])
    assert d_r <= kc.TOL_PX and ke.same_nonfinite(g["next_pts"], r["next_pts"])
    if name == "nonfinite":  # the ordinary points of the same warps and CTAs come out as they do alone
        od = k["ordinary"]
        a = track(k, pts=(k["prev_pts"][od], k["next_pts"][od]))
        assert ke.bits_equal(a["next_pts"], g["next_pts"][od]) and np.array_equal(a["iters"], g["iters"][od])


def test_rebuilt_handle_equals_fresh_builds():
    """One handle rebuilt at 752 x 480 with derivatives, 60 x 40 without, 645 x 485 with, 1 x 1 without (the build reuses
    its allocation where the new pyramid fits): after each build its levels and derivatives have the digests of a fresh
    handle's, and tracking from it is bit-identical to tracking from the fresh one."""
    c = gpu()
    reused = capi.KltPyramid(c)
    for (w, h), derivs in (((752, 480), True), ((60, 40), False), ((645, 485), True), ((1, 1), False)):
        img = kc.pyr_image(w, h)
        f = c.frame_from_level0(img, 1)
        reused.build(f, derivs)
        fresh = c.klt_pyramid(f, derivs)
        assert reused.n_levels == fresh.n_levels == len(ke.binding_klt.level_sizes(w, h))
        assert digests(reused, derivs) == digests(fresh, derivs), (w, h)
        other = c.klt_pyramid(f, not derivs)  # the other role: track the image onto itself, shifted guesses
        rng = np.random.default_rng(w)
        p0 = (rng.random((40, 2)) * [w + 20, h + 20] - 10).astype(np.float32)
        p1 = (p0 + rng.random((40, 2)).astype(np.float32) - 0.5).astype(np.float32)
        runs = [c.klt_track(x, other, p0, p1) if derivs else c.klt_track(other, x, p0, p1) for x in (reused, fresh)]
        assert ke.bits_equal(runs[0]["next_pts"], runs[1]["next_pts"]), (w, h)
        for key in ("status", "level_reason", "iters"):
            assert np.array_equal(runs[0][key], runs[1][key]), (w, h, key)
        fresh.destroy(); other.destroy(); f.destroy()
    reused.destroy()


def test_pool_frames_as_source():
    """A pyramid built from the first and the last frame of a FramePool equals one built from frame_from_level0."""
    c = gpu()
    w, h = 645, 485
    imgs = np.stack([kc.pyr_image(w, h, seed) for seed in (3, 4, 5)])
    pool = capi.FramePool(c, w, h, 3, len(imgs))
    pool.upload_array(imgs)
    for i in (0, len(imgs) - 1):
        f = c.frame_from_level0(imgs[i], 1)
        a, b = c.klt_pyramid(pool.frames[i], True), c.klt_pyramid(f, True)
        assert a.n_levels == b.n_levels == 5 and digests(a, True) == digests(b, True), i
        a.destroy(); b.destroy(); f.destroy()
    pool.destroy()


def test_abi_edges():
    """SVO_B200_EINVAL for eps < 0, eps NaN, max_level < 0 (OpenCV clamps those; the ABI refuses them), a download level
    out of range, derivatives from a pyramid built without them, and a build that would need a ninth level (refused on the
    host: no launch, the handle keeps its previous build).  exit_out NULL and prev_pts == next_pts_io give what separate
    buffers and a non-NULL exit_out give."""
    c = gpu()
    lib = c.lib
    k = ke.case("level_3")
    fp, fc = c.frame_from_level0(k["prev"], 1), c.frame_from_level0(k["cur"], 1)
    pp, pc = c.klt_pyramid(fp, True), c.klt_pyramid(fc, False)
    n = 16
    p0 = np.ascontiguousarray(k["prev_pts"][:n])
    st = np.zeros(n, np.uint8)

    def call(opt, pts, io):
        return lib.svo_b200_klt_track(c.h, pp.h, pc.h, C.byref(opt), n, capi._p(pts), capi._p(io), capi._p(st), None)

    io = p0.copy()
    assert call(capi.KltOptions(30, 4, 30, 0.001), p0, io) == 0
    for opt in (capi.KltOptions(30, 4, 30, -1e-9), capi.KltOptions(30, 4, 30, float("nan")), capi.KltOptions(30, -1, 30, 0.001)):
        assert call(opt, p0, p0.copy()) == -1
    with_exit = c.klt_track(pp, pc, p0, p0)
    without = c.klt_track(pp, pc, p0, p0, want_exit=False)
    assert ke.bits_equal(with_exit["next_pts"], without["next_pts"]) and np.array_equal(with_exit["status"], without["status"])
    assert ke.bits_equal(io, with_exit["next_pts"])
    alias = p0.copy()  # prev_pts and next_pts_io one buffer
    assert call(capi.KltOptions(30, 4, 30, 0.001), alias, alias) == 0
    assert ke.bits_equal(alias, with_exit["next_pts"]) and np.array_equal(st, with_exit["status"])

    def download(p, level, derivs):
        img = np.zeros((480, 640), np.uint8)
        der = np.zeros((480, 640, 2), np.int16) if derivs else None
        return lib.svo_b200_klt_pyramid_download(c.h, p.h, level, capi._p(img), capi._p(der))

    assert download(pp, 0, True) == 0 and download(pc, 0, False) == 0
    assert download(pp, -1, False) == -1 and download(pp, pp.n_levels, False) == -1
    assert download(pc, 0, True) == -1  # built without derivatives

    big = np.zeros((7936, 7936), np.uint8)
    fb = c.frame_from_level0(big, 1)
    before, launches = digests(pp, True), c.launch_count()
    for m in (8, 9, 1000):
        assert lib.svo_b200_klt_pyramid_build(c.h, pp.h, fb.h, m, 1) == -1
        assert b"levels" in lib.svo_b200_last_error(c.h)
    assert c.launch_count() == launches and pp.n_levels == 4 and digests(pp, True) == before
    fresh = capi.KltPyramid(c)
    assert lib.svo_b200_klt_pyramid_build(c.h, fresh.h, fb.h, 8, 0) == -1 and fresh.n_levels == 0
    assert lib.svo_b200_klt_pyramid_build(c.h, fresh.h, fb.h, 7, 0) == 0 and fresh.n_levels == 8
    for x in (pp, pc, fresh):
        x.destroy()
    for f in (fp, fc, fb):
        f.destroy()
