"""GPU: the KLT kernels (svo_b200_klt_*) against the oracle (bit for bit in decisions, 1e-4 px in points) and against
OpenCV's own buildOpticalFlowPyramid / calcOpticalFlowPyrLK (recorded in tests/golden/ref/test_klt_gpu.npz; OpenCV is not
needed here), on the cases of tests/klt_cases.py; batch sizes; argument errors; the C++ host mirror."""
import os
import subprocess

import numpy as np
import pytest

from rpg_svo_b200 import capi
from tests import klt_cases as kc
from tests.ref_golden import ref, sha256_u8  # noqa: F401 (ref: fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_ctx = []


def gpu():
    """The module's context, created at first use (after a test's recorded reference calls)."""
    if not _ctx:
        _ctx.append(capi.Context(0))
    return _ctx[0]


def track(k, prev=None, cur=None, pts=None):
    c = gpu()
    fp, fc = c.frame_from_level0(k["prev"], 1), c.frame_from_level0(k["cur"], 1)
    pp, pc = c.klt_pyramid(fp, True), c.klt_pyramid(fc, False)
    p0, p1 = (k["prev_pts"], k["next_pts"]) if pts is None else pts
    g = c.klt_track(pp, pc, p0, p1, k["max_level"], k["max_iter"], k["eps"])
    for x in (pp, pc):
        x.destroy()
    fp.destroy(); fc.destroy()
    return g


@pytest.mark.parametrize("size", kc.PYR_SIZES, ids=[f"{w}x{h}" for w, h in kc.PYR_SIZES])
def test_device_pyramid_equals_opencv(size, ref):
    """The device's levels and derivatives have OpenCV's digests; its level count is OpenCV's."""
    w, h = size
    img = kc.pyr_image(w, h)
    r = kc.ref_pyramid(ref, img)
    c = gpu()
    f = c.frame_from_level0(img, 1)
    p = c.klt_pyramid(f, True)
    assert p.n_levels == r["n_levels"]
    for l in range(p.n_levels):
        im, der = p.download(l, True)
        assert np.array_equal(sha256_u8(im), r["images"][l]), l
        assert np.array_equal(sha256_u8(der), r["derivs"][l]), l
    q = c.klt_pyramid(f, False)  # a build without derivatives: same images
    assert q.n_levels == p.n_levels and np.array_equal(q.download(q.n_levels - 1)[0], p.download(p.n_levels - 1)[0])
    p.destroy(); q.destroy(); f.destroy()


@pytest.mark.parametrize("name", kc.NAMES)
def test_kernel_equals_oracle_and_opencv(name, ref):
    """Against the oracle: status, exit reasons of every level and per-level step counts exact, points within 1e-4 px.
    Against OpenCV: statuses exact, points within the CPU pin's tolerance."""
    k = kc.case(name)
    r = kc.ref_run(ref, k)
    o = kc.oracle_run(k)
    g = track(k)
    assert np.array_equal(g["status"], o["status"]) and np.array_equal(g["status"], r["status"])
    assert np.array_equal(g["reason"], o["reason"])
    assert np.array_equal(g["level_reason"], o["level_reason"])
    assert np.array_equal(g["iters"], o["iters"])
    d_o = float(np.abs(g["next_pts"] - o["next_pts"]).max())
    m = r["status"] == 1
    d_r = float(np.abs(g["next_pts"][m] - r["next_pts"][m]).max()) if m.any() else 0.0
    print(f"{name}: max |kernel - oracle| = {d_o:.3g} px, max |kernel - OpenCV| = {d_r:.3g} px (tracked points)")
    assert d_o <= 1e-4 and d_r <= kc.TOL_PX


def test_kernel_reaches_every_branch():
    """Each branch the cases are built for, as the kernel reports it."""
    R = {n: track(kc.case(n)) for n in kc.NAMES}
    assert {capi.KLT_CONVERGED, capi.KLT_HALF_STEP, capi.KLT_OUT_OF_BOUNDS} <= set(R["shift_640"]["reason"].tolist())
    assert np.all(R["shift_640"]["level_reason"][:, 4:] == -1)                                  # 4 levels at 640 x 480
    assert np.all(R["shift_644"]["level_reason"][:, 4] >= 0) and np.all(R["shift_644"]["level_reason"][:, 5:] == -1)  # 5
    assert np.all(R["iter_1"]["level_reason"][:, :4] == capi.KLT_MAX_ITER) and np.all(R["iter_1"]["iters"][:, :4] == 1)
    t = R["iter_30_tight"]
    assert np.all((t["reason"] == capi.KLT_HALF_STEP) | (t["reason"] == capi.KLT_MAX_ITER) | (t["reason"] == capi.KLT_OUT_OF_BOUNDS))
    assert np.sum((R["far_flow"]["reason"] == capi.KLT_MAX_ITER) & (R["far_flow"]["iters"][:, 0] == 30)) > 50  # the limit at 30
    f = R["far_flow"]
    assert np.any((f["level_reason"][:, 3] == capi.KLT_OUT_OF_BOUNDS) & (f["level_reason"][:, 0] >= 0))
    assert np.sum(f["status"]) > 0 and np.sum(f["status"] == 0) > 0
    assert np.all(R["flat"]["reason"][:120] == capi.KLT_SMALL_EIG) and np.all(R["flat"]["status"][:120] == 0)
    b = R["border"]
    assert np.all(b["reason"][[*range(16), *range(20, 36)]] != capi.KLT_OUT_OF_BOUNDS)
    assert np.all(b["reason"][[16, 17, 18, 19, 36, 37, 38, 39]] == capi.KLT_OUT_OF_BOUNDS)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 4097])
def test_batches_equal_single_launches(n):
    """N points in one launch give what N one-point launches give (4 points per CTA: partial CTAs, many CTAs)."""
    k = kc.case("shift_640")
    rng = np.random.default_rng(n)
    p0 = (rng.random((n, 2)) * [660, 500] - 10).astype(np.float32)
    g = track(k, pts=(p0, p0))
    assert len(g["status"]) == n
    idx = range(n) if n <= 33 else rng.choice(n, 24, replace=False)
    for i in idx:
        s = track(k, pts=(p0[i:i + 1], p0[i:i + 1]))
        assert s["status"][0] == g["status"][i] and s["reason"][0] == g["reason"][i]
        assert np.array_equal(s["next_pts"][0].view(np.uint32), g["next_pts"][i].view(np.uint32))
        assert np.array_equal(s["iters"][0], g["iters"][i])


def test_abi_rejects_bad_arguments():
    """SVO_B200_EINVAL for a window other than 30, a NULL pyramid, N < 0 and a previous pyramid without derivatives."""
    c = gpu()
    k = kc.case("iter_1")
    fp, fc = c.frame_from_level0(k["prev"], 1), c.frame_from_level0(k["cur"], 1)
    pp, pc = c.klt_pyramid(fp, True), c.klt_pyramid(fc, False)
    p = k["prev_pts"][:4]
    lib = c.lib
    o = capi.KltOptions(30, 4, 30, 0.001)
    st = np.zeros(4, np.uint8)
    p1 = p.copy()

    def call(prev, nxt, opt, n):
        return lib.svo_b200_klt_track(c.h, prev, nxt, capi.C.byref(opt), n, capi._p(p), capi._p(p1), capi._p(st), None)

    assert call(pp.h, pc.h, o, 4) == 0
    assert call(pp.h, pc.h, capi.KltOptions(31, 4, 30, 0.001), 4) == -1
    assert call(pp.h, pc.h, capi.KltOptions(21, 4, 30, 0.001), 4) == -1
    assert call(None, pc.h, o, 4) == -1 and call(pp.h, None, o, 4) == -1
    assert call(pp.h, pc.h, o, -1) == -1
    assert call(pc.h, pc.h, o, 4) == -1  # built without derivatives
    assert call(pp.h, pc.h, o, 0) == 0
    for x in (pp, pc):
        x.destroy()
    fp.destroy(); fc.destroy()


def test_host_track_klt_equals_numpy_statement():
    """host_klt_demo (svo::initialization::detectFeatures + trackKlt over the device) against a numpy statement of
    initialization.cpp:107-169 on the same device outputs: erase order, f_cur from the pinhole and the ATAN camera,
    disparities widened from float differences."""
    exe = os.path.join(ROOT, "rpg_svo_b200", "host", "host_klt_demo")
    for cam in ("pinhole", "atan"):
        out = subprocess.run([exe, cam], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        lines = out.stdout.splitlines()
        frames = [ln for ln in lines if ln.startswith("frame ")]
        assert len(frames) == 3 and all("tracked" in ln for ln in frames), out.stdout
        rows = np.array([[float(v) for v in ln.split()[1:]] for ln in lines if ln.startswith("pt ")])
        _check_host_rows(cam, rows)


def _camera(cam):
    from rpg_svo_b200 import synth

    return synth.reference_param_camera("atan") if cam == "atan" else synth.camera_for(752, 480)


def _c2f(cam, px):
    """vk::PinholeCamera / vk::ATANCamera cam2world for undistorted pinhole and the ATAN model (numpy statement)."""
    c = _camera(cam)
    x = (px[:, 0] - c.cx) / c.fx
    y = (px[:, 1] - c.cy) / c.fy
    if cam == "atan":
        s = c.d[0]
        r = np.sqrt(x * x + y * y)
        tans_inv = 1.0 / (2.0 * np.tan(s / 2.0))
        fac = np.where(r > 0.01, np.tan(r * s) * tans_inv / np.where(r > 0.01, r, 1.0), 1.0)
        x, y = fac * x, fac * y
    n = np.sqrt(x * x + y * y + 1.0)
    return np.stack([x / n, y / n, 1.0 / n], 1)


def _check_host_rows(cam, rows):
    """rows: frame, index, px_ref (2), px_cur (2), f_cur (3), disparity -- what the demo kept, in order."""
    from tests.klt_host_scene import scene

    c = gpu()
    imgs, n_levels = scene()
    f0 = c.frame_from_level0(imgs[0], n_levels)
    det = c.fast_detect(f0, 30, 3, 20.0)
    px_ref = np.stack([det["x"], det["y"]], 1).astype(np.float32)  # cv::Point2f(ftr->px[0], ftr->px[1])
    keep = np.arange(len(px_ref))
    px_cur = px_ref.copy()
    p0 = c.klt_pyramid(f0, True)
    for fi in range(1, len(imgs)):
        f = c.frame_from_level0(imgs[fi], n_levels)
        p = c.klt_pyramid(f, False)
        g = c.klt_track(p0, p, px_ref, px_cur, 4, 30, 0.001, want_exit=False)
        ok = g["status"] == 1
        px_ref, px_cur, keep = px_ref[ok], g["next_pts"][ok], keep[ok]  # erase in order
        fc = _c2f(cam, px_cur.astype(np.float64))
        dd = (px_ref - px_cur).astype(np.float64)  # float differences, widened
        disp = np.sqrt(dd[:, 0] ** 2 + dd[:, 1] ** 2)
        r = rows[rows[:, 0] == fi]
        assert len(r) == len(px_cur), (fi, len(r), len(px_cur))
        assert np.array_equal(r[:, 1].astype(int), keep)
        assert np.array_equal(r[:, 2:4].astype(np.float32), px_ref) and np.array_equal(r[:, 4:6].astype(np.float32), px_cur)
        assert np.allclose(r[:, 6:9], fc, rtol=0, atol=1e-12)
        assert np.allclose(r[:, 9], disp, rtol=1e-15, atol=0)
        p.destroy(); f.destroy()
    p0.destroy(); f0.destroy()
