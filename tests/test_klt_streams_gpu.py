"""GPU: svo_b200_klt_track_streams -- S streams' calcOpticalFlowPyrLK in one launch -- and svo_b200_klt_pyramid_build_streams
-- S LK pyramids with one launch per stage -- against single svo_b200_klt_track / svo_b200_klt_pyramid_build calls (bit for
bit, float32 points as uint32 bits), against the oracle (decisions and step counts exact, points within 1e-4 px) and against
OpenCV's own calcOpticalFlowPyrLK / buildOpticalFlowPyramid (recorded in tests/golden/ref/test_klt_streams_gpu.npz; OpenCV
is not needed here); launch counts, shapes up to 257 streams, every refusal (which must launch and write nothing), and the
C++ host mirror svo::streams::trackKlt against sequential initialization::trackKlt calls."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from rpg_svo_b200 import capi
from tests import klt_cases as kc
from tests import klt_edge_cases as ke
from tests.ref_golden import ref, sha256_u8  # noqa: F401 (ref: fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL = -1
_ctx = []

# the cases run as streams of one call: every klt_cases case and the edge cases that change the level count, the sizes,
# the options or the handles (the 3968 x 3968 capacity case stays with test_klt_edges_gpu.py)
EDGE_NAMES = ["nonfinite", "tiny_1x1", "tiny_2x3", "tiny_17x29", "tiny_31x31", "tiny_62x62", "tiny_645x485", "binary", "iter_0",
              "iter_neg3", "eps_10", "level_0", "level_7", "mixed_levels", "same_handle"]


def gpu():
    """The module's context, created at first use (after a test's recorded reference calls)."""
    if not _ctx:
        _ctx.append(capi.Context(0))
    return _ctx[0]


def u32(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


class Pair:
    """Case k's pyramids, built as test_klt_edges_gpu.py builds them: prev with derivatives, next without, to
    max(max_level, 4) unless the case names the two depths (the tracker's option is then the deeper one); one handle for
    both where the case asks for it."""

    def __init__(self, c, k):
        lp, ln = k["levels"] or (max(k["max_level"], 4),) * 2
        self.frames = [c.frame_from_level0(k["prev"], 1)]
        self.prev = c.klt_pyramid(self.frames[0], True, lp)
        if k["same_handle"]:
            self.next = self.prev
        else:
            self.frames.append(c.frame_from_level0(k["cur"], 1))
            self.next = c.klt_pyramid(self.frames[1], False, ln)
        self.max_level = max(lp, ln) if k["levels"] else k["max_level"]
        self.k = k

    def args(self, pts=None, want_exit=True):
        p0, p1 = (self.k["prev_pts"], self.k["next_pts"]) if pts is None else pts
        return dict(prev=self.prev, nxt=self.next, prev_pts=p0, next_pts=p1, max_level=self.max_level,
                    max_iter=self.k["max_iter"], eps=self.k["eps"], want_exit=want_exit)

    def destroy(self):
        for p in {id(self.prev): self.prev, id(self.next): self.next}.values():
            p.destroy()
        for f in self.frames:
            f.destroy()


def same_as_single(c, args, b):
    """Stream `b` of a batched call equals one klt_track call with the same arguments, bit for bit."""
    s = c.klt_track(**args)
    assert np.array_equal(u32(s["next_pts"]), u32(b["next_pts"]))
    assert np.array_equal(s["status"], b["status"])
    assert set(s) == set(b)
    for key in ("reason", "level_reason", "iters"):
        if key in s:
            assert np.array_equal(s[key], b[key]), key


def batched(c, streams, launches=1):
    n0 = c.launch_count()
    out = c.klt_track_streams(streams)
    assert c.launch_count() == n0 + launches
    return out


def test_heterogeneous_streams_equal_single_calls_and_oracle():
    """One call over every case of klt_cases and the edge cases above (four image sizes and the tiny ones, far flow, flat
    blocks, the border, non-finite coordinates, per-stream max_level / max_iter / eps), a stream of 0 points, exit records
    off in every third stream, and two streams that share one reference pyramid."""
    c = gpu()
    cases = [kc.case(n) for n in kc.NAMES] + [ke.case(n) for n in EDGE_NAMES]
    for k in cases:
        k.setdefault("levels", None)
        k.setdefault("same_handle", False)
    pairs = [Pair(c, k) for k in cases]
    streams = [p.args(want_exit=i % 3 != 2) for i, p in enumerate(pairs)]
    sh = pairs[kc.NAMES.index("shift_640")]
    half = (sh.k["prev_pts"][::2] + np.float32(0.5), sh.k["next_pts"][::2] + np.float32(1.25))
    streams.append(sh.args(pts=half))                                            # shares shift_640's pyramids
    streams.append(sh.args(pts=(np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32))))  # N = 0
    out = batched(c, streams)
    assert len(out[-1]["status"]) == 0
    for a, b in zip(streams, out):
        same_as_single(c, a, b)
    for k, a, b in zip(cases, streams, out):
        o = kc.oracle_run(k)
        assert np.array_equal(b["status"], o["status"]), k["name"]
        if "reason" in b:
            assert np.array_equal(b["reason"], o["reason"]) and np.array_equal(b["level_reason"], o["level_reason"]), k["name"]
            assert np.array_equal(b["iters"], o["iters"]), k["name"]
        fin = np.isfinite(o["next_pts"])
        assert ke.same_nonfinite(b["next_pts"], o["next_pts"]), k["name"]
        assert float(np.abs(b["next_pts"][fin] - o["next_pts"][fin]).max(initial=0.0)) <= 1e-4, k["name"]
    reasons = np.concatenate([b["reason"] for b in out if "reason" in b])
    assert {capi.KLT_CONVERGED, capi.KLT_HALF_STEP, capi.KLT_MAX_ITER, capi.KLT_OUT_OF_BOUNDS, capi.KLT_SMALL_EIG} <= set(reasons.tolist())
    for p in pairs:
        p.destroy()


def test_stream_equals_opencv(ref):
    """shift_752 as the middle stream of a three-stream call: statuses exact, tracked points within TOL_PX of OpenCV."""
    k = kc.case("shift_752")
    r = kc.ref_run(ref, k)
    c = gpu()
    others = [kc.case("shift_640"), kc.case("far_flow")]
    pairs = [Pair(c, dict(x, levels=None, same_handle=False)) for x in (others[0], k, others[1])]
    out = batched(c, [p.args() for p in pairs])
    g = out[1]
    m = r["status"] == 1
    d_r = float(np.abs(g["next_pts"][m] - r["next_pts"][m]).max())
    print(f"shift_752 in a 3-stream call: {int(m.sum())}/{len(m)} tracked, max |kernel - OpenCV| = {d_r:.3g} px")
    assert np.array_equal(g["status"], r["status"]) and d_r <= kc.TOL_PX
    for p in pairs:
        p.destroy()


def digests(p, derivs):
    return [(sha256_u8(im).tobytes(), None if d is None else sha256_u8(d).tobytes())
            for im, d in (p.download(l, derivs) for l in range(p.n_levels))]


def expected_launches(specs):
    """1 (level 0) + L_max - 1 (pyrDown) + 1 if any entry has derivatives (Scharr)."""
    L_max = max(len(ke.binding_klt.level_sizes(f.width, f.height, m)) for f, _, m in specs)
    return 1 + (L_max - 1) + (1 if any(d for _, d, _ in specs) else 0)


def test_batched_build_equals_single_builds_and_opencv(ref):
    """The sizes of PYR_SIZES with derivatives at max_level 4 (against OpenCV's recorded digests), the same without at
    max_level 2, 752 x 480 at max_level 0 and 7, and a frame-pool frame, in one call: every level and derivative equals a
    single build, and the call makes 1 + (L_max - 1) + 1 launches."""
    imgs = [kc.pyr_image(w, h) for w, h in kc.PYR_SIZES]
    refs = [kc.ref_pyramid(ref, img) for img in imgs]
    c = gpu()
    frames = [c.frame_from_level0(img, 1) for img in imgs]
    pool = capi.FramePool(c, 645, 485, 3, 3)
    pool.upload_array(np.stack([kc.pyr_image(645, 485, seed) for seed in (3, 4, 5)]))
    specs = [(f, True, 4) for f in frames] + [(f, False, 2) for f in frames] + [(frames[1], True, 0), (frames[1], False, 7),
                                                                                 (pool.frames[1], True, 4)]
    n0 = c.launch_count()
    pyrs = c.klt_pyramids([dict(frame=f, derivatives=d, max_level=m) for f, d, m in specs])
    assert c.launch_count() - n0 == expected_launches(specs) == 6                # 644 x 484: 5 levels
    for p, (f, d, m) in zip(pyrs, specs):
        single = c.klt_pyramid(f, d, m)
        assert p.n_levels == single.n_levels == len(ke.binding_klt.level_sizes(f.width, f.height, m))
        assert digests(p, d) == digests(single, d), (f.width, f.height, d, m)
        single.destroy()
    for p, r in zip(pyrs[:len(imgs)], refs):
        assert p.n_levels == r["n_levels"]
        for l in range(p.n_levels):
            im, der = p.download(l, True)
            assert np.array_equal(sha256_u8(im), r["images"][l]) and np.array_equal(sha256_u8(der), r["derivs"][l]), l
    for p in pyrs:
        p.destroy()
    # the launch count does not grow with S
    for S in (1, 20):
        n0 = c.launch_count()
        pyrs = c.klt_pyramids([dict(frame=frames[1], derivatives=True)] * S)
        assert c.launch_count() - n0 == 5
        for p in pyrs:
            p.destroy()
    n0 = c.launch_count()
    assert c.klt_pyramids([]) == [] and c.launch_count() == n0                  # S == 0: no launch
    for f in frames:
        f.destroy()
    pool.destroy()


def test_rebuilt_handles_equal_fresh_builds():
    """Two handles rebuilt by batched calls, larger and smaller (60 x 40 -> 752 x 480 -> 1 x 1 with and without
    derivatives): after each call both equal fresh single builds."""
    c = gpu()
    imgs = {s: kc.pyr_image(*s) for s in ((60, 40), (752, 480), (1, 1), (645, 485))}
    frames = {s: c.frame_from_level0(img, 1) for s, img in imgs.items()}
    handles = [capi.KltPyramid(c), capi.KltPyramid(c)]
    rounds = [[((60, 40), False), ((752, 480), True)], [((752, 480), True), ((60, 40), False)],
              [((1, 1), False), ((645, 485), True)], [((645, 485), False), ((1, 1), True)]]
    for rd in rounds:
        c.klt_pyramids([dict(frame=frames[s], derivatives=d) for s, d in rd], handles)
        for h, (s, d) in zip(handles, rd):
            fresh = c.klt_pyramid(frames[s], d)
            assert h.n_levels == fresh.n_levels and digests(h, d) == digests(fresh, d), (s, d)
            fresh.destroy()
    for h in handles:
        h.destroy()
    for f in frames.values():
        f.destroy()


@pytest.mark.parametrize("S", [0, 1, 2, 33, 132, 257])
def test_shapes_over_shared_handles(S):
    """S streams over three shared pairs of handles, 1 to 40 points each, exit records in every other stream: one launch
    for S > 0 (none for S == 0), every stream equal to its single call (all of them up to 33 streams, 24 sampled above)."""
    c = gpu()
    cases = [kc.case("shift_640"), kc.case("iter_1"), ke.case("tiny_62x62")]
    pairs = [Pair(c, dict(k, levels=None, same_handle=False)) for k in cases]
    rng = np.random.default_rng(S)
    streams = []
    for s in range(S):
        p = pairs[s % 3]
        n = int(rng.integers(1, 41))
        idx = rng.choice(len(p.k["prev_pts"]), n)
        streams.append(p.args(pts=(p.k["prev_pts"][idx], p.k["next_pts"][idx]), want_exit=s % 2 == 0))
    out = batched(c, streams, 1 if S else 0)
    assert len(out) == S
    for s in (range(S) if S <= 33 else rng.choice(S, 24, replace=False)):
        same_as_single(c, streams[s], out[s])
    for p in pairs:
        p.destroy()


def test_partial_ctas():
    """A stream of 4097 points between streams of 1 and 3 points (4 points per CTA): each equals its single call."""
    c = gpu()
    p = Pair(c, dict(kc.case("shift_640"), levels=None, same_handle=False))
    rng = np.random.default_rng(4097)
    pts = [(rng.random((n, 2)) * [660, 500] - 10).astype(np.float32) for n in (1, 4097, 3)]
    streams = [p.args(pts=(q, q)) for q in pts]
    out = batched(c, streams)
    for a, b in zip(streams, out):
        same_as_single(c, a, b)
    p.destroy()


def test_refusals_write_nothing():
    """Each refusal returns SVO_B200_EINVAL with no launch, every stream's outputs keep the sentinels written before the
    call, and every handle keeps its levels and contents."""
    c = gpu()
    lib = c.lib
    k640, k752 = kc.case("iter_1"), kc.case("shift_752")
    pa, pb = Pair(c, dict(k640, levels=None, same_handle=False)), Pair(c, dict(k752, levels=None, same_handle=False))
    base = [pa.args(pts=(k640["prev_pts"][:20], k640["next_pts"][:20])), pb.args(pts=(k752["prev_pts"][:9], k752["next_pts"][:9])),
            pa.args(pts=(k640["prev_pts"][20:25], k640["next_pts"][20:25]), want_exit=False)]

    def prepared():
        prep = [capi._klt_prepare(**a) for a in base]
        for ks, (p1, st, ex, n), _ in prep:
            p1[:] = np.float32(-7.5)
            st[:] = 7
            if ex is not None:
                for e in ex:
                    e.reason = 99
        return prep

    def untouched(prep):
        for ks, (p1, st, ex, n), _ in prep:
            assert np.all(p1 == np.float32(-7.5)) and np.all(st == 7)
            assert ex is None or all(e.reason == 99 for e in ex)

    before = {id(p): digests(p, p is pa.prev or p is pb.prev) for p in (pa.prev, pa.next, pb.prev, pb.next)}
    bad_opts = [capi.KltOptions(31, 4, 30, 0.001), capi.KltOptions(30, -1, 30, 0.001), capi.KltOptions(30, 4, 30, -1e-9),
                capi.KltOptions(30, 4, 30, float("nan"))]
    # per stream: NULL pyramids, N < 0, a previous pyramid without derivatives, a next pyramid of another size, bad options
    mutations = [("prev", lambda s: None), ("next", lambda s: None), ("N", lambda s: -1), ("prev", lambda s: pa.next.h.value),
                 ("next", lambda s: (pa if s == 1 else pb).next.h.value)]
    mutations += [("opt", lambda s, o=o: C.cast(C.pointer(o), C.c_void_p).value) for o in bad_opts]
    for s in range(3):
        for field, value in mutations:
            prep = prepared()
            setattr(prep[s][0], field, value(s))
            arr = (capi.KltStream * 3)(*[p[0] for p in prep])
            n0 = c.launch_count()
            assert lib.svo_b200_klt_track_streams(c.h, 3, arr) == EINVAL, (s, field)
            assert c.launch_count() == n0
            assert f"stream {s}".encode() in lib.svo_b200_last_error(c.h)
            untouched(prep)
    prep = prepared()
    arr = (capi.KltStream * 3)(*[p[0] for p in prep])
    assert lib.svo_b200_klt_track_streams(c.h, -1, arr) == EINVAL and lib.svo_b200_klt_track_streams(c.h, 2, None) == EINVAL
    untouched(prep)
    n0 = c.launch_count()
    assert lib.svo_b200_klt_track_streams(c.h, 0, None) == 0 and c.launch_count() == n0
    # the build: a handle listed twice, a level cut past SVO_B200_MAX_LEVELS, S < 0, a NULL table
    big = c.frame_from_level0(np.zeros((7936, 7936), np.uint8), 1)
    fa = pa.frames[0]
    entries = [[(pa.prev, fa, 4, 1), (pb.next, fa, 4, 0), (pa.prev, fa, 2, 1)],
               [(pa.prev, fa, 4, 1), (pb.next, big, 8, 0)],
               [(pa.next, fa, 4, 0), (pb.prev, fa, -1, 1)],
               [(pa.next, fa, 4, 0), (pb.prev, fa, 4, 2)]]
    for e in entries:
        arr = (capi.KltBuild * len(e))(*[capi.KltBuild(p.h.value, f.h.value, m, d) for p, f, m, d in e])
        n0 = c.launch_count()
        assert lib.svo_b200_klt_pyramid_build_streams(c.h, len(e), arr) == EINVAL
        assert c.launch_count() == n0
    assert lib.svo_b200_klt_pyramid_build_streams(c.h, -1, arr) == EINVAL
    assert lib.svo_b200_klt_pyramid_build_streams(c.h, 1, None) == EINVAL
    for p in (pa.prev, pa.next, pb.prev, pb.next):
        assert digests(p, p is pa.prev or p is pb.prev) == before[id(p)]
    assert pa.prev.n_levels == 4 and pb.prev.n_levels == 4
    big.destroy()
    pa.destroy(); pb.destroy()


def test_host_streams_track_klt_equals_sequential_calls():
    """host_klt_streams_demo: six streams (pinhole and ATAN cameras, 752 x 480 and 640 x 480, two sharing one first
    keyframe) over three frames; svo::streams::trackKlt leaves px_ref, px_cur, f_ref, f_cur and the disparities exactly as
    one initialization::trackKlt call per stream leaves them, and every refusal throws with every vector unchanged."""
    from tests.test_host_cpp_gpu import build_demo

    out = subprocess.run([build_demo("host_klt_streams_demo")], capture_output=True, text=True, timeout=600)
    print(out.stdout, out.stderr)
    rows = {}
    refusal = None
    for line in out.stdout.splitlines():
        m = re.match(r"(sequential|batched)\s+([0-9a-f]{16}) points (\d+)$", line)
        if m:
            rows[m.group(1)] = (m.group(2), int(m.group(3)))
        m = re.match(r"refusals thrown (\d+) of (\d+) vectors (unchanged|changed)$", line)
        if m:
            refusal = (int(m.group(1)), int(m.group(2)), m.group(3))
    assert rows["sequential"] == rows["batched"] and rows["batched"][1] > 0
    tracked = [int(m.group(1)) for m in re.finditer(r"frame \d stream \d tracked (\d+)", out.stdout)]
    assert len(tracked) == 18 and min(tracked) > 0
    assert refusal == (4, 4, "unchanged")
    assert out.returncode == 0
