"""GPU: svo_b200_fast_detect_streams -- S streams' FastDetector::detect in one launch -- against S single calls of
svo_b200_fast_detect and against the oracle, bit for bit (scores as float32 bits), over streams that differ in frame size,
pyramid depth, cell size, FAST threshold b, tie mode, detection threshold, occupancy and cap; streams that share frame
handles or use frame-pool frames; shapes up to 257 streams; and every refusal, which must launch and write nothing."""
import ctypes as C

import numpy as np
import pytest

from rpg_svo_b200 import capi, synth
from tests import fast_numpy
from tests.ref_golden import ref  # noqa: F401 (ref: fixture)

pytestmark = pytest.mark.gpu

OUT_KEYS = ("x", "y", "level", "score")


def _n_cells(w, h, cell):
    return int(np.ceil(w / cell)) * int(np.ceil(h / cell))


def _same(g, b, score=True):
    assert g["n"] == b["n"]
    for k in OUT_KEYS if score else OUT_KEYS[:3]:
        assert g[k].dtype == b[k].dtype and g[k].tobytes() == b[k].tobytes(), k


def _streams_call(ctx, streams, null_score=()):
    """fast_detect_streams through raw ctypes, score_out NULL for the streams in null_score (their score arrays must stay
    zero); returns one dict per stream, as fast_detect returns."""
    prep = [capi._detect_prepare(**s) for s in streams]
    for s in null_score:
        prep[s][0].score_out = None
    arr = (capi.DetectStream * max(len(prep), 1))(*[p[0] for p in prep])
    n0 = ctx.launch_count()
    ctx._check(ctx.lib.svo_b200_fast_detect_streams(ctx.h, len(prep), arr))
    assert ctx.launch_count() == n0 + (1 if prep else 0)                         # one launch for every stream
    out = [capi._detect_result(o, n) for _, o, n, _ in prep]
    for s in null_score:
        assert not out[s]["score"].any()
    return out


def _pyramid(fr):
    return [fr.download_level(l) for l in range(fr.n_levels)]


def _heterogeneous(ctx):
    """(frames to free, pool, stream dicts): one stream per row below, options chosen to reach every branch."""
    imgs = {}
    for key, (w, h, seed) in {"752": (752, 480, 21), "640": (640, 480, 22), "644": (644, 484, 23), "1080p": (1920, 1080, 24),
                              "97": (97, 61, 25)}.items():
        imgs[key] = synth.make_two_view(seed, width=w, height=h, n_levels=4)["ref_pyr"]
    imgs["flat"] = synth.build_pyramid(np.full((120, 160), 77, np.uint8), 3)
    noise = np.random.default_rng(11).integers(0, 256, (240, 320), dtype=np.uint8)
    noise[100:140, 100:200] = 128                                                   # a flat region: no corners
    imgs["noise"] = synth.build_pyramid(noise, 3)
    imgs["checker"] = fast_numpy.images(3, 160, 120)["checker"]                 # every corner scores 254
    frames = {k: ctx.frame(p) for k, p in imgs.items()}
    pool = capi.FramePool(ctx, 752, 480, 4, 2)
    pool.upload_array(np.stack([imgs["752"][0], synth.make_two_view(26, n_levels=4)["ref_pyr"][0]]))
    frames["pool0"], frames["pool1"] = pool.frames
    rng = np.random.default_rng(5)

    def occ(key, cell, kind):
        f = frames[key]
        n = _n_cells(f.width, f.height, cell)
        return None if kind is None else np.ones(n, np.uint8) if kind == "full" else (rng.uniform(size=n) < kind).astype(np.uint8)

    rows = [  # frame, cell, levels, threshold, occupancy, b, ties, cap
        ("752", 30, 3, 20.0, None, 20, 0, 8192),
        ("752", 16, 4, 0.0, 0.3, 0, 1, 8192),                                      # the same handle, other options
        ("640", 50, 2, 150.0, None, 20, 0, 8192),
        ("644", 60, 1, -0.0, 0.5, 20, 1, 8192),
        ("1080p", 30, 4, 20.0, 0.2, 20, 0, 8192),
        ("1080p", 16, 3, 1e30, None, 20, 1, 8192),                                  # every cell emits the placeholder
        ("97", 16, 4, 0.0, None, 0, 0, 8192),
        ("97", 50, 2, 20.0, "full", 20, 0, 8192),                                   # fully occupied: nothing
        ("flat", 30, 3, 20.0, None, 20, 0, 8192),                                   # no corner at all
        ("noise", 16, 3, 20.0, None, 20, 1, 8192),
        ("checker", 16, 3, 0.0, 0.4, 254, 0, 8192),                                # b = 254 leaves corners here only
        ("noise", 50, 2, 150.0, None, 0, 1, 8192),
        ("noise", 60, 3, 0.0, None, 20, 0, 0),                                      # cap 0: only n
        ("noise", 16, 2, 0.0, None, 20, 0, 7),                                      # cap below the corner count
        ("pool0", 30, 3, 20.0, 0.25, 20, 0, 8192),
        ("pool1", 30, 4, 0.0, None, 20, 1, 8192),
        ("pool0", 50, 4, float(np.float32(1e30)), None, 20, 0, 8192),              # at exactly float32(1e30): none
        ("640", 30, 3, 20.0, "full", 0, 1, 8192),
        ("checker", 30, 2, 0.0, None, 254, 1, 8192),
    ]
    streams = [dict(frame=frames[f], cell_size=c, n_pyr_levels=L, detection_threshold=t, grid_occupancy=occ(f, c, o),
                    fast_threshold=b, nonmax_ties_suppress=ties, cap=cap) for f, c, L, t, o, b, ties, cap in rows]
    return [frames[k] for k in imgs], pool, streams


def test_detect_streams_heterogeneous_equal_single_calls(ctx, oracle):
    frames, pool, streams = _heterogeneous(ctx)
    singles = [ctx.fast_detect(**s) for s in streams]
    null_score = (2, 7, 10)
    batched = _streams_call(ctx, streams, null_score)
    for s, (g, b) in enumerate(zip(singles, batched)):
        _same(g, b, score=s not in null_score)
    assert _streams_call(ctx, streams[:1])[0]["n"] == singles[0]["n"]
    n = [g["n"] for g in singles]
    assert n[5] == _n_cells(1920, 1080, 16) and not singles[5]["x"].any()        # placeholders
    assert n[7] == n[8] == n[16] == n[17] == 0 and n[12] > 0 and n[13] > 7 and len(batched[13]["x"]) == 7
    assert min(n[i] for i in (0, 1, 2, 3, 4, 6, 9, 10, 11, 14, 15)) > 0       # 18: equal checker corners all suppressed
    # every stream also equals the oracle on the pyramid the device holds
    for s, (st, g) in enumerate(zip(streams, singles)):
        o = oracle.fast_detect(_pyramid(st["frame"]), st["n_pyr_levels"], st["cell_size"], st["detection_threshold"],
                               st["grid_occupancy"], cap=8192, nonmax_ties_suppress=st["nonmax_ties_suppress"],
                               fast_threshold=st["fast_threshold"])
        k = min(st["cap"], len(o["x"]))
        assert g["n"] == len(o["x"]), s
        for key in OUT_KEYS:
            assert g[key].tobytes() == o[key][:k].tobytes(), (s, key)
    for f in frames:
        f.destroy()
    pool.destroy()


def _ref_case():
    d = synth.make_two_view(31, n_levels=5)
    occ = (np.random.default_rng(3).uniform(size=26 * 16) < 0.3).astype(np.uint8)
    return d["ref_pyr"], occ


def test_detect_streams_vs_compiled_reference(ctx, ref):
    pyr, occ = _ref_case()
    fr = ctx.frame(pyr)
    other = ctx.frame(synth.build_pyramid(np.random.default_rng(4).integers(0, 256, (240, 320), dtype=np.uint8), 3))
    b = ctx.fast_detect_streams([dict(frame=other, cell_size=16, n_pyr_levels=2, detection_threshold=0.0),
                                 dict(frame=fr, cell_size=30, n_pyr_levels=3, detection_threshold=20.0, grid_occupancy=occ)])[1]
    r = ref.fast_detect(pyr[0], 5, 3, 30, 20.0, occ)
    assert b["n"] == len(r["x"]) > 100
    for k in ("x", "y", "level"):
        assert np.array_equal(b[k], r[k]), k
    fr.destroy(); other.destroy()


@pytest.mark.parametrize("S", [0, 1, 2, 33, 132, 257])
def test_detect_streams_shapes(ctx, S):
    """S streams over three frames they share (one of them a pool frame), options and occupancy drawn per stream."""
    pyrs = [synth.make_two_view(40 + k, width=w, height=h, n_levels=4)["ref_pyr"]
            for k, (w, h) in enumerate([(752, 480), (640, 480), (644, 484)])]
    own = [ctx.frame(p) for p in pyrs[1:]]
    pool = capi.FramePool(ctx, 752, 480, 4, 1)
    pool.upload_array(pyrs[0][0][None])
    frames = [pool.frames[0]] + own
    rng = np.random.default_rng(S)
    streams = []
    for s in range(S):
        f = frames[s % 3]
        cell = int(rng.choice([16, 30, 50, 60]))
        streams.append(dict(frame=f, cell_size=cell, n_pyr_levels=int(rng.integers(1, 5)),
                            detection_threshold=float(rng.choice([0.0, 20.0, 150.0])),
                            grid_occupancy=(rng.uniform(size=_n_cells(f.width, f.height, cell)) < 0.3).astype(np.uint8)
                            if rng.uniform() < 0.5 else None,
                            fast_threshold=int(rng.choice([0, 20, 254])), nonmax_ties_suppress=int(rng.integers(0, 2)),
                            cap=int(rng.choice([0, 5, 8192]))))
    singles = [ctx.fast_detect(**s) for s in streams]
    n0 = ctx.launch_count()
    batched = ctx.fast_detect_streams(streams)
    assert ctx.launch_count() == n0 + (S > 0)
    assert len(batched) == S
    for g, b in zip(singles, batched):
        _same(g, b)
    for f in own:
        f.destroy()
    pool.destroy()


def test_detect_streams_refusals_write_nothing(ctx):
    pyr = synth.make_two_view(50, width=320, height=240, n_levels=3)["ref_pyr"]
    fr = ctx.frame(pyr)

    def base():
        return [dict(frame=fr, cell_size=30, n_pyr_levels=3, detection_threshold=0.0),
                dict(frame=fr, cell_size=16, n_pyr_levels=2, detection_threshold=20.0, grid_occupancy=np.zeros(300, np.uint8)),
                dict(frame=fr, cell_size=50, n_pyr_levels=1, detection_threshold=0.0)]

    bads = [dict(cell_size=0), dict(n_pyr_levels=4), dict(n_pyr_levels=0), dict(fast_threshold=255), dict(fast_threshold=-1),
            dict(detection_threshold=-1.0), dict(detection_threshold=float("nan"))]
    cases = [(1, b) for b in bads] + [(1, "null frame"), (2, "null x_out"), (0, "null n_out"), (2, "cap -1")]
    for j, (i, bad) in enumerate(cases):
        args = base()
        if isinstance(bad, dict):
            args[i].update(bad)
        prep = [capi._detect_prepare(**a) for a in args]
        for _, o, n, _ in prep:
            for v in o.values():
                v[...] = 77
            n.value = 77
        if bad == "null frame":
            prep[i][0].frame = None
        elif bad == "null x_out":
            prep[i][0].x_out = None
        elif bad == "null n_out":
            prep[i][0].n_out = None
        elif bad == "cap -1":
            prep[i][0].cap = -1
        arr = (capi.DetectStream * 3)(*[p[0] for p in prep])
        for call in ("streams", "single"):
            n0 = ctx.launch_count()
            if call == "streams":
                rc = ctx.lib.svo_b200_fast_detect_streams(ctx.h, 3, arr)
            else:
                ds = prep[i][0]
                rc = ctx.lib.svo_b200_fast_detect(ctx.h, *[C.c_void_p(getattr(ds, f)) if f != "cap" else ds.cap
                                                           for f, _ in capi.DetectStream._fields_])
            assert rc == -1, (j, call)                                               # SVO_B200_EINVAL
            assert ctx.launch_count() == n0, (j, call)
            for _, o, n, _ in prep:
                assert n.value == 77, (j, call)
                for k, v in o.items():
                    assert np.all(v == 77), (j, call, k)
    n0 = ctx.launch_count()
    assert ctx.lib.svo_b200_fast_detect_streams(ctx.h, -1, None) == -1
    assert ctx.lib.svo_b200_fast_detect_streams(ctx.h, 2, None) == -1
    arr = (capi.DetectStream * 1)(capi._detect_prepare(**base()[0])[0])
    assert ctx.lib.svo_b200_fast_detect_streams(ctx.h, -1, arr) == -1
    assert ctx.lib.svo_b200_fast_detect_streams(ctx.h, 0, None) == 0
    assert ctx.lib.svo_b200_fast_detect_streams(ctx.h, 0, arr) == 0
    assert ctx.launch_count() == n0
    with pytest.raises(capi.SvoB200Error):
        ctx.fast_detect_streams([dict(frame=fr, cell_size=30, n_pyr_levels=5, detection_threshold=0.0)])
    fr.destroy()
