"""S single-stream calls against one multi-stream call of the depth filter, the reprojector, the FAST detector and the KLT
tracker, on one GPU.

Depth filter: C2-like streams (752x480, 2000 seeds each, one keyframe per stream).  Reprojector: the map of bench.py's
reprojector row (synth.make_map_case(4001, n_kfs=10, n_points=1200, n_candidates=150)) per stream; the streams cycle through
four maps of that shape (seeds 4001..4004).  FAST detector: the keyframe seeding of DepthFilter::initializeSeeds, one
752x480 keyframe with 3 pyramid levels per stream, 30-px cells, the cells of about 120 existing features occupied; the
streams cycle through four such keyframes.  KLT: one step of the two-view initialisation per stream (scripts/bench_klt.py's
workload: a 752x480 pair, 350 points, window 30, max_level 4), the new frame's LK pyramid build plus the tracking, against
a reference pyramid built once per stream; single = one pyramid build and one track call per stream, batched = one
svo_b200_klt_pyramid_build_streams and one svo_b200_klt_track_streams call; the streams cycle through four pairs.  Frames:
each stream's new frame (bench_frames), device and wall time as medians.  For
S = 1, 8, 32, 132 it times,
with CUDA events on the context's stream around the whole host call (staging, launch(es), copies back and, for the
reprojector and the detector, the host replay or decode), S back-to-back single calls and one batched call, alternating them; it reports the medians
of --reps runs after --warmup runs of each, the kernel-only time of the batched launch (svo_b200_last_kernel_ms; for KLT the
build's launches plus the tracking launch, from a run of their own), and
checks that both produce the same bits.  Prints one JSON line per (stage, S) and the card it ran on.

    python scripts/bench_streams.py [--reps 50] [--warmup 5] [--streams 1,8,32,132] [--stages depth_filter,reprojector,fast_detect,klt,frames]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rpg_svo_b200 import capi, synth  # noqa: E402
from tests import klt_cases as kc  # noqa: E402


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # the measurement still stands; the card is then unknown
        return {"error": str(e)}


def timed(ctx, fn) -> float:
    import torch

    s = torch.cuda.ExternalStream(ctx.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    out = fn()
    e1.record(s)
    e1.synchronize()
    return e0.elapsed_time(e1), out


def bench(ctx, name, single, batched, same, reps, warmup, S, kernel=None):
    """kernel: the batched call's device time from a run of its own, where it is more than the last entry point's kernels."""
    for _ in range(warmup):
        single(); batched()
    ts, tb, tk = [], [], []
    for _ in range(reps):
        t, a = timed(ctx, single)
        ts.append(t)
        t, b = timed(ctx, batched)
        tb.append(t)
        tk.append(ctx.last_kernel_ms() if kernel is None else kernel())
    assert same(a, b), f"{name} S={S}: batched results differ from single calls"
    r = dict(stage=name, S=S, single_calls_ms=float(np.median(ts)), batched_ms=float(np.median(tb)),
             batched_kernel_ms=float(np.median(tk)), speedup=float(np.median(ts) / np.median(tb)), reps=reps)
    print(json.dumps(r), flush=True)
    return r


def _frame_states(frames):
    return [(f.download_level(l).tobytes(), f.download_level_tiled(l).tobytes()) for f in frames for l in range(f.n_levels)]


def _timed_pair(ctx, fn):
    """(device ms from CUDA events around fn, wall ms from before fn to after a synchronise)."""
    import time

    import torch

    s = torch.cuda.ExternalStream(ctx.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record(s)
    fn()
    e1.record(s)
    ctx.synchronize()
    t1 = time.perf_counter()
    return e0.elapsed_time(e1), 1e3 * (t1 - t0)


def _frames_leg(ctx, name, single, batched, S, reps, warmup, extra):
    for _ in range(warmup):
        single(); batched()
    ds, ws, db, wb, ks, kb = [], [], [], [], [], []
    for _ in range(reps):
        d, w = _timed_pair(ctx, single)
        ds.append(d); ws.append(w); ks.append(ctx.last_kernel_ms())
        d, w = _timed_pair(ctx, batched)
        db.append(d); wb.append(w); kb.append(ctx.last_kernel_ms())
    med = lambda x: float(np.median(x))  # noqa: E731
    r = dict(stage=name, S=S, single_device_ms=med(ds), single_wall_ms=med(ws), batched_device_ms=med(db), batched_wall_ms=med(wb),
             single_last_kernel_ms=med(ks), batched_kernel_ms=med(kb), device_speedup=med(ds) / med(db),
             wall_speedup=med(ws) / med(wb), reps=reps, **extra)
    print(json.dumps(r), flush=True)
    return r


def bench_frames(ctx, Ss, reps, warmup):
    """S single svo_b200_frame_upload calls against one svo_b200_frame_upload_streams call: one 5-level frame per stream (what
    FrameHandlerMono builds: max(n_pyr_levels, klt_max_level + 1)), sizes cycling through 752x480, 640x480 and 644x484, level
    0 from pinned host buffers.  single_last_kernel_ms is the last single call's kernels (its S = 1 value is one upload).  Then
    one 64-frame window of a 7-level 752x480 pool: one svo_b200_frame_pool_upload against one batched call over its 64 frames."""
    import torch

    sizes = [(752, 480), (640, 480), (644, 484)]
    out = []
    for S in Ss:
        shapes = [sizes[s % 3] for s in range(S)]
        host = [torch.from_numpy(np.random.default_rng(900 + s).integers(0, 256, (h, w), dtype=np.uint8)).pin_memory()
                for s, (w, h) in enumerate(shapes)]
        fs = [capi.Frame(ctx, w, h, 5) for w, h in shapes]
        fb = [capi.Frame(ctx, w, h, 5) for w, h in shapes]

        def single(fs=fs, host=host):
            for f, im in zip(fs, host):
                f.upload_ptrs([im.data_ptr()])

        def batched(fb=fb, host=host):
            ctx.frames_upload([(f, im.data_ptr()) for f, im in zip(fb, host)])

        out.append(_frames_leg(ctx, "frames", single, batched, S, reps, warmup, {}))
        assert _frame_states(fs) == _frame_states(fb), f"frames S={S}: batched pyramids differ from single uploads"
        for f in fs + fb:
            f.destroy()
    pool_s, pool_b = capi.FramePool(ctx, 752, 480, 7, 64), capi.FramePool(ctx, 752, 480, 7, 64)
    host = torch.from_numpy(np.random.default_rng(964).integers(0, 256, (64, 480, 752), dtype=np.uint8)).pin_memory()
    ptrs = [host[i].data_ptr() for i in range(64)]
    out.append(_frames_leg(ctx, "frames_pool_window", lambda: pool_s.upload(0, 64, host.data_ptr(), 752 * 480),
                           lambda: ctx.frames_upload(list(zip(pool_b.frames, ptrs))), 64, reps, warmup,
                           dict(note="single = one frame_pool_upload of a 64-frame 7-level 752x480 window")))
    assert _frame_states(pool_s.frames) == _frame_states(pool_b.frames), "pool window: batched pyramids differ"
    pool_s.destroy(); pool_b.destroy()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--streams", default="1,8,32,132")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    ap.add_argument("--stages", default="depth_filter,reprojector,fast_detect,klt,frames")
    a = ap.parse_args()
    Ss = [int(x) for x in a.streams.split(",")]
    stages = a.stages.split(",")
    ctx = capi.Context(0)
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    results = [dict(card=info)]

    # ---- depth filter: C2-like streams ----
    if "depth_filter" in stages:
        scenes = [synth.make_depth_case(500 + k) for k in range(4)]
        frames = [(ctx.frame(c["ref_pyr"]), ctx.frame(c["cur_pyr"])) for c in scenes]
        for S in Ss:
            sc = [scenes[s % 4] for s in range(S)]
            fr = [frames[s % 4] for s in range(S)]
            keys = ("ftr_px", "ftr_f", "ftr_level", "ftr_type", "ftr_grad", "batch_id")

            def single(sc=sc, fr=fr):
                return [ctx.depth_filter_update([f[0]], [c["T_ref_w"]], f[1], c["T_cur_w"], c["cam"], c["ref_index"],
                                                *[c[k] for k in keys], c["batch_counter"], c["seeds"]) for c, f in zip(sc, fr)]

            streams = [dict(cur=f[1], cur_T_f_w=c["T_cur_w"], cam=c["cam"], batch_counter=c["batch_counter"],
                            ref_index=np.full(c["M"], s % 4, np.int32), seeds=c["seeds"], **{k: c[k] for k in keys})
                       for s, (c, f) in enumerate(zip(sc, fr))]

            def batched(streams=streams):
                return ctx.depth_filter_update_streams(streams, [f[0] for f in frames], [c["T_ref_w"] for c in scenes])

            def same(x, y):
                return all(np.ascontiguousarray(p[k]).tobytes() == np.ascontiguousarray(q[k]).tobytes()
                           for p, q in zip(x, y) for k in ("a", "b", "mu", "sigma2", "status", "px_cur", "z", "n_zmssd"))

            results.append(bench(ctx, "depth_filter", single, batched, same, a.reps, a.warmup, S))

    # ---- reprojector: bench.py's map per stream ----
    if "reprojector" in stages:
        maps = [synth.make_map_case(4001 + k, n_kfs=10, n_points=1200, n_candidates=150) for k in range(4)]
        mfr = [([ctx.frame(p) for p in m["kf_pyr"]], ctx.frame(m["cur_pyr"])) for m in maps]
        for S in Ss:
            args = [dict(view=maps[s % 4]["view"], kf_frames=mfr[s % 4][0], cur=mfr[s % 4][1], cur_T_f_w=maps[s % 4]["cur_T_f_w"],
                         cam=maps[s % 4]["cam"], options=maps[s % 4]["options"], cell_order=maps[s % 4]["cell_order"],
                         pt_type=maps[s % 4]["pt_type"], pt_n_failed=maps[s % 4]["pt_n_failed"],
                         pt_n_succeeded=maps[s % 4]["pt_n_succeeded"]) for s in range(S)]

            def single(args=args):
                return [ctx.reproject_map(**x) for x in args]

            def batched(args=args):
                return ctx.reproject_map_streams(args)

            def same(x, y):
                return all((np.ascontiguousarray(p[k]).tobytes() == np.ascontiguousarray(q[k]).tobytes())
                           if isinstance(p[k], np.ndarray) else p[k] == q[k] for p, q in zip(x, y) for k in p)

            results.append(bench(ctx, "reprojector", single, batched, same, a.reps, a.warmup, S))

    # ---- FAST detector: keyframe seeding ----
    if "fast_detect" in stages:
        kfs = []
        for k in range(4):
            pyr = synth.make_two_view(600 + k, n_levels=3)["ref_pyr"]
            rng = np.random.default_rng(600 + k)
            occ = np.zeros(26 * 16, np.uint8)                                       # ceil(752/30) x ceil(480/30) cells
            px = rng.uniform([0, 0], [752, 480], (120, 2)).astype(int)             # the keyframe's existing features
            occ[(px[:, 1] // 30) * 26 + px[:, 0] // 30] = 1
            kfs.append((ctx.frame(pyr), occ))
        for S in Ss:
            args = [dict(frame=kfs[s % 4][0], cell_size=30, n_pyr_levels=3, detection_threshold=20.0, grid_occupancy=kfs[s % 4][1])
                    for s in range(S)]

            def single(args=args):
                return [ctx.fast_detect(**x) for x in args]

            def batched(args=args):
                return ctx.fast_detect_streams(args)

            def same(x, y):
                return all(p["n"] == q["n"] and all(p[k].tobytes() == q[k].tobytes() for k in ("x", "y", "level", "score"))
                           for p, q in zip(x, y))

            results.append(bench(ctx, "fast_detect", single, batched, same, a.reps, a.warmup, S))

    # ---- KLT: one step of the two-view initialisation per stream (scripts/bench_klt.py's workload) ----
    if "klt" in stages:
        pairs = []
        for k in range(4):
            rng = np.random.default_rng(700 + k)
            prev, cur = kc._pair(rng, 752, 480)
            p0 = kc._pts(rng, 350, 752, 480, 0.0)
            fr, fc = ctx.frame_from_level0(prev, 1), ctx.frame_from_level0(cur, 1)
            pairs.append((fr, fc, ctx.klt_pyramid(fr, True), p0))                  # the reference pyramid: built once
        for S in Ss:
            prs = [pairs[s % 4] for s in range(S)]
            own = [capi.KltPyramid(ctx) for _ in range(S)]                          # each stream's new-frame pyramid

            def single(prs=prs, own=own):
                out = []
                for (_, fc, pr, p0), pc in zip(prs, own):
                    pc.build(fc, False)
                    out.append(ctx.klt_track(pr, pc, p0, p0, want_exit=False))
                return out

            def batched(prs=prs, own=own):
                ctx.klt_pyramids([dict(frame=x[1], derivatives=False) for x in prs], own)
                return ctx.klt_track_streams([dict(prev=pr, nxt=pc, prev_pts=p0, next_pts=p0, want_exit=False)
                                              for (_, _, pr, p0), pc in zip(prs, own)])

            def kernel(prs=prs, own=own):  # the build's launches plus the tracking launch
                ctx.klt_pyramids([dict(frame=x[1], derivatives=False) for x in prs], own)
                k = ctx.last_kernel_ms()
                ctx.klt_track_streams([dict(prev=pr, nxt=pc, prev_pts=p0, next_pts=p0, want_exit=False)
                                       for (_, _, pr, p0), pc in zip(prs, own)])
                return k + ctx.last_kernel_ms()

            def same(x, y):
                return all(p[k].tobytes() == q[k].tobytes() for p, q in zip(x, y) for k in ("next_pts", "status"))

            results.append(bench(ctx, "klt", single, batched, same, a.reps, a.warmup, S, kernel))
            for pc in own:
                pc.destroy()
    # ---- frames: every stream's new frame, level 0 from pinned host memory, pyramid on the device ----
    if "frames" in stages:
        results += bench_frames(ctx, Ss, a.reps, a.warmup)
    if a.out:
        with open(a.out, "w") as f:
            for r in results:
                f.write(json.dumps(r) + "\n")
    ctx.close()


if __name__ == "__main__":
    main()
