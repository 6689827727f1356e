"""Time one step of the two-view initialisation's KLT tracking (initialization::trackKlt) at 752 x 480 with about 350
points: the new frame's LK pyramid build plus the tracking launch, on the device; and OpenCV's calcOpticalFlowPyrLK on the
host (one thread and all threads) where OpenCV's Python module is installed.  Prints one JSON line with the card's name
and power limit (nvidia-smi) beside the figures.

usage: python scripts/bench_klt.py [--steps 200] [--warmup 20] [--points 350]
"""
import argparse
import json
import os
import platform
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rpg_svo_b200 import capi  # noqa: E402
from tests import klt_cases as kc  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--points", type=int, default=350)
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    prev, cur = kc._pair(rng, 752, 480)
    p0 = kc._pts(rng, a.points, 752, 480, 0.0)
    res = dict(workload=f"trackKlt step 752x480, {a.points} points, win 30, max_level 4, 30 iters, eps 0.001")

    ctx = capi.Context(0)
    fr, fc = ctx.frame_from_level0(prev, 1), ctx.frame_from_level0(cur, 1)
    pr = ctx.klt_pyramid(fr, True)
    pc = capi.KltPyramid(ctx)
    pyr_ms, trk_ms, wall = [], [], []
    for i in range(a.warmup + a.steps):
        ctx.synchronize()
        t0 = time.perf_counter()
        pc.build(fc, False)
        k0 = ctx.last_kernel_ms()
        g = ctx.klt_track(pr, pc, p0, p0, want_exit=False)
        t1 = time.perf_counter()
        if i >= a.warmup:
            pyr_ms.append(k0)
            trk_ms.append(ctx.last_kernel_ms())
            wall.append((t1 - t0) * 1e3)
    res.update(device_pyramid_ms=float(np.median(pyr_ms)), device_track_ms=float(np.median(trk_ms)),
               device_step_ms=float(np.median(np.add(pyr_ms, trk_ms))), host_wall_step_ms=float(np.median(wall)),
               tracked=int(g["status"].sum()), gpu=card())
    pr.destroy(); pc.destroy(); fr.destroy(); fc.destroy(); ctx.close()

    try:
        import cv2
    except ImportError:
        cv2 = None
    if cv2 is not None:
        crit = (cv2.TERM_CRITERIA_COUNT | cv2.TERM_CRITERIA_EPS, 30, 0.001)
        q = p0.reshape(-1, 1, 2)
        for nt, key in ((1, "opencv_1_thread_ms"), (cv2.getNumberOfCPUs(), "opencv_all_threads_ms")):
            cv2.setNumThreads(nt)
            ts = []
            for i in range(a.warmup + a.steps):
                t0 = time.perf_counter()
                cv2.calcOpticalFlowPyrLK(prev, cur, q, q.copy(), winSize=(30, 30), maxLevel=4, criteria=crit,
                                         flags=cv2.OPTFLOW_USE_INITIAL_FLOW)
                if i >= a.warmup:
                    ts.append((time.perf_counter() - t0) * 1e3)
            res[key] = float(np.median(ts))
        res.update(host_cpu=platform.processor() or platform.machine(), host_threads=cv2.getNumberOfCPUs())
    else:
        res["opencv"] = "not installed on this host: not measured"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
