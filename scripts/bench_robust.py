"""Device time of the robust alignment kernel (MAD scale, Tukey weights) against the unweighted one on the same pairs.

One synthetic 640x480 pair with 300 features (levels 4..0, 30 iterations at most), run as one pair, as a batch of 32 pairs
and as a full batch of 3168 pairs (every pair of a batch is the same pair).  The time is the library's CUDA-event time around
the kernel launch (Context.last_kernel_ms), median over --reps launches after --warmup; prints one JSON line with the GPU's
name, power limit and maximum SM clock.

    python scripts/bench_robust.py [--reps 50] [--warmup 5]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rpg_svo_b200 import capi, synth  # noqa: E402


def gpu_conditions() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = (x.strip() for x in q[0].split(",")) if q else ("?", "?", "?")
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def time_batch(ctx, d, ref, cur, B, robust, reps, warmup) -> float:
    ctx.sia_robust(capi.SCALE_MAD if robust else capi.SCALE_UNIT, capi.WEIGHT_TUKEY)
    n = len(d["px"])
    off = np.arange(B + 1, dtype=np.int32) * n
    rep = lambda a: np.ascontiguousarray(np.tile(a, (B,) + (1,) * (a.ndim - 1)))  # noqa: E731
    T0 = np.tile(synth.se3_identity().reshape(1, 12), (B, 1))
    ctx.sia_batch_stage([ref] * B, [cur] * B, d["cam"], T0, off, rep(d["px"]), rep(d["f"]), rep(d["pos"]), rep(d["has_point"]),
                        np.tile(d["ref_pos"], (B, 1)), 4, 0, 30)
    ms = []
    for k in range(warmup + reps):
        ctx.sia_batch_run()
        ctx.synchronize()
        if k >= warmup:
            ms.append(ctx.last_kernel_ms())
    assert (ctx.sia_last_launch()["threads"] == 256) == robust  # the robust kernel runs 256 threads, no sia_kernel geometry does
    return float(np.median(ms))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    d = synth.make_frame_pair(2024, n_feat=300)
    ctx = capi.Context(0)
    ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
    out = dict(gpu_conditions(), features=300, levels="4..0", weight="tukey", scale="mad")
    for B in (1, 32, 3168):
        for robust in (False, True):  # alternated per batch size in one process
            ms = time_batch(ctx, d, ref, cur, B, robust, a.reps, a.warmup)
            key = f"{'robust' if robust else 'plain'}_B{B}"
            out[key + "_ms"] = round(ms, 4)
            out[key + "_us_per_pair"] = round(1e3 * ms / B, 3)
    ctx.sia_robust(capi.SCALE_UNIT, capi.WEIGHT_UNIT)
    ref.destroy(); cur.destroy(); ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
