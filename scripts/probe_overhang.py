"""Per-launch overhang of back-to-back full-batch alignment launches (run on the GPU box): device time per launch of the
flagship workload's batch at B = 396 x {1, 2, 4, 8, 16} pairs -- whole waves of three 160-thread CTAs on each of 132 SMs --
each timed over about 0.5 s of back-to-back launches, and the fit T(B) = a*B + c.  c is what a launch costs beyond its
pairs' share of the wave time: the ramp, the drain of its last wave and the gap to the next launch.
   python scripts/probe_overhang.py            (SVO_B200_LIB selects another build of the library)"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from rpg_svo_b200 import capi

SIZES = [396 * m for m in (1, 2, 4, 8, 16)]
SECONDS = 0.5  # device time per size


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        row = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"card": row[0], "power_limit_w": float(row[1]), "sm_mhz": float(row[2]), "sm_max_mhz": float(row[3])}
    except Exception as e:  # the figures stand without it, but say why it is missing
        return {"card": torch.cuda.get_device_name(0), "nvidia_smi": repr(e)}


def main():
    Bmax = max(SIZES)
    inp = bench.make_inputs(0, Bmax, "cuda:0")
    ctx = capi.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", 0))
    pool = capi.FramePool(ctx, bench.W, bench.H, bench.NLEVELS, Bmax + 1)
    host_l0 = inp["level0"].cpu().pin_memory()
    pool.upload(0, Bmax + 1, host_l0.data_ptr(), bench.W * bench.H)
    ctx.synchronize()
    fr = pool.frames

    def timed(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            ctx.sia_batch_run()
        e1.record(stream)
        ctx.synchronize()
        return 1e3 * e0.elapsed_time(e1) / reps

    rows = []
    for B in SIZES:
        n = B * bench.NFEAT
        ctx.sia_batch_stage(fr[:B], fr[1:B + 1], inp["cam"], inp["T0"][:B], inp["off"][:B + 1], inp["px"][:n], inp["f"][:n],
                            inp["pos"][:n], inp["hp"][:n], inp["ref_pos"][:B], bench.MAX_LEVEL, bench.MIN_LEVEL, bench.NITER)
        timed(3)  # warm-up, and an estimate that sizes the timed window
        launch = ctx.sia_last_launch()
        reps = max(20, int(SECONDS / (timed(5) * 1e-6)))
        us = timed(reps)
        rows.append({"B": B, "us_per_launch": us, "reps": reps, "threads": launch["threads"],
                     "ctas_per_pair": launch["ctas_per_pair"]})
    info = gpu_info()
    Bs = np.array([r["B"] for r in rows], float)
    Ts = np.array([r["us_per_launch"] for r in rows])
    a, c = np.polyfit(Bs, Ts, 1)
    T3168 = float(np.interp(3168, Bs, Ts))
    for r in rows:
        r["fit_residual_us"] = float(r["us_per_launch"] - (a * r["B"] + c))
        print(json.dumps(r))
    print(json.dumps({"lib": os.environ.get("SVO_B200_LIB", "in-tree"), "a_us_per_pair": float(a), "c_us": float(c),
                      "T3168_us": T3168, "c_over_T3168": float(c) / T3168, **info}))


main()
