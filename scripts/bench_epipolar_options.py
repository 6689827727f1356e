"""The depth-filter launch of bench.py's C2 row (DepthFilter::updateSeeds, 2000 seeds, 752x480,
synth.make_depth_case(2031, 2000, baseline=0.3)) under four Matcher::Options settings:

  default        Matcher::Options() -- depth_filter_kernel<false>, the instantiation bench.py times
  general_0.7-   the general instantiation depth_filter_kernel<true> at the defaults but for an edgelet angle one double
                 below 0.7 (the setting that runs it while computing what the defaults compute, but for an edgelet whose
                 cosangle is exactly that double)
  align_1d       align1D along the epipolar line in place of align2D
  no_subpix      the scan's best step as the match, no alignment after the scan

Kernel time by CUDA events inside the library (svo_b200_last_kernel_ms), the settings alternated over --reps rounds after
--warmup rounds; medians in ms, with the card's name and power limit read in the same run.  One JSON line.

    python scripts/bench_epipolar_options.py [--reps 50] [--warmup 5]
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

SETTINGS = {
    "default": {},
    "general_0.7-": dict(edgelet_max_angle=float(np.nextafter(0.7, 0.0))),
    "align_1d": dict(align_1d=True),
    "no_subpix": dict(subpix_refinement=False),
}


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # the measurement still stands; the card is then unknown
        return {"error": str(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    ctx = capi.Context(0)
    c = synth.make_depth_case(2031, 2000, baseline=0.3)
    ref, cur = ctx.frame(c["ref_pyr"]), ctx.frame(c["cur_pyr"])
    dargs = ([ref], [c["T_ref_w"]], cur, c["T_cur_w"], c["cam"], c["ref_index"], c["ftr_px"], c["ftr_f"], c["ftr_level"],
             c["ftr_type"], c["ftr_grad"], c["batch_id"], c["batch_counter"], c["seeds"])
    times = {k: [] for k in SETTINGS}
    outs = {}
    for rnd in range(a.warmup + a.reps):
        for name, opt in SETTINGS.items():
            ctx.set_epipolar_options(**opt)
            outs[name] = ctx.depth_filter_update(*dargs)
            if rnd >= a.warmup:
                times[name].append(ctx.last_kernel_ms())
    ctx.set_epipolar_options()
    res = {name: {"kernel_ms_median": float(np.median(t)), "kernel_ms_min": float(np.min(t)),
                  "updated": int((outs[name]["status"] >= 5).sum()), "zmssd_evals": int(outs[name]["n_zmssd"].sum())}
           for name, t in times.items()}
    same = all(np.array_equal(outs["default"][k], outs["general_0.7-"][k]) for k in ("a", "b", "mu", "sigma2", "status"))
    print(json.dumps({"bench": "epipolar_options_C2", "seeds": 2000, "reps": a.reps, "card": card(), "settings": res,
                      "general_at_defaults_equals_default": bool(same)}))
    ref.destroy(); cur.destroy(); ctx.close()


if __name__ == "__main__":
    main()
