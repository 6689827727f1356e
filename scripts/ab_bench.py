#!/usr/bin/env python
"""A/B of libsvo_b200.so builds on the flagship workload: bench.py runs once per library per round, the libraries
alternating (SVO_B200_LIB), so that drift of the shared machine (clocks, power cap, neighbours) hits every arm alike.  Prints
per arm the `value` runs, their median and spread, `latency_B1`, `c4_32_per_gpu`, the `e2e` values, every
`roofline_by_kernel` row's `kernel_ms`, `pose_rmse_vs_ref` and the sampled clocks; then runs each library once more with --dump-outputs and compares every output array bit for bit against the
first library's.

   python scripts/ab_bench.py --rounds 3 parent=/path/to/parent.so new=rpg_svo_b200/libsvo_b200.so [-- extra bench.py args]

Run from the repository root on the GPU.  Everything it writes goes to --out (default: a temporary directory)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_bench(lib: str, args: list[str]) -> dict:
    env = dict(os.environ, SVO_B200_LIB=os.path.abspath(lib))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1"] + args, env=env, cwd=ROOT,
                         capture_output=True, text=True)
    if out.returncode != 0:
        raise SystemExit(f"bench.py failed with {lib}:\n{out.stderr[-3000:]}")
    return json.loads(out.stdout.strip().splitlines()[-1])


def bits(a: np.ndarray) -> np.ndarray:
    return a.view(np.uint64) if a.dtype.itemsize == 8 else a.view(np.uint32)


def main():
    argv = sys.argv[1:]
    extra = argv[argv.index("--") + 1:] if "--" in argv else []
    argv = argv[:argv.index("--")] if "--" in argv else argv
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("arms", nargs="+", help="name=path/to/libsvo_b200.so, the first is the reference of the bit comparison")
    a = ap.parse_args(argv)
    arms = [s.split("=", 1) for s in a.arms]
    out_dir = a.out or tempfile.mkdtemp(prefix="ab_bench_")
    runs = {name: [] for name, _ in arms}
    for _ in range(a.rounds):
        for name, lib in arms:
            runs[name].append(run_bench(lib, extra))
    for name, _ in arms:
        r = runs[name]
        v = np.array([x["value"] for x in r])
        med = float(np.median(v))
        print(json.dumps({"arm": name, "value": [round(x) for x in v], "median": round(med),
                          "spread_pct": round(100 * float(v.max() - v.min()) / med, 2),
                          "latency_B1_us": [round(x["latency_B1"]["device_us_per_pair"], 2) for x in r],
                          "c4_32_us": [round(x["c4_32_per_gpu"]["device_us_per_launch"], 2) for x in r],
                          "e2e": [round(x["e2e"]["value"]) if x.get("e2e") else None for x in r],
                          "roofline_kernel_ms": {k: [round(x["roofline_by_kernel"][k]["kernel_ms"], 4) for x in r]
                                                 for k in r[0].get("roofline_by_kernel", {})},
                          "pose_rmse_vs_ref": r[-1]["pose_rmse_vs_ref"], "clocks": [x["clocks"] for x in r]}))
    dump_args = ["--steps", "20", "--no-e2e", "--no-cpu", "--no-extras"]
    for name, lib in arms:
        run_bench(lib, dump_args + ["--dump-outputs", os.path.join(out_dir, name)])
    ref = arms[0][0]
    for name, _ in arms[1:]:
        for f in sorted(os.listdir(os.path.join(out_dir, ref))):
            x, y = np.load(os.path.join(out_dir, ref, f)), np.load(os.path.join(out_dir, name, f))
            same = x.shape == y.shape and np.array_equal(bits(x), bits(y))
            print(f"{name} vs {ref}: {f} {'bit-identical' if same else 'DIFFERENT'}")
    print("outputs in", out_dir)


if __name__ == "__main__":
    main()
