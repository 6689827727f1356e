#!/usr/bin/env python
"""Static instruction count of one sia_kernel instantiation by PHASE of the kernel body (inlined callees are attributed to
the kernel-body line they were inlined at), plus local-memory (spill) instructions per phase.
   python scripts/sass_phases.py build/sparse_align.o 'sia_kernelILi2ELb0ELi160ELi3ELi1ELb0' """
import collections, os, re, subprocess, sys, tempfile
obj, pat = sys.argv[1], sys.argv[2]
tmp = tempfile.mkdtemp()
subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(obj)], cwd=tmp, check=True, capture_output=True)
cubin = [os.path.join(tmp, f) for f in os.listdir(tmp) if f.endswith(".cubin")][0]
txt = subprocess.run(["nvdisasm", "-gi", cubin], capture_output=True, text=True).stdout
src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "rpg_svo_b200", "csrc", "sparse_align.cu")).read().splitlines()
# phase boundaries from marker comments in the kernel body
def find(s):
    for i, l in enumerate(src):
        if s in l: return i + 1
    raise SystemExit("marker not found: " + s)
marks = [("prologue", find("__global__ void __launch_bounds__(MAXT, MINB) sia_kernel")),
         ("level_setup", find("for (int level = lvl_hi; level >= lvl_lo; --level)")),
         ("precompute", find("// ---- precomputeReferencePatches")),
         ("hsum+factor", find("pair_sum_h_to_warp0<FPT, CS, XG, SS, SH")),
         ("pass", find("// ---- Gauss-Newton iterations at this level")),
         ("reduce", find("// ---- pair-wide sums: per-warp transposed reduction")),
         ("tail", find("SIA_DBG(long long ti2 = 0;)")),
         ("eval/out", find("if (EVAL) {\n") if False else find("// ---- outputs ----")),
         ("end", find("// Host side"))]
def phase(ln):
    name = "other"
    for n, lo in marks:
        if ln >= lo: name = n
    return name
cur_fn, loc = None, None
cnt, spill, calls = collections.Counter(), collections.Counter(), collections.Counter()
for l in txt.splitlines():
    m = re.match(r"\s*\.section\s+\.text\.(\S+),", l)
    if m: cur_fn = m.group(1); loc = None; continue
    if cur_fn is None or pat not in cur_fn: continue
    if "//## File" in l:
        lines = [int(x) for f, x in re.findall(r'"([^"]+)", line (\d+)', l) if f.endswith("sparse_align.cu")]
        body = [x for x in lines if marks[0][1] <= x < marks[-1][1]]
        loc = body[-1] if body else (lines[-1] if lines else None)
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_]+)", l)
    if m:
        ph = phase(loc) if loc else "unknown"
        cnt[ph] += 1
        if m.group(1) in ("LDL", "STL"): spill[(ph, m.group(1))] += 1
        if m.group(1) == "CALL": calls[ph] += 1
tot = sum(cnt.values())
print(f"{pat}: {tot} instructions = {tot * 16 / 1024:.0f} KB")
for n, _ in marks[:-1] + [("other", 0), ("unknown", 0)]:
    if cnt[n]: print(f"  {n:14s} {cnt[n]:6d}  ({cnt[n] * 16 / 1024:5.1f} KB)  LDL {spill[(n, 'LDL')]:3d} STL {spill[(n, 'STL')]:3d} CALL {calls[n]:2d}")
