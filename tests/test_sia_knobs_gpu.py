"""GPU: the alignment kernel's opt-in SVO_B200_SIA_* knobs, each in a child process of its own (the library reads them once
per process), against the oracle and -- where a knob only moves data or changes residency -- bit for bit against the
child with the default knobs.  Also: every instantiation launch_sia can dispatch to, and every staging mode, was reached.

The children run tests/sia_knob_child.py and exit when it is done; nothing is left running."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import sia_cases as sc
from tests import sia_knob_child as child

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

KNOBS = {"default": {}, "BQ=1": {"SVO_B200_SIA_BQ": "1"}, "FPT2=2": {"SVO_B200_SIA_FPT2": "2"},
         "FPT2=0": {"SVO_B200_SIA_FPT2": "0"}, "MINB=3": {"SVO_B200_SIA_MINB": "3"}, "WINDOWS=0": {"SVO_B200_SIA_WINDOWS": "0"},
         "PREFETCH=0": {"SVO_B200_SIA_PREFETCH": "0"}, "ASYNC=0": {"SVO_B200_SIA_ASYNC": "0"},
         "PLAIN=0": {"SVO_B200_SIA_PLAIN": "0"}, "UPFRONT=0": {"SVO_B200_SIA_UPFRONT": "0"},
         "STAGE_KB=1": {"SVO_B200_SIA_STAGE_KB": "1"}, "STAGE_KB=64": {"SVO_B200_SIA_STAGE_KB": "64"}}
# Knobs that change where data is staged, how the sums travel, how many CTAs an SM holds or which camera code is compiled
# (the undistorted pinhole's projection is the same fma in both): same instantiation geometry, hence the same arithmetic in
# the same order -- results bit-identical with the default child.  The patch cache (BQ) rebuilds dx, dy from the cached
# bilinear rows with the same __fmul_rn / __fsub_rn the patch precomputation uses.  FPT2=0 and UPFRONT=0 instead move the
# automatic choice to another geometry (320 x 1 instead of 160 x 2; the per-level instead of the upfront cluster flow): other
# warps sum other features, so those launches agree with the default to rounding only -- the oracle's tolerances apply,
# and every launch whose geometry did not change must still be bit-identical.
BIT_IDENTICAL = {"BQ=1", "FPT2=2", "MINB=3", "WINDOWS=0", "PREFETCH=0", "ASYNC=0", "PLAIN=0", "STAGE_KB=1", "STAGE_KB=64"}


@pytest.fixture(scope="module")
def children(tmp_path_factory):
    out = {}
    base_env = {k: v for k, v in os.environ.items() if not k.startswith("SVO_B200_SIA_")}
    d = tmp_path_factory.mktemp("sia_knobs")
    for name, knob in KNOBS.items():
        path = str(d / (name.replace("=", "_") + ".npz"))
        p = subprocess.run([sys.executable, "-m", "tests.sia_knob_child", path], cwd=ROOT, env=dict(base_env, **knob),
                           capture_output=True, text=True, timeout=600)
        assert p.returncode == 0, f"{name}: exit {p.returncode}\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}"
        with np.load(path, allow_pickle=False) as z:
            out[name] = ({k: z[k] for k in z.files if k != "launches"}, json.loads(str(z["launches"])))
    return out


@pytest.fixture(scope="module")
def oracle_results(oracle):
    res = {}
    for name, d in child.cases().items():
        res[name] = sc.oracle_run(oracle, d)
        lv = child.RES_LEVEL[name]
        res[name + "/res"] = oracle.sparse_residuals(d["ref_pyr"][lv], d["cur_pyr"][lv], lv, d["cam"], d["T_gt"], d["px"], d["f"],
                                                     d["pos"], d["has_point"], d["ref_pos"])
    base = sc.base_pair()
    res["batch64"] = [sc.oracle_run(oracle, p) for p in child.batch_parts(base)]
    return res


def _geom(L):
    return (L["ctas_per_pair"], L["threads"], L["features_per_thread"], bool(L["upfront"]))


def _g(arrays, key):
    tr = [dict(level=int(a[0]), iter=int(a[1]), accepted=int(a[2]), n_meas=int(a[3]), chi2=float(c))
          for a, c in zip(arrays[key + "/trace_i"], arrays[key + "/trace_chi2"])]
    return dict(T=arrays[key + "/T"], visible=arrays[key + "/visible"], n_tracked=int(arrays[key + "/n_tracked"]), trace=tr)


def _took_effect(name, L, D):
    """The knob is visible in the launch records (L: this child's, D: the default child's)."""
    if name == "BQ=1":
        assert L["batch64"]["patch_cache"] == 1 and L["batch64"]["min_blocks"] == 4
        assert L["pair300/cta-2fpt"]["patch_cache"] == 1 and L["atan/cta-2fpt"]["patch_cache"] == 1
    elif name == "FPT2=2":
        assert _geom(L["batch64"]) == (1, 160, 2, False) and L["batch64"]["stage_cap"] > D["batch64"]["stage_cap"]
    elif name == "FPT2=0":
        assert _geom(L["batch64"]) == (1, 320, 1, False)
    elif name == "MINB=3":
        assert L["pair300/cta-1fpt"]["min_blocks"] == 3 and L["pair300/cta-1fpt/res"]["min_blocks"] == 3
    elif name == "WINDOWS=0":
        assert D["pair300/cta-1fpt"]["stages"]["0"] == "window" and L["pair300/cta-1fpt"]["stages"]["0"] == "global"
        assert all(m != "window" for r in L.values() for m in r["stages"].values())
    elif name == "PREFETCH=0":
        assert all(r["prefetch"] == 0 for r in L.values()) and all(r["prefetch"] == 1 for r in D.values())
    elif name == "ASYNC=0":
        assert D["pair300/auto"]["async_exchange"] == 1 and L["pair300/auto"]["async_exchange"] == 0
        assert L["pair300/auto"]["upfront"] == 1
    elif name == "PLAIN=0":
        assert D["pair300/auto"]["general_camera"] == 0 and all(r["general_camera"] == 1 for r in L.values())
    elif name == "UPFRONT=0":
        assert _geom(D["pair300/auto"]) == (4, 96, 1, True) and _geom(L["pair300/auto"]) == (4, 96, 1, False)
    elif name == "STAGE_KB=1":
        assert D["pair300/auto"]["stages"]["2"] == "image" and L["pair300/auto"]["stages"]["2"] != "image"
    elif name == "STAGE_KB=64":
        assert L["pair300/auto"]["stage_cap"] == 64 * 1024 > D["pair300/auto"]["stage_cap"]


def _same_bits(a, b):
    """Equal bit for bit (NaN residuals included)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("name", list(KNOBS))
def test_knob(children, oracle_results, name):
    A, L = children[name]
    DA, D = children["default"]
    assert set(L) == set(D) and set(A) == set(DA)
    _took_effect(name, L, D)
    # oracle parity of every case, configuration and residual pass
    for key, rec in L.items():
        case = key.split("/")[0]
        if key == "batch64":
            off = A["batch64/offsets"]
            for k, o in enumerate(oracle_results["batch64"]):
                g = dict(T=A["batch64/T"][k], visible=A["batch64/visible"][off[k]:off[k + 1]], n_tracked=int(A["batch64/n_tracked"][k]))
                sc.assert_parity(g, o, n_feat=int(off[k + 1] - off[k]))
        elif key.endswith("/res"):
            g = {k: A[f"{key}/{k}"] for k in ("visible", "in_image", "ref_patch", "residuals")}
            g["n_meas"] = int(A[f"{key}/n_meas"])
            sc.assert_residual_parity(g, oracle_results[case + "/res"])
        else:
            sc.assert_parity(_g(A, key), oracle_results[case])
    # bit identity with the default child wherever the instantiation geometry is the same
    changed = [k for k in L if _geom(L[k]) != _geom(D[k])]
    if name in BIT_IDENTICAL:
        assert not changed, changed
    for arr in A:
        key = arr.rsplit("/", 1)[0]
        launch = "batch64" if key.startswith("batch64") else key
        if launch in changed:
            continue
        a, b = A[arr], DA[arr]
        if arr.endswith("/res/ref_patch"):
            # the patch cache is defined for visible features only: the rows of the others are whatever the shared memory
            # behind them held (the reference leaves its cv::Mat cache uninitialised there as well), which depends on the
            # shared-memory layout a knob selects
            v = DA[key + "/visible"].astype(bool)
            a, b = a[v], b[v]
        assert _same_bits(a, b), (name, arr)


# ---- every instantiation and every staging mode was reached ------------------------------------------------------------
def _inst(r):
    return (r["residuals_only"], r["ctas_per_pair"], r["threads"], r["features_per_thread"], r["min_blocks"], r["general_camera"],
            r["upfront"])


# (residuals pass, CTAs per pair, threads, features per thread, MINB, general camera, upfront): the branches of launch_sia
ALIGN_INSTANTIATIONS = [(0, 2, 96, 1, 2, 1, 0), (0, 4, 96, 1, 1, 0, 1), (0, 4, 96, 1, 1, 1, 1), (0, 4, 96, 1, 2, 0, 0),
                        (0, 4, 96, 1, 2, 1, 0), (0, 8, 96, 1, 2, 1, 0), (0, 1, 320, 1, 3, 1, 0), (0, 1, 320, 1, 2, 0, 0),
                        (0, 1, 320, 1, 2, 1, 0), (0, 1, 384, 1, 2, 1, 0), (0, 1, 512, 1, 1, 1, 0), (0, 1, 160, 2, 4, 0, 0),
                        (0, 1, 160, 2, 4, 1, 0), (0, 1, 160, 2, 3, 0, 0), (0, 1, 160, 2, 3, 1, 0), (0, 1, 512, 2, 1, 1, 0)]
RESIDUAL_INSTANTIATIONS = [(1, 2, 96, 1, 2, 1, 0), (1, 4, 96, 1, 2, 1, 0), (1, 8, 96, 1, 2, 1, 0), (1, 1, 320, 1, 3, 1, 0),
                           (1, 1, 320, 1, 2, 1, 0), (1, 1, 384, 1, 2, 1, 0), (1, 1, 512, 1, 1, 1, 0), (1, 1, 160, 2, 4, 1, 0),
                           (1, 1, 160, 2, 3, 1, 0), (1, 1, 512, 2, 1, 1, 0)]
# in-process launches that reach the rest: (config, features, camera)
SWEEP = [((-1, 0, -1), 100, "pinhole"), ((-1, 0, -1), 100, "atan"), ((4, 0, 0), 100, "pinhole"), ((4, 0, 0), 100, "atan"),
         ((2, 0, -1), 100, "pinhole"), ((8, 0, -1), 100, "pinhole"), ((1, 1, -1), 300, "pinhole"), ((1, 1, -1), 300, "atan"),
         ((1, 1, -1), 350, "pinhole"), ((1, 1, -1), 450, "pinhole"), ((1, 2, -1), 300, "pinhole"), ((1, 2, -1), 300, "atan"),
         ((-1, 0, -1), 700, "pinhole")]


def test_every_instantiation_and_staging_mode_is_reached(ctx, children):
    records = [r for _, L in children.values() for r in L.values()]
    base = sc.base_pair()
    cam = synth.reference_param_camera("atan")
    atan = synth.make_frame_pair(1000, width=cam.width, height=cam.height, n_feat=300, n_levels=5, cam=cam)
    frames = {"pinhole": (ctx.frame(base["ref_pyr"]), ctx.frame(base["cur_pyr"])),
              "atan": (ctx.frame(atan["ref_pyr"]), ctx.frame(atan["cur_pyr"]))}
    try:
        for cfg, n, kind in SWEEP:
            ctx.sia_config(cfg[0], cfg[1])
            ctx.sia_upfront(cfg[2])
            d = sc.subset(base if kind == "pinhole" else atan, n)
            sc.gpu_run(ctx, d, frames=frames[kind])
            records.append(ctx.sia_last_launch())
            ctx.sparse_residuals(*frames[kind], d["cam"], 1, synth.se3_identity(), d["px"], d["f"], d["pos"], d["has_point"],
                                 d["ref_pos"])
            records.append(ctx.sia_last_launch())
    finally:
        ctx.sia_config(-1, 0)
        ctx.sia_upfront(-1)
        for fr in frames.values():
            for f in fr:
                f.destroy()
    reached = {}
    for r in records:
        reached.setdefault(_inst(r), set()).update(str(m) for m in r["stages"].values())
    print("\nresiduals CTAs threads FPT MINB general-camera upfront | staging modes reached")
    for inst in ALIGN_INSTANTIATIONS + RESIDUAL_INSTANTIATIONS:
        print(" ".join(f"{v:>4}" for v in inst), "|", ", ".join(sorted(reached.get(inst, {"NOT REACHED"}))))
    missing = [i for i in ALIGN_INSTANTIATIONS + RESIDUAL_INSTANTIATIONS if i not in reached]
    assert not missing, missing
    assert set(reached) <= set(ALIGN_INSTANTIATIONS + RESIDUAL_INSTANTIATIONS), set(reached) - set(ALIGN_INSTANTIATIONS + RESIDUAL_INSTANTIATIONS)
    modes = set().union(*reached.values())
    assert {"global", "image", "window"} <= modes, modes
