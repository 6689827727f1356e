"""Child process of test_sia_knobs_gpu.py: `python -m tests.sia_knob_child OUT.npz`.

The library reads its SVO_B200_SIA_* tuning knobs once per process, so every knob setting runs this fixed script in a
process of its own: the 300-feature pair, a 648x488 border case (windows copied as two 8-byte halves), a 640x480 border
case, each in four launch configurations with a residual pass, and one 64-pair batch.  Every output and every
svo_b200_sia_last_launch record goes into OUT.npz; the process exits when done."""
import json
import sys

import numpy as np

from rpg_svo_b200 import capi, synth
from tests import sia_cases as sc

CONFIGS = {"auto": (-1, 0, -1), "cta-1fpt": (1, 1, -1), "cta-2fpt": (1, 2, -1), "cluster-4-per-level": (4, 0, 0)}
RES_LEVEL = {"pair300": 0, "odd648": 0, "border": 2, "atan": 1}


def cases():
    pair300 = synth.make_frame_pair(1000, n_feat=300, n_levels=5)
    pair300["T_gt"] = pair300["T_cur_ref_gt"]
    cam = synth.reference_param_camera("atan")
    atan = synth.make_frame_pair(1000, width=cam.width, height=cam.height, n_feat=300, n_levels=5, cam=cam)
    atan["T_gt"] = atan["T_cur_ref_gt"]
    return {"pair300": pair300, "odd648": sc.odd_pair((648, 488)), "border": sc.border_pair(5, 640, 480, 300), "atan": atan}


# the distorted camera runs in the one-CTA configurations only: it reaches the general-camera instantiations that the
# pinhole cases leave to the SVO_B200_SIA_PLAIN=0 child (the throughput geometry with the patch cache among them)
CASE_CONFIGS = {"atan": ("cta-1fpt", "cta-2fpt")}


def batch_parts(d):
    """64 pairs on one frame pair: feature counts from 1 to 300, every one-CTA slot edge among them."""
    counts = [1, 17, 159, 160, 161, 299, 300] + [int(n) for n in np.linspace(20, 300, 57).astype(int)]
    return [sc.subset(d, n) for n in counts]


def main(out_path):
    ctx = capi.Context(0)
    arrays, launches = {}, {}
    for name, d in cases().items():
        ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
        for cname, cfg in CONFIGS.items():
            if cname not in CASE_CONFIGS.get(name, CONFIGS):
                continue
            ctx.sia_config(cfg[0], cfg[1])
            ctx.sia_upfront(cfg[2])
            key = f"{name}/{cname}"
            g = sc.gpu_run(ctx, d, frames=(ref, cur))
            launches[key] = ctx.sia_last_launch()
            tr = g["trace"]
            arrays.update({f"{key}/T": g["T"], f"{key}/H": g["H"], f"{key}/visible": g["visible"],
                           f"{key}/n_tracked": np.int64(g["n_tracked"]),
                           f"{key}/trace_i": np.array([[t["level"], t["iter"], t["accepted"], t["n_meas"]] for t in tr], np.int64),
                           f"{key}/trace_chi2": np.array([t["chi2"] for t in tr])})
            lv = RES_LEVEL[name]
            r = ctx.sparse_residuals(ref, cur, d["cam"], lv, d["T_gt"], d["px"], d["f"], d["pos"], d["has_point"], d["ref_pos"])
            launches[key + "/res"] = ctx.sia_last_launch()
            for k in ("visible", "in_image", "ref_patch", "residuals", "H", "Jres"):
                arrays[f"{key}/res/{k}"] = r[k]
            arrays[f"{key}/res/n_meas"] = np.int64(r["n_meas"])
            arrays[f"{key}/res/chi2"] = np.float64(r["chi2"])
        ref.destroy()
        cur.destroy()
    # one 64-pair batch with the automatic choice (one CTA per pair, the throughput geometry)
    ctx.sia_config(-1, 0)
    ctx.sia_upfront(-1)
    d = sc.base_pair()
    parts = batch_parts(d)
    ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
    B = len(parts)
    off = np.concatenate([[0], np.cumsum([len(p["px"]) for p in parts])]).astype(np.int32)
    ctx.sia_batch_stage([ref] * B, [cur] * B, d["cam"], np.tile(synth.se3_identity(), (B, 1, 1)), off,
                        np.concatenate([p["px"] for p in parts]), np.concatenate([p["f"] for p in parts]),
                        np.concatenate([p["pos"] for p in parts]), np.concatenate([p["has_point"] for p in parts]),
                        np.stack([p["ref_pos"] for p in parts]), 4, 0)
    ctx.sia_batch_run()
    r = ctx.sia_batch_fetch(want_H=True)
    launches["batch64"] = ctx.sia_last_launch()
    arrays.update({"batch64/T": r["T"], "batch64/H": r["H"], "batch64/visible": r["visible"],
                   "batch64/n_tracked": r["stats"]["n_tracked"].astype(np.int64), "batch64/offsets": off})
    ref.destroy()
    cur.destroy()
    ctx.close()
    np.savez(out_path, launches=np.array(json.dumps(launches)), **arrays)


if __name__ == "__main__":
    main(sys.argv[1])
