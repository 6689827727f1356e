"""The grid of Matcher::Options settings and inputs on which the epipolar search and the depth filter are pinned
(tests/test_epipolar_options_pins.py against the compiled reference, tests/test_epipolar_options_gpu.py on the kernel).

Settings: every combination of align_1d, subpix_refinement and epi_search_edgelet_filtering at the default angle 0.7, and
with the filter on, the angles 0 (never rejects), 1.5 (rejects every edgelet that reaches the test) and NaN (never rejects:
`cosangle < NaN` is false).  Inputs, for the pinhole camera of the reference's tests, its radial-tangential pinhole and its
ATAN camera (the distorted models make unproject2d(uv_best) differ from cam2world(px_cur)): corners and edgelets at levels
0..2, each searched over a long segment (the scan), a short one (epi_length < 2: align at the midpoint) and a zero-length
one (d_min == d_max: px_A == px_B, so align_1d's direction is 0 / 0), against two keyframes."""
from __future__ import annotations

import itertools
import math
from functools import lru_cache

import numpy as np

from rpg_svo_b200 import synth

CAMERAS = {
    "pinhole": synth.camera_for(752, 480),
    "pinhole_radtan": synth.reference_param_camera("pinhole_radtan"),
    "atan": synth.reference_param_camera("atan"),
}
N_LEVELS = 3  # Config::nPyrLevels() = 3: max_search_level 2

FLAGS = [dict(align_1d=a, subpix_refinement=s, edgelet_filtering=f)
         for a, s, f in itertools.product((False, True), (True, False), (True, False))]
ANGLES = (0.0, 1.5, math.nan)


def settings():
    """(label, options dict) of the grid; the first is the defaults."""
    out = []
    for fl in FLAGS:
        out.append((f"a{int(fl['align_1d'])}s{int(fl['subpix_refinement'])}f{int(fl['edgelet_filtering'])}_0.7",
                    dict(fl, edgelet_max_angle=0.7)))
        if fl["edgelet_filtering"]:
            out += [(f"a{int(fl['align_1d'])}s{int(fl['subpix_refinement'])}f1_{ang}", dict(fl, edgelet_max_angle=ang))
                    for ang in ANGLES]
    return out


@lru_cache(maxsize=None)
def scene(name: str) -> dict:
    """Two keyframes and a current frame of the textured plane, and 16 features per keyframe (every third an edgelet)."""
    cam = CAMERAS[name]
    a = synth.make_two_view(1200, cam=cam, baseline=0.2, n_levels=N_LEVELS)
    b = synth.make_two_view(1201, cam=cam, baseline=0.1, n_levels=N_LEVELS)
    rng = np.random.default_rng(1202)
    kf_pyr, kf_T = [a["ref_pyr"], b["ref_pyr"]], [a["T_ref_w"], b["T_ref_w"]]
    feats = []
    for r, T_r in enumerate(kf_T):
        for j in range(16):
            L = j % 3
            px = np.floor(np.array([rng.uniform(60, cam.width - 60), rng.uniform(60, cam.height - 60)]) / (1 << L)) * (1 << L)
            f = cam.cam2world(px[None])[0]
            d = float(np.linalg.norm(synth.intersect(a["plane"], T_r, f[None])[0] - synth.se3_inv(T_r)[:, 3]))
            ang = rng.uniform(0, 2 * np.pi)
            feats.append(dict(ref=r, px=px, f=f, level=L, type=int(j % 3 == 1), grad=np.array([np.cos(ang), np.sin(ang)]),
                              depth=d))
    return dict(cam=cam, kf_pyr=kf_pyr, kf_T=kf_T, cur_pyr=a["cur_pyr"], T_cur_w=a["T_cur_w"], plane=a["plane"], feats=feats)


RANGES = {"scan": 0.3, "short": 0.002, "zero": 0.0}


def candidates(name: str) -> dict:
    """Every feature of scene(name) over every range of RANGES: arrays for the kernel's match-only launch."""
    s = scene(name)
    rows = [(ft, kind, rel) for ft in s["feats"] for kind, rel in RANGES.items()]
    d = np.array([ft["depth"] for ft, _, _ in rows])
    rel = np.array([rel for _, _, rel in rows])
    return dict(kind=[k for _, k, _ in rows], ref_index=np.array([ft["ref"] for ft, _, _ in rows], np.int32),
                ftr_px=np.array([ft["px"] for ft, _, _ in rows]), ftr_f=np.array([ft["f"] for ft, _, _ in rows]),
                ftr_level=np.array([ft["level"] for ft, _, _ in rows], np.int32),
                ftr_type=np.array([ft["type"] for ft, _, _ in rows], np.int32),
                ftr_grad=np.array([ft["grad"] for ft, _, _ in rows]), d_est=d,
                d_min=np.where(rel > 0, d / (1 + rel), d), d_max=np.where(rel > 0, d / np.maximum(1 - rel, 1e-3), d))


def seeds(name: str) -> dict:
    """Depth-filter seeds on both keyframes: the scene's features with seeds whose mean is near the true depth and whose
    range spans a long segment (every fourth seed a tight one: the short-line branch)."""
    s = scene(name)
    fs = s["feats"]
    n = len(fs)
    d = np.array([ft["depth"] for ft in fs])
    mu = (1.0 / (d * np.where(np.arange(n) % 2 == 0, 1.05, 0.97))).astype(np.float32)
    zr = np.float32(2.0)
    sigma2 = np.where(np.arange(n) % 4 == 3, np.float32(1e-7), zr * zr / np.float32(36)).astype(np.float32)
    sd = dict(a=np.full(n, 10, np.float32), b=np.full(n, 10, np.float32), mu=mu, z_range=np.full(n, zr, np.float32),
              sigma2=sigma2)
    return dict(ref_index=np.array([ft["ref"] for ft in fs], np.int32), ftr_px=np.array([ft["px"] for ft in fs]),
                ftr_f=np.array([ft["f"] for ft in fs]), ftr_level=np.array([ft["level"] for ft in fs], np.int32),
                ftr_type=np.array([ft["type"] for ft in fs], np.int32), ftr_grad=np.array([ft["grad"] for ft in fs]),
                batch_id=np.full(n, 5, np.int32), batch_counter=6, seeds=sd)


def oracle_match(epi, name: str, j: int, opt: dict) -> dict:
    """The oracle (oracle/binding_epipolar.py) on candidate j of candidates(name)."""
    s, c = scene(name), candidates(name)
    r = int(c["ref_index"][j])
    T_cur_ref = synth.se3_mul(s["T_cur_w"], synth.se3_inv(s["kf_T"][r]))
    return epi.find_epipolar_match_direct(s["kf_pyr"][r], s["cur_pyr"], s["cam"], T_cur_ref, c["ftr_px"][j], c["ftr_f"][j],
                                          int(c["ftr_level"][j]), int(c["ftr_type"][j]), c["ftr_grad"][j], c["d_est"][j],
                                          c["d_min"][j], c["d_max"][j], N_LEVELS - 1, opt=opt)


def ref_match(ref, name: str, j: int, opt: dict) -> dict:
    """The compiled reference on candidate j through the `ref` fixture (tests/ref_golden.py): its recorded outputs, or --
    when recording -- oracle/_ref/libsvo_ref_epipolar.so through oracle/binding_epipolar.py."""
    from oracle import binding_epipolar

    if ref.record_dir:
        ref.oracle = binding_epipolar
    s, c = scene(name), candidates(name)
    r = int(c["ref_index"][j])
    return ref.call("matcher_epipolar", s["kf_pyr"][r][0], s["cur_pyr"][0], N_LEVELS, s["cam"], s["kf_T"][r], s["T_cur_w"],
                    c["ftr_px"][j], c["ftr_f"][j], int(c["ftr_level"][j]), int(c["ftr_type"][j]), c["ftr_grad"][j],
                    float(c["d_est"][j]), float(c["d_min"][j]), float(c["d_max"][j]), opt=opt)


def ref_update(ref, name: str, opt: dict) -> dict:
    from oracle import binding_epipolar

    if ref.record_dir:
        ref.oracle = binding_epipolar
    s, k = scene(name), seeds(name)
    return ref.call("depth_filter_update_epipolar", [p[0] for p in s["kf_pyr"]], s["kf_T"], s["cur_pyr"][0], s["T_cur_w"],
                    N_LEVELS, s["cam"], k["ref_index"], k["ftr_px"], k["ftr_f"], k["ftr_level"], k["ftr_type"], k["ftr_grad"],
                    k["batch_id"], k["batch_counter"], k["seeds"], opt=opt)


def oracle_update(epi, name: str, opt: dict) -> dict:
    s, k = scene(name), seeds(name)
    return epi.depth_filter_update(s["kf_pyr"], s["kf_T"], s["cur_pyr"], s["T_cur_w"], s["cam"], k["ref_index"], k["ftr_px"],
                                   k["ftr_f"], k["ftr_level"], k["ftr_type"], k["ftr_grad"], k["batch_id"], k["batch_counter"],
                                   k["seeds"], max_search_level=N_LEVELS - 1, opt=opt)


def cosangle_threshold(epi, name: str, j: int, opt: dict) -> float:
    """The edgelet filter's cosangle of candidate j, as the largest angle the oracle does not reject it at: the filter
    rejects iff cosangle < angle, so the search over the doubles of [0, 1] ends on cosangle exactly."""
    lo, hi = np.float64(0.0).view(np.int64), np.float64(1.0).view(np.int64)  # kept at 0; rejected at 1 (checked by caller)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if oracle_match(epi, name, j, dict(opt, edgelet_max_angle=float(np.int64(mid).view(np.float64))))["reject"]:
            hi = mid
        else:
            lo = mid
    return float(np.int64(lo).view(np.float64))


def threshold_candidates(name: str) -> list[int]:
    """Two edgelets per camera whose filter test is reached (the scan and the short range of the first two edgelets)."""
    c = candidates(name)
    return [j for j in range(len(c["kind"])) if c["ftr_type"][j] == 1 and c["kind"][j] in ("scan", "short")][:2]
