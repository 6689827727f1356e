"""Cases for the depth filter's seed update (depth_filter_kernel's computeTau + updateSeed), all on real epipolar matches.

a, b and z_range do not enter the match, so they can take any value on top of a real one; mu and sigma2 set the search
window.  The cases:
  - small_parallax: current frames whose parallax at the seeds runs from ~0.3 to ~3 pixel angles (px_error_angle =
    2 atan(1 / (2 fx)) ~ 3.2e-3 rad): gamma_plus on both sides of 0, the fmax(1e-7, z - tau) clamp, and bearings on both
    sides of depthFromTriangulation's det = 1e-6,
  - evolved: a, b from 0.5 to 1e4 (among them the values 1 to 50 inlier or outlier updates reach from the constructor's
    a = b = 10), sigma2 from 1e-10 up to windows so wide that z_inv_max clamps at 1e-8, other z_range,
  - degenerate: a or b zero, both zero, subnormal, negative or NaN; a + b overflowing to inf; a + b >= 2^24, where float
    a + b + 1.0f absorbs the 1 and the double ab + 1. does not; z_range 0, negative, subnormal, inf, NaN; sigma2
    subnormal, where mu / sigma2 overflows inside m,
  - no_match: a current frame of noise, where the scan scores nothing, for NO_MATCH's b + 1 at b = 2^24, inf and NaN.
"""
from __future__ import annotations

import math

import numpy as np

from rpg_svo_b200 import synth
from tests import depth_update_hp as hp

SMALL_BASELINES = (0.002, 0.004, 0.008, 0.016, 0.05)


def small_parallax(seed: int, baseline: float, n_seeds: int = 240) -> dict:
    c = synth.make_depth_case(seed, n_seeds=n_seeds, baseline=baseline)
    c["batch_id"][:] = 5
    return c


def parallax_px(c) -> np.ndarray:
    """Per seed, the angle at the true point between the two cameras' rays, in pixel angles."""
    T_ref_cur = synth.se3_mul(c["T_ref_w"], synth.se3_inv(c["T_cur_w"]))
    p = c["ftr_f"] * c["depth_gt"][:, None]
    q = p - T_ref_cur[:, 3]
    cosang = np.sum(p * q, axis=1) / (np.linalg.norm(p, axis=1) * np.linalg.norm(q, axis=1))
    return np.arccos(np.clip(cosang, -1, 1)) / hp.px_error_angle(c["cam"].fx)


def _walk(n: int, inlier: bool) -> tuple[float, float]:
    """a, b after n updates of a constructor seed (a = b = 10, mu = 0.5, sigma2 = 1/9, z_range = 2) by inliers (x at
    mu) or outliers (x 40 sigma away)."""
    a, b, mu, zr, s2 = 10.0, 10.0, 0.5, 2.0, hp.f32(1 / 9)
    for _ in range(n):
        x = mu if inlier else hp.f32(mu + 40 * math.sqrt(s2 + 1e-4))
        a, b, mu, s2 = hp.update_seed(x, hp.f32(1e-4), a, b, mu, zr, s2, hp.c_expf)
        if inlier:  # keep the window open: an inlier seed that converged would stop being updated
            s2 = max(s2, hp.f32(1e-3))
    return a, b


def evolved(seed: int = 41, n_seeds: int = 480) -> dict:
    c = synth.make_depth_case(seed, n_seeds=n_seeds, baseline=0.12)
    c["batch_id"][:] = 5
    rng = np.random.default_rng(seed)
    walks = [_walk(n, inl) for n in (1, 2, 5, 12, 25, 50) for inl in (True, False)]
    grid = [(a, b) for a in (0.5, 3.0, 57.0, 1e4) for b in (0.5, 10.0, 1e4)]
    ab = np.array((walks + grid) * (n_seeds // len(walks + grid) + 1), np.float32)[:n_seeds]
    s = c["seeds"]
    s["a"], s["b"] = ab[:, 0].copy(), ab[:, 1].copy()
    s["z_range"] = rng.choice(np.array([2.0, 0.5, 10.0, 1e-3, 100.0], np.float32), n_seeds)
    inv = 1.0 / c["depth_gt"]
    s["mu"] = (inv * (1 + rng.normal(0, 0.02, n_seeds))).astype(np.float32)
    s["sigma2"] = (10.0 ** rng.uniform(-10, -1, n_seeds)).astype(np.float32)
    wide = rng.uniform(size=n_seeds) < 0.1  # mu - sqrt(sigma2) < 0: z_inv_max = 1e-8
    s["sigma2"][wide] = (inv[wide] ** 2 * rng.uniform(1.5, 4, wide.sum())).astype(np.float32)
    c["wide"] = wide
    return c


DEGENERATE = {  # name: (field, values)
    "a_zero": ("a", [0.0]), "b_zero": ("b", [0.0]), "ab_zero": ("ab", [0.0]),
    "a_subnormal": ("a", [1e-45, 1e-40]), "b_subnormal": ("b", [1e-45, 1e-40]),
    "a_negative": ("a", [-3.0, -0.5]), "b_negative": ("b", [-3.0, -0.5]),
    "a_nan": ("a", [math.nan]), "b_nan": ("b", [math.nan]),
    "ab_overflow": ("ab", [3e38, 2e38]),
    "ab_2p24": ("a24", [2.0 ** 24, 2.0 ** 24 + 2, 1e7, 3e7]),
    "b_2p24": ("b", [2.0 ** 24, math.inf]),
    "zr_zero": ("z_range", [0.0]), "zr_negative": ("z_range", [-2.0]), "zr_subnormal": ("z_range", [1e-45, 1e-39]),
    "zr_inf": ("z_range", [math.inf]), "zr_nan": ("z_range", [math.nan]),
    "sigma2_subnormal": ("sigma2", [1e-40, 1e-45, 1e-38]),
}


def degenerate(seed: int = 43, per: int = 12) -> dict:
    """Seeds started near their true depth with a narrow window (so most match), each group with one degenerate field."""
    n = per * len(DEGENERATE)
    c = synth.make_depth_case(seed, n_seeds=n, baseline=0.12)
    c["batch_id"][:] = 5
    s = c["seeds"]
    s["mu"] = (1.0 / c["depth_gt"]).astype(np.float32)
    s["sigma2"][:] = np.float32(1e-4)
    group = np.repeat(np.array(list(DEGENERATE)), per)
    for g, (field, vals) in DEGENERATE.items():
        idx = np.flatnonzero(group == g)
        v = np.resize(np.array(vals, np.float32), len(idx))
        if field == "ab":
            s["a"][idx] = v
            s["b"][idx] = v
        elif field == "a24":
            s["a"][idx] = v
            s["b"][idx] = np.resize(np.array([1.0, 3.0, 7.0], np.float32), len(idx))
        else:
            s[field][idx] = v
    c["group"] = group
    return c


NO_MATCH_B = (2.0 ** 24, 2.0 ** 24 - 1, 2.0 ** 25, math.inf, math.nan, 3.4028235e38, 10.0)


def no_match(seed: int = 45, n_seeds: int = 140) -> dict:
    c = synth.make_depth_case(seed, n_seeds=n_seeds, baseline=0.3)
    c["batch_id"][:] = 5
    noise = np.random.default_rng(seed).integers(0, 256, c["cur_pyr"][0].shape, dtype=np.uint8)
    c["cur_pyr"] = synth.build_pyramid(noise, len(c["cur_pyr"]))
    c["seeds"]["b"] = np.resize(np.array(NO_MATCH_B, np.float32), n_seeds)
    return c


def edge_tuples() -> list[tuple]:
    """(x, tau2, a, b, mu, z_range, sigma2) for updateSeed alone: the degenerate values above on an ordinary update,
    plus non-finite x and tau2 and an update whose exponent underflows."""
    base = dict(x=0.5, tau2=1e-4, a=10.0, b=10.0, mu=0.52, z_range=2.0, sigma2=1e-3)
    out = [tuple(base.values())]
    for field, vals in DEGENERATE.values():
        for v in vals:
            d = dict(base)
            if field == "ab":
                d["a"] = d["b"] = v
            elif field == "a24":
                d["a"], d["b"] = v, 1.0
            else:
                d[field] = v
            out.append(tuple(d.values()))
    for k, v in (("x", math.inf), ("x", math.nan), ("x", 0.0), ("tau2", 0.0), ("tau2", math.inf), ("tau2", math.nan),
                 ("tau2", 1e-45), ("sigma2", 0.0), ("sigma2", -1e-3), ("sigma2", math.inf), ("mu", math.nan),
                 ("x", 30.0), ("mu", -0.5), ("sigma2", 1e-10), ("tau2", 1e-12)):
        d = dict(base)
        d[k] = v
        out.append(tuple(d.values()))
    return [tuple(float(np.float32(v)) for v in t) for t in out]
