"""Cases at the corners of the plain alignment kernel's Gauss-Newton driver (gn_tail and the per-level loop of sia_kernel),
shared by test_sia_driver_pins.py (oracle vs the compiled reference, and the float64 statement below vs the oracle) and
test_sia_driver_edges_gpu.py (kernel vs oracle and vs the float64 statement).

Most cases run on one 640x480 frame pair (scene(): 300 features on the tilted plane), so that they can share a batch:
  iters_<n>          n_iter 0, 1, 2 and -1 (0: the loop never runs, no visibility, n_tracked 0; -1: the reference's size_t
                     n_iter_ wraps around, no limit)
  eps_zero / eps_huge / eps_nan   eps 0 and NaN (no accepted step stops a level), 1e30 (the first accepted step does)
  levels_<max>_<min> level ranges of the five-level pyramid; depth6_5_0 / depth7_6_0 the full range of six levels (640x480)
                     and of seven (1280x960)
  rollback_<k>       initial poses 2-10 cm / 1-3 degrees off: chi2 rises and the step is rolled back at most levels
  no_points          has_point all 0; coarse_empty: every feature 24-47 px from the border, level 4 has no patch
  zero_residual      cur == ref at the identity, features on a float-exact grid: every residual is 0, x = 0, chi2 = 0
  zero_eps_<0|neg>   the same with eps 0 (x = 0 stops every level: m <= eps at equality) and eps -5e-324 (never stops)
  textureless        constant images: H = 0, the pivoted factorisation's k == 0 exit, x = 0
  few_<n>            1, 2, 3, 6, 12 features: H rank deficient (one feature: rank 2, two: rank 4, the pivoted
                     LDL^T) or nearly so
  large_angle        12 features, a start 0.6 rad off: the first accepted step has |omega| >= 0.5 (se3_exp's closed form)
  theta_below / theta_above   12 features, starts 0.41 rad off about y / z: an accepted step with theta^2 just below / just
                     above 0.25, where se3_exp switches from the series to the closed form
  nan_px / inf_px / nan_f / inf_f / nan_pos / inf_pos   five features of the scene poisoned
  zero_depth         five features with pos == ref_pos (xyz_ref = 0: a NaN Jacobian), started 30 cm along the optical axis
                     so that they project into the image: H is NaN, the solve fails, stop latches and every level rolls back
  zero_depth_id      the same from the identity: they project to 0/0, never into the image, and contribute nothing
  fz_zero            five bearings with f_z == 0 exactly: 1/z = inf in their Jacobian rows, never in the image
  behind             ten features with the bearing negated: behind both cameras, projecting onto the same pixels
  far_proj           ten bearings with z = 1e-9: projections at ~1e11 px, past the kernel's 1e6 px guard
  nan_ref_pos / nan_T0   every depth / the start pose NaN: no measurement at any level

The float64 statement of the driver (pose_update_errors, expected_flags, check_stats, solve_errors) restates what each
iteration of a trace must satisfy, independently of the oracle's code."""
import functools
import math

import numpy as np

from oracle import binding as ob
from rpg_svo_b200 import synth
from tests import sia_cases as sc
from tests import sia_robust_edge_cases as ec

# sc.decision_margin generalised to any eps: no case compared iteration by iteration is nearer a flipped decision
MARGIN = 2e-5
# below this many features H is (nearly) singular: the reference's answer is rounding noise (sc.RANK_OK)
RANK_OK = sc.RANK_OK
# 12 features from a start 0.6 rad off: H is near singular, the kernel's and the oracle's chi2 differ by ~1e-4 relative, so
# the kernel is held to the float64 statement and to the oracle's mask, n_tracked and first pass only
NEAR_SINGULAR = ("large_angle", "theta_below", "theta_above")
THETA = {"theta_below": 4, "theta_above": 5}  # the axis of the 0.41 rad start
POISONED = np.arange(33, 300, 52)[:5]  # the poisoned features of the non-finite cases


@functools.lru_cache(maxsize=None)
def scene():
    d = synth.make_frame_pair(77, n_feat=300)
    d["has_point"][:] = 1
    return d


@functools.lru_cache(maxsize=None)
def _pyramid_scene(n_levels):
    w, h = (640, 480) if n_levels <= 6 else (1280, 960)  # 640x480 has no room for features at level 6
    d = synth.make_frame_pair(78, width=w, height=h, n_feat=300, n_levels=n_levels)
    d["has_point"][:] = 1
    return d


def _with(d, **kw):
    q = dict(d)
    for k in ("px", "f", "pos", "has_point"):
        q[k] = np.ascontiguousarray(d[k]).copy()
    q.update(kw)
    return q


def _far_pose(seed, trans, rot_deg):
    rng = np.random.default_rng(seed)
    xi = np.concatenate([rng.uniform(-trans, trans, 3), np.deg2rad(rng.uniform(-rot_deg, rot_deg, 3))])
    return synth.se3_mul(synth.se3_exp(xi), scene()["T_cur_ref_gt"])


def _zero_residual_pair():
    """cur == ref, features on a 1/64 px grid (exact in f32: the projection at the identity lands on the same f32 pixel)."""
    d = _with(scene())
    px = np.round(d["px"] * 64.0) / 64.0
    d["px"], d["f"] = px, np.ascontiguousarray(d["cam"].cam2world(px))
    d["pos"] = np.ascontiguousarray(synth.intersect(synth.Plane.tilted(), d["T_ref_w"], d["f"]))
    d["cur_pyr"] = d["ref_pyr"]
    return d


def _poisoned(kind):
    d = _with(scene())
    i = POISONED
    if kind in ("nan_px", "inf_px"):
        d["px"][i, i % 2] = np.nan if kind == "nan_px" else np.inf
    elif kind in ("nan_f", "inf_f"):
        d["f"][i, 2] = np.nan if kind == "nan_f" else -np.inf
    elif kind in ("nan_pos", "inf_pos"):
        d["pos"][i, 0] = np.nan if kind == "nan_pos" else np.inf
    elif kind in ("zero_depth", "zero_depth_id"):
        d["pos"][i] = d["ref_pos"]
    elif kind == "fz_zero":
        d["f"][i] = np.array([0.6, 0.8, 0.0])
    elif kind == "behind":
        j = np.arange(BEHIND, 300, 29)[:10]
        d["f"][j] = -d["f"][j]
    elif kind == "far_proj":
        j = np.arange(11, 300, 29)[:10]
        f = np.stack([np.ones(10), 0.5 * np.ones(10), np.full(10, 1e-9)], axis=1)
        d["f"][j] = f / np.linalg.norm(f, axis=1, keepdims=True)
    return d


def build(name):
    def case(p, n_iter=30, eps=1e-6, max_level=None, min_level=0, T0=None):
        return dict(name=name, p=p, n_iter=n_iter, eps=eps, max_level=p["n_levels"] - 1 if max_level is None else max_level,
                    min_level=min_level, T0=synth.se3_identity() if T0 is None else np.asarray(T0, np.float64))

    s = scene()
    parts = name.split("_")
    if parts[0] == "iters":
        return case(s, n_iter=-1 if parts[1] == "neg" else int(parts[1]))
    if name == "eps_zero":
        return case(s, eps=0.0, n_iter=6)
    if name == "eps_huge":
        return case(s, eps=1e30)
    if name == "eps_nan":
        return case(s, eps=float("nan"), n_iter=6)
    if parts[0] == "levels":
        return case(s, max_level=int(parts[1]), min_level=int(parts[2]))
    if parts[0].startswith("depth"):
        return case(_pyramid_scene(int(parts[0][5:])), max_level=int(parts[1]), min_level=int(parts[2]))
    if parts[0] == "rollback":
        return case(s, T0=_far_pose(*ROLLBACK[name]))
    if name == "no_points":
        return case(_with(s, has_point=np.zeros(300, np.uint8)))
    if name == "coarse_empty":
        return case(ec.strip_pair(73))
    if name == "zero_residual":
        return case(_zero_residual_pair())
    if name == "zero_eps_0":
        return case(_zero_residual_pair(), eps=0.0, n_iter=5)
    if name == "zero_eps_neg":
        return case(_zero_residual_pair(), eps=-5e-324, n_iter=5)
    if name == "textureless":
        flat = [np.full_like(im, 128) for im in s["ref_pyr"]]
        return case(_with(s, ref_pyr=flat, cur_pyr=flat))
    if parts[0] == "few":
        n = int(parts[1])
        return case(sc.subset(s, n, clear_edges=False))
    if name == "large_angle":
        d = sc.subset(s, 12, clear_edges=False)
        return case(d, T0=synth.se3_exp(np.array([0.02, -0.01, 0.0, 0.0, 0.0, LARGE_ANGLE])))
    if name in THETA:
        xi = np.zeros(6)
        xi[THETA[name]] = 0.41
        return case(sc.subset(s, 12, clear_edges=False), T0=synth.se3_exp(xi))
    if name == "nan_ref_pos":
        return case(_with(s, ref_pos=np.full(3, np.nan)))
    if name == "nan_T0":
        T0 = synth.se3_identity()
        T0[1, 3] = np.nan
        return case(s, T0=T0)
    if name == "zero_depth":
        return case(_poisoned(name), T0=synth.se3_exp(np.array([0.01, 0.005, 0.3, 0.0, 0.0, 0.0])))
    if name in NONFINITE:
        return case(_poisoned(name))
    raise KeyError(name)


BEHIND = 0  # the first of the features the behind case turns around
ROLLBACK = {"rollback_1": (1, 0.1, 3.0), "rollback_2": (6, 0.1, 3.0), "rollback_3": (3, 0.05, 1.0)}
LARGE_ANGLE = 0.6  # rad about the optical axis
NONFINITE = ("nan_px", "inf_px", "nan_f", "inf_f", "nan_pos", "inf_pos", "zero_depth", "zero_depth_id", "fz_zero", "behind",
             "far_proj")
LEVEL_RANGES = ("levels_4_4", "levels_3_3", "levels_2_2", "levels_1_1", "levels_0_0", "levels_4_2", "levels_3_0",
                "levels_3_1", "depth6_5_0", "depth7_6_0")
NAMES = (["iters_0", "iters_1", "iters_2", "iters_neg", "eps_zero", "eps_huge", "eps_nan"] + list(LEVEL_RANGES) +
         list(ROLLBACK) + ["no_points", "coarse_empty", "zero_residual", "zero_eps_0", "zero_eps_neg", "textureless",
                           "few_1", "few_2", "few_3", "few_6", "few_12", "large_angle", "theta_below", "theta_above", "nan_ref_pos", "nan_T0"] + list(NONFINITE))

# cases the compiled reference runs: its eps is fixed at 1e-6, and it takes the reference camera's position from the
# reference frame's pose, not as an input (nan_ref_pos moves it; the zero-depth cases need it bit for bit, and the
# reference's own -R^T t differs from ref_pos in the last bits, leaving those points at ~1e-16 m instead of 0).  It builds the pyramids from level 0 itself,
# which the cases with hand-made levels (flat images, one level 0 for both frames) still allow.
REF_CASES = [n for n in NAMES if not n.startswith(("eps_", "zero_eps_")) and n not in ("nan_ref_pos", "zero_depth", "zero_depth_id")]
# cases with the batch's options (30 iterations, eps 1e-6, levels 4..0 of a 640x480 pyramid)
BATCHABLE = ["rollback_1", "rollback_2", "rollback_3", "no_points", "coarse_empty", "zero_residual", "textureless", "few_1",
             "few_2", "few_3", "few_6", "few_12", "large_angle", "theta_below", "theta_above", "nan_ref_pos", "nan_T0"] + list(NONFINITE)


@functools.lru_cache(maxsize=None)
def case(name):
    return build(name)


def oracle_run(k, eps=None):
    p = k["p"]
    return ob.sparse_img_align(p["ref_pyr"], p["cur_pyr"], p["cam"], k["T0"], p["px"], p["f"], p["pos"], p["has_point"],
                               p["ref_pos"], k["max_level"], k["min_level"], k["n_iter"], k["eps"] if eps is None else eps)


def ref_run(ref, k):
    """The compiled reference's SparseImgAlign::run on case k (eps fixed at 1e-6 there), started at T_cur_w = T0 T_ref_w."""
    p = k["p"]
    return ref.call("sparse_img_align", p["ref_pyr"][0], p["cur_pyr"][0], p["n_levels"], p["cam"], p["T_ref_w"],
                    synth.se3_mul(k["T0"], p["T_ref_w"]), p["px"], p["f"], p["pos"], p["has_point"], k["max_level"],
                    k["min_level"], k["n_iter"])


def xmax(x):
    """|x|_inf as the driver forms it (NaN propagates as in fmax / Eigen's maxCoeff: NaN only if every entry is)."""
    return float(np.nanmax(np.abs(x))) if not np.all(np.isnan(x)) else float("nan")


def margin(o, eps):
    """sc.decision_margin with the case's eps (only where eps is finite and positive: otherwise no step can stop a level)."""
    m, prev = np.inf, None
    for t in o["trace"]:
        if t["iter"] > 0 and prev is not None and np.isfinite(prev) and prev > 0 and np.isfinite(t["chi2"]):
            m = min(m, abs(t["chi2"] - prev) / prev)
        if t["accepted"]:
            prev = t["chi2"]
            if eps > 0 and np.isfinite(eps) and xmax(t["x"]) > 0:
                m = min(m, abs(math.log(xmax(t["x"]) / eps)))
    return m


# ---- the float64 statement ------------------------------------------------------------------------------------------------
def se3_exp64(xi):
    """[upsilon, omega] -> 3x4 [R | V upsilon], R and V from the closed form (Taylor series below |omega| = 1e-4)."""
    ups, om = np.asarray(xi[:3], np.float64), np.asarray(xi[3:], np.float64)
    th2 = float(om @ om)
    th = math.sqrt(th2)
    O = synth.hat(om)
    if th < 1e-4:
        a = 1 - th2 / 6 + th2 * th2 / 120
        b = 0.5 - th2 / 24 + th2 * th2 / 720
        c = 1 / 6 - th2 / 120 + th2 * th2 / 5040
    else:
        a, b, c = math.sin(th) / th, (1 - math.cos(th)) / th2, (th - math.sin(th)) / (th2 * th)
    R = np.eye(3) + a * O + b * (O @ O)
    V = np.eye(3) + b * O + c * (O @ O)
    return np.hstack([R, (V @ ups)[:, None]])


def pose_update_errors(trace, T0):
    """Walk the trace as the driver does: an accepted iteration k must give T_k = T_(k-1) exp(-x_k) (returned: the largest
    |T_k - T_(k-1) exp(-x_k)| and the largest |R^T R - I| of any T_k); a rejected one must give back, bit for bit, the pose
    the last accepted step of its level started from (the level's first pose if none was accepted) -- asserted here."""
    cur = np.asarray(T0, np.float64)
    err = orth = 0.0
    level = None
    old = cur
    for i, t in enumerate(trace):
        if t["level"] != level:
            level, old = t["level"], cur
        if t["accepted"]:
            want = synth.se3_mul(cur, se3_exp64(-np.asarray(t["x"])))
            if np.all(np.isfinite(want)):
                err = max(err, float(np.abs(t["T"] - want).max()))
                R = t["T"][:, :3]
                orth = max(orth, float(np.abs(R.T @ R - np.eye(3)).max()))
            old, cur = cur, t["T"]
        else:
            assert np.array_equal(t["T"], old, equal_nan=True), (i, t["T"], old)
            cur = t["T"]
    return err, orth


def expected_flags(trace, levels, n_iter, eps):
    """The termination rule restated: per level (max..min) the iterations 0, 1, ... run until the first accepted step with
    |x|_inf <= eps, the first rejected one, or n_iter (none if negative); an iteration is rejected when stop has latched (a NaN x[0] at any
    earlier or this iteration, of any level) or when iter > 0 and its chi2 exceeds the last accepted one.  Returns the
    [(level, iter, accepted)] the trace's own chi2 and x imply; the trace must be exactly that."""
    out, stop, prev, pos = [], False, 1e10, 0
    for level in levels:
        for it in range(n_iter if n_iter >= 0 else 1 << 64):  # negative: the reference's size_t n_iter_, no limit
            if pos >= len(trace):
                return out + [("missing", level, it)]
            t = trace[pos]
            pos += 1
            stop = stop or bool(np.isnan(t["x"][0]))
            acc = not (stop or (it > 0 and t["chi2"] > prev))
            out.append((level, it, int(acc)))
            if not acc:
                break
            prev = t["chi2"]
            if xmax(t["x"]) <= eps:
                break
    return out + [("extra",) for _ in trace[pos:]]


def check_flags(trace, k):
    levels = list(range(k["max_level"], k["min_level"] - 1, -1)) if len(k["p"]["px"]) else []
    got = [(t["level"], t["iter"], t["accepted"]) for t in trace]
    assert got == expected_flags(trace, levels, k["n_iter"], k["eps"]), got


def check_stats(stats, trace, k):
    """n_iters = the trace length, sum_in_image = the patches in the image summed over the iterations, n_tracked = the last
    pass's patches (0 when no iteration ran: n_meas_ is reset by run() and only the loop counts)."""
    assert stats["n_iters"] == len(trace), (stats, len(trace))
    assert stats["sum_in_image"] == sum(t["n_meas"] for t in trace) // 16, stats
    want = trace[-1]["n_meas"] // 16 if trace and k["n_iter"] != 0 else 0
    assert stats["n_tracked"] == want, (stats, want)


def solve_errors(trace, k, residuals, kappa_max=1e12):
    """For every iteration: H and Jres of a residual pass at that level and at the pose the iteration linearised at (the
    pose after the previous iteration; the visibility the coarser levels left), x of H x = Jres in float64 vs the trace's x.
    Returns [(|dx|_inf / |x|_inf, cond(H))] for the iterations with cond(H) <= kappa_max and a finite x; `residuals(level, T,
    visible_in)` is the oracle's or the kernel's residual pass."""
    out, vis, T, level, lvl_vis = [], np.zeros(len(k["p"]["px"]), np.uint8), k["T0"], None, None
    for t in trace:
        if t["level"] != level:
            if lvl_vis is not None:
                vis = lvl_vis
            level = t["level"]
        r = residuals(level, T, vis)
        lvl_vis = r["visible"]
        T = t["T"]
        H, b = np.asarray(r["H"], np.float64), np.asarray(r["Jres"], np.float64)
        if not (np.all(np.isfinite(H)) and np.all(np.isfinite(t["x"]))) or not H.any():
            continue
        kappa = np.linalg.cond(H)
        if kappa > kappa_max:
            continue
        x = np.linalg.solve(H, b)
        out.append((float(np.abs(np.asarray(t["x"]) - x).max() / max(np.abs(x).max(), 1e-300)), float(kappa)))
    return out


def min_pivot_ratio(H):
    """The smallest d_j / max diag of H's unpivoted LDL^T (fact6_compute_upper takes the pivoted path below 1e-13)."""
    H = np.asarray(H, np.float64)
    md = np.abs(np.diag(H)).max()
    if not md > 0:
        return 0.0
    L, d = np.eye(6), np.zeros(6)
    for j in range(6):
        d[j] = H[j, j] - (L[j, :j] ** 2) @ d[:j]
        for i in range(j + 1, 6):
            L[i, j] = (H[i, j] - (L[i, :j] * L[j, :j]) @ d[:j]) / d[j] if d[j] != 0 else 0.0
    return float(d.min() / md)
