"""The pose optimizer's case catalogue for the high-precision statement of tests/pose_hp.py: observation counts around
the kernel's 512-thread strides and its shared-memory capacity, iteration counts across the scale switch at iteration 5,
every way the loop ends, the EPS stop and the culling test at their edges, the covariance after a roll-back, non-finite
and extreme-depth observations.  Shared by the CPU pins (tests/test_pose_hp_pins.py) and the GPU tests
(tests/test_pose_hp_gpu.py).

A case is a dict: name, the eight arguments of pose_optimize (`args`), `exact` (every residual is computed without
rounding: identity pose, points at z = 1, bearings with f_z = 1) and `edge`, what the statement must show it reaches."""
from __future__ import annotations

import dataclasses
from fractions import Fraction

import numpy as np

from rpg_svo_b200 import synth

CAPACITY_N = 3400   # near the largest frame one CTA's shared memory holds (3464 observations with 227 KB per block)


def case(name, c, n_iter=10, reproj_thresh=2.0, fx=None, exact=False, edge=None):
    fx = float(c["cam"].fx if fx is None else fx)
    return dict(name=name, cam=dataclasses.replace(c["cam"], fx=fx), args=(float(reproj_thresh), int(n_iter), fx, np.asarray(c["T_init"], np.float64),
                                 np.asarray(c["f"], np.float64), np.asarray(c["pos"], np.float64),
                                 np.asarray(c["level"], np.int32), np.asarray(c["has_point"], np.uint8)),
                exact=exact, edge=edge or {})


def robust_frame(seed, rot_deg=2.0, n=120, noise=0.5, ofrac=0.2, olo=3.0, ohi=8.0, trans=0.02):
    """A frame whose robust weights keep moving: `rot_deg` of initial rotation error, and a fraction `ofrac` of
    observations pushed off by olo..ohi times the MAD scale at the initial pose -- around the Tukey cutoff (4.6851 scales),
    and again around it once iteration 5 switches to 0.85 px."""
    rng = np.random.default_rng(seed)
    cam = synth.camera_for(752, 480)
    T_true = synth.base_pose()
    px = np.stack([rng.uniform(20, 732, n), rng.uniform(20, 460, n)], 1)
    pos = synth.intersect(synth.Plane.tilted(), T_true, cam.cam2world(px))
    noisy = px + rng.normal(0, noise, (n, 2))
    w = rng.normal(size=3)
    w *= np.deg2rad(rot_deg) / np.linalg.norm(w)
    T_init = synth.se3_mul(synth.se3_exp(np.concatenate([rng.uniform(-trans, trans, 3), w])), T_true)
    # the MAD scale at T_init in pixels, as the optimizer computes it (float median of the unit-plane errors, times fx)
    p = pos @ T_init[:, :3].T + T_init[:, 3]
    fb = cam.cam2world(noisy)
    e = np.linalg.norm(fb[:, :2] / fb[:, 2:] - p[:, :2] / p[:, 2:], axis=1).astype(np.float32)
    s_px = float(np.float32(1.48) * np.partition(e, n // 2)[n // 2]) * cam.fx
    k = int(ofrac * n)
    idx = rng.choice(n, k, replace=False)
    ang = rng.uniform(0, 2 * np.pi, k)
    noisy[idx] += np.stack([np.cos(ang), np.sin(ang)], 1) * (rng.uniform(olo, ohi, k) * s_px)[:, None]
    return dict(cam=cam, f=cam.cam2world(noisy), pos=pos, level=np.zeros(n, np.int32), has_point=np.ones(n, np.uint8),
                T_init=T_init)


def count_cases():
    out = []
    for n in (1, 2, 3, 40, 41, 511, 512, 513, 1024, 1025):
        c = synth.make_pose_opt_case(700 + n, n, 752, 480, px_noise=0.05, outlier_frac=0.1)
        c["has_point"][:] = 1
        out.append(case(f"n{n}", c, n_iter=10 if n <= 513 else 4))
    c = synth.make_pose_opt_case(123, CAPACITY_N, 1920, 1080)
    out.append(case(f"n{CAPACITY_N}_capacity", c, n_iter=2))
    return out


def iteration_cases():
    """One frame that has not converged by iteration 5, at n_iter = 0, 1, 4, 5, 6, 7, 10 and 30: the switch to 0.85 px
    at iteration 5 changes its weights."""
    c = robust_frame(0, 2.0, noise=0.5, ofrac=0.2)
    return [case(f"iters{k}", c, n_iter=k, edge=dict(unconverged_at=5 if k >= 6 else None)) for k in (0, 1, 4, 5, 6, 7, 10, 30)]


def rollback_at_switch_case():
    """Small errors (a MAD scale of ~0.15 px): the switch to 0.85 px raises every weight and with them chi2, so
    iteration 5 rolls back -- to the pose iteration 4 started from -- and the covariance is the inverse of that rejected
    iteration's A."""
    c = robust_frame(0, 0.01, noise=0.05, ofrac=0.2, trans=0.0003)
    return case("rollback_at_switch", c, n_iter=30, edge=dict(end="rollback", at=5))


def eps_cases():
    """Noise-free observations of a pose perturbed by a twist whose largest component is 1e-10 (1 -+ 3e-2): the first
    step's max|dT| lies 3 % below (stop after one iteration) or above (one more) EPS = 1e-10.  3 % is the smallest margin
    of the form 10^-k / 3 that the statement's bound on the step decides (at 1 % the step's bound, ~1e-12, is the margin)."""
    out = []
    for side, k in (("below", 1 - 3e-2), ("above", 1 + 3e-2)):
        c = synth.make_pose_opt_case(31, 60, 752, 480, px_noise=0.0, outlier_frac=0.0)
        c["has_point"][:] = 1
        T_true = c["T_true"]
        p = c["pos"] @ T_true[:, :3].T + T_true[:, 3]
        c["f"] = p / np.linalg.norm(p, axis=1, keepdims=True)
        xi = np.array([1.0, -0.4, 0.3, 0.2, -0.5, 0.1]) * 1e-10 * k
        c["T_init"] = synth.se3_mul(synth.se3_exp(xi), T_true)
        out.append(case(f"eps_{side}", c, n_iter=10, edge=dict(eps_side=side)))
    return out


def _unit_plane_frame(ex, level, fx):
    """Identity pose, points (0, 0, 1), bearings (ex * 2^level, 0, 1): every residual is exactly (ex, 0), computed
    without a rounding (x / 1, a difference with 0, a power-of-two scale), and sqrt(fl(ex^2)) = |ex|."""
    n = len(ex)
    cam = synth.camera_for(752, 480)
    f = np.zeros((n, 3))
    f[:, 0] = np.asarray(ex) * np.exp2(np.asarray(level, np.float64))
    f[:, 2] = 1.0
    pos = np.tile([0.0, 0.0, 1.0], (n, 1))
    return dict(cam=cam, f=f, pos=pos, level=np.asarray(level, np.int32), has_point=np.ones(n, np.uint8),
                T_init=synth.se3_identity())


def cull_cases():
    """The culling test sqrt(e^2) > fl(reproj_thresh / fx) at its edge: errors of exactly the threshold and its two
    neighbouring doubles, at levels 0-4 and 30, for quotients that are not exact.  Strict `>`: the threshold itself stays."""
    out = []
    for rt, fx in ((2.0, 315.5), (2.0, 470.3), (1.5, 1234.567)):
        th = np.float64(rt) / np.float64(fx)
        assert Fraction(float(th)) * Fraction(fx) != Fraction(rt)   # the quotient is rounded
        ex, lv = [], []
        for level in (0, 1, 2, 3, 4, 30):
            for v in (np.nextafter(th, 0.0), th, np.nextafter(th, 1.0)):
                ex.append(v)
                lv.append(level)
        out.append(case(f"cull_{rt}_{fx}", _unit_plane_frame(ex, lv, fx), n_iter=0, reproj_thresh=rt, fx=fx, exact=True,
                        edge=dict(cull_exact=True)))
    # more than half culled: error_final is the median of the pre-culling errors, a culled one
    th = np.float64(2.0) / np.float64(315.5)
    ex = [th * 10] * 6 + [th * 0.25] * 3
    out.append(case("cull_majority", _unit_plane_frame(ex, [0] * 9, 315.5), n_iter=0, fx=315.5, exact=True,
                    edge=dict(cull_majority=True)))
    return out


def extreme_cases():
    """Non-finite and extreme observations, each in an otherwise ordinary 40-observation frame (observation 0 altered)."""
    out = []

    def base(seed):
        c = synth.make_pose_opt_case(seed, 40, 752, 480, px_noise=0.05, outlier_frac=0.0)
        c["has_point"][:] = 1
        return c

    for name, key, val in (("pos_nan", "pos", [np.nan, 0.1, 3.0]), ("f_z0", "f", [0.1, 0.05, 0.0])):
        c = base(51)
        c[key][0] = val
        out.append(case(name, c, edge=dict(end="nan")))
    # identity pose so that z is what is written: on the plane, tiny, huge, behind
    for name, z in (("z0", 0.0), ("z_2^-130", 2.0 ** -130), ("z_2^-128", 2.0 ** -128), ("z_2^128", 2.0 ** 128),
                    ("z_2^130", 2.0 ** 130), ("behind", -3.0)):
        c = base(52)
        c["pos"] = c["pos"] @ c["T_true"][:, :3].T + c["T_true"][:, 3]   # camera-frame points: T_init = identity is exact
        c["T_init"] = synth.se3_identity()
        # beyond the camera (|z| >= 1) the point lies on the bearing (0.05, 0.02, 1); near the plane it sits at x = 0.05,
        # y = 0.02, so that project2d(xyz) = (0.05, 0.02) / z: within 2^-128 of the plane its error overflows the float to
        # inf, its Tukey weight is 0 and it adds exact zeros to A and b (J J^T ~ 2^260 stays finite), and it is culled
        s = abs(z) if abs(z) > 1.0 else 1.0
        c["pos"][0] = [0.05 * s, 0.02 * s, z]
        c["f"][0] = [0.05, 0.02, 1.0]
        out.append(case(name, c, n_iter=10))
    # a float-subnormal MAD scale: 4 observations with an exactly zero error, 5 on the optical axis with 1e-40-sized ones
    n0, n1 = 4, 5
    rng = np.random.default_rng(3)
    uv = rng.uniform(-0.3, 0.3, (n0, 2))
    d = 2.0 ** rng.integers(0, 3, n0)
    f = np.concatenate([np.column_stack([uv, np.ones(n0)]), np.column_stack([np.arange(1, n1 + 1) * 1e-40, np.zeros(n1), np.ones(n1)])])
    pos = np.concatenate([np.column_stack([uv, np.ones(n0)]) * d[:, None], np.tile([0.0, 0.0, 1.0], (n1, 1)) * [[1], [2], [4], [1], [2]]])
    c = dict(cam=synth.camera_for(752, 480), f=f, pos=pos, level=np.zeros(n0 + n1, np.int32), has_point=np.ones(n0 + n1, np.uint8),
             T_init=synth.se3_identity())
    out.append(case("subnormal_scale", c, n_iter=3, exact=True, edge=dict(subnormal_scale=True)))
    return out


def empty_case():
    c = synth.make_pose_opt_case(9, 16, 640, 480)
    c["has_point"][:] = 0
    return case("empty", c, edge=dict(end="empty"))


def all_cases():
    return (count_cases() + iteration_cases() + [rollback_at_switch_case()] + eps_cases() + cull_cases() + extreme_cases()
            + [empty_case()])


def ref_args(c):
    """The arguments of the compiled reference's pose_optimize: the camera in place of fx (its errorMultiplier2() is fx)."""
    a = c["args"]
    return a[:2] + (c["cam"],) + a[3:]


# cases whose A is rank-deficient (1 and 2 observations): the step along the null space is rounding noise in every
# implementation, and so are the pose and the iteration at which chi2 stops falling; only what iteration 0 and the
# culling decide is compared there (the flags, num_obs, estimated_scale, error_init)
RANK_DEFICIENT = {"n1", "n2"}
# noise-free frames: every error is ~1e-11 with ~1e-15 of rounding in any implementation, so the reference's and the
# kernel's MAD scale, medians, weights and covariance agree to ~1e-4 relative, not 1e-9 (the statement's candidate
# intervals and covariance bound hold both)
NOISE_FREE = {"eps_below", "eps_above"}
# frames with a NaN error: the reference orders the NaN with std::nth_element, the kernel and the statement above +inf
NAN_MEDIAN = {"pos_nan"}
