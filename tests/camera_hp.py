"""An exactly rounded statement of vikit's two camera functions as the library spells them (rpg_svo_b200/csrc/svo_math.cuh
`cam_world2cam` / `cam_cam2world`, with the constants `cam_to_dev` derives; the oracle's `Cam` restates the same
operations), for the tests of the oracle and of the device code every projecting kernel inlines.

Every double operation is computed exactly (Fraction) and rounded once to nearest-even, fma counted as one rounding, in
the order svo_math.cuh writes it; (float) casts round once to binary32.  atan and tan are parameters: they are the only
operations of the two functions that are not correctly rounded.  With glibc's atan / tan (`c_atan` / `c_tan`, which the
oracle calls) the statement gives the oracle's one result; for the device, `world2cam_candidates` / `cam2world_candidates`
run it with every value within ATAN_ULP / TAN_ULP of the correctly rounded one (the CUDA C++ Programming Guide's bound for
double atan and tan), at most five results per call.  The constants tans = 2 tan(s / 2), 1 / tans, 1 / s, 1 / fx and
1 / fy are computed on the host with glibc's tan in both the library and the oracle, so they are fixed here too.

Branch decisions (r < 0.001, dist_r > 0.01) are taken on the statement's own rounded r and dist_r, so exact ties are
defined.  `Exact` evaluates the same formulas unrounded at 40 digits, the check on the statement itself.
"""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass
from fractions import Fraction

import numpy as np
from mpmath import mp, mpf

from tests import depth_update_hp as dhp

mp.dps = 40
ATAN_ULP = 2   # CUDA C++ Programming Guide, double-precision functions: atan(x) 2 ulp (full range)
TAN_ULP = 2    # tan(x) 2 ulp (full range)
PINHOLE, ATAN = 0, 1


dhp._libm.tan.restype, dhp._libm.tan.argtypes = ctypes.c_double, [ctypes.c_double]


def c_atan(x: float) -> float:
    """glibc's atan, as the oracle calls it (math.atan is the same function behind Python's domain checks)."""
    return dhp.c_atan(x)


def c_tan(x: float) -> float:
    """glibc's tan (NaN for +-inf, where math.tan raises)."""
    return float(dhp._libm.tan(x))


@dataclass(frozen=True)
class CamConst:
    """The CamDev of ctx.h: the camera's parameters and the constants `cam_to_dev` derives (with glibc's tan)."""
    fx: float
    fy: float
    cx: float
    cy: float
    model: int
    d: tuple
    distorted: bool
    fx_inv: float
    fy_inv: float
    s_inv: float
    tans: float
    tans_inv: float


def cam_const(cam) -> CamConst:
    d = tuple(float(v) for v in (list(cam.d) + [0.0] * 5)[:5])
    s_inv = tans = tans_inv = 0.0
    if cam.model == PINHOLE:
        distorted = abs(d[0]) > 0.0000001
    else:
        distorted = d[0] != 0.0
        if distorted:
            tans = 2.0 * math.tan(d[0] / 2.0)
            tans_inv, s_inv = 1.0 / tans, 1.0 / d[0]
    return CamConst(float(cam.fx), float(cam.fy), float(cam.cx), float(cam.cy), int(cam.model), d, distorted,
                    1.0 / cam.fx, 1.0 / cam.fy, s_inv, tans, tans_inv)


# ---- arithmetic ---------------------------------------------------------------------------------------------------------
class IEEE:
    """binary64, every operation rounded once to nearest-even (non-finite operands as IEEE)."""
    add = staticmethod(lambda x, y: dhp.add(x, y, "d"))
    sub = staticmethod(lambda x, y: dhp.sub(x, y, "d"))
    mul = staticmethod(lambda x, y: dhp.mul(x, y, "d"))
    div = staticmethod(lambda x, y: dhp.div(x, y, "d"))
    sqrt = staticmethod(lambda x: dhp.sqrt(x, "d"))
    f32 = staticmethod(dhp.f32)
    const = staticmethod(float)

    @staticmethod
    def fma(a, b, c):
        if dhp._fin(a, b, c):
            return dhp.rnd(Fraction(a) * Fraction(b) + Fraction(c), "d")
        if math.isnan(a) or math.isnan(b) or math.isnan(c):
            return math.nan
        if math.isinf(a) or math.isinf(b):  # an infinite product (NaN for inf * 0), then the sum as IEEE
            p = math.nan if a == 0 or b == 0 else math.copysign(math.inf, a) * math.copysign(1.0, b)
            return p + c
        return c  # finite product, infinite addend


class Exact:
    """The same formulas unrounded at 40 digits ((float) casts still round: they are vikit's, not the arithmetic's)."""
    add = staticmethod(lambda x, y: x + y)
    sub = staticmethod(lambda x, y: x - y)
    mul = staticmethod(lambda x, y: x * y)
    div = staticmethod(lambda x, y: x / y)
    sqrt = staticmethod(mp.sqrt)
    fma = staticmethod(lambda a, b, c: a * b + c)
    const = staticmethod(mpf)

    @staticmethod
    def f32(x):
        return mpf(math.copysign(dhp._rn32(abs(x)), x))


# ---- the two functions --------------------------------------------------------------------------------------------------
def world2cam_uv(c: CamConst, x, y, atan=c_atan, A=IEEE):
    """cam_world2cam(c, x, y): (u, v, branch).  branch: "plain" (fx x + cx), "radtan", "atan_small" (r < 0.001: factor
    1), "atan"."""
    K = A.const
    if not c.distorted:
        return A.fma(K(c.fx), x, K(c.cx)), A.fma(K(c.fy), y, K(c.cy)), "plain"
    if c.model == PINHOLE:
        d = [K(v) for v in c.d]
        r2 = A.fma(x, x, A.mul(y, y))
        r4 = A.mul(r2, r2)
        r6 = A.mul(r4, r2)
        a1 = A.mul(A.mul(K(2.0), x), y)
        a2 = A.fma(A.mul(K(2.0), x), x, r2)
        a3 = A.fma(A.mul(K(2.0), y), y, r2)
        cdist = A.fma(d[4], r6, A.fma(d[1], r4, A.fma(d[0], r2, K(1.0))))
        xd = A.fma(d[3], a2, A.fma(d[2], a1, A.mul(x, cdist)))
        yd = A.fma(d[3], a1, A.fma(d[2], a3, A.mul(y, cdist)))
        return A.fma(xd, K(c.fx), K(c.cx)), A.fma(yd, K(c.fy), K(c.cy)), "radtan"
    r = A.sqrt(A.fma(x, x, A.mul(y, y)))
    if r < 0.001:
        factor, br = K(1.0), "atan_small"
    else:
        factor, br = A.div(A.mul(K(c.s_inv), atan(A.mul(r, K(c.tans)))), r), "atan"
    return A.fma(A.mul(K(c.fx), factor), x, K(c.cx)), A.fma(A.mul(K(c.fy), factor), y, K(c.cy)), br


def project(x, y, z, A=IEEE):
    """project2d: xyz.head<2>() / z."""
    return A.div(x, z), A.div(y, z)


def world2cam(c: CamConst, xyz, atan=c_atan, A=IEEE):
    x, y = project(*[A.const(float(v)) for v in xyz], A=A)
    return world2cam_uv(c, x, y, atan, A)


def cam2world(c: CamConst, u, v, tan=c_tan, A=IEEE):
    """cam_cam2world(c, u, v): (f0, f1, f2, branch).  branch: "pinhole", "radtan", "atan_inner" (dist_r <= 0.01:
    d_factor 1) or "atan" (with "_s0" for an ATAN camera with s = 0)."""
    K = A.const
    u, v = K(float(u)), K(float(v))
    if c.model == PINHOLE:
        if not c.distorted:
            x, y, br = A.div(A.sub(u, K(c.cx)), K(c.fx)), A.div(A.sub(v, K(c.cy)), K(c.fy)), "pinhole"
        else:
            d = [K(t) for t in c.d]
            x0 = A.mul(A.sub(A.f32(u), K(c.cx)), K(c.fx_inv))
            y0 = A.mul(A.sub(A.f32(v), K(c.cy)), K(c.fy_inv))
            x, y = x0, y0
            for _ in range(5):
                r2 = A.add(A.mul(x, x), A.mul(y, y))
                icdist = A.div(K(1.0), A.add(K(1.0), A.mul(A.add(A.mul(A.add(A.mul(d[4], r2), d[1]), r2), d[0]), r2)))
                dX = A.add(A.mul(A.mul(A.mul(K(2.0), d[2]), x), y), A.mul(d[3], A.add(r2, A.mul(A.mul(K(2.0), x), x))))
                dY = A.add(A.mul(d[2], A.add(r2, A.mul(A.mul(K(2.0), y), y))), A.mul(A.mul(A.mul(K(2.0), d[3]), x), y))
                x, y = A.mul(A.sub(x0, dX), icdist), A.mul(A.sub(y0, dY), icdist)
            x, y, br = A.f32(x), A.f32(y), "radtan"
    else:
        dx = A.mul(A.sub(u, K(c.cx)), K(c.fx_inv))
        dy = A.mul(A.sub(v, K(c.cy)), K(c.fy_inv))
        dist_r = A.sqrt(A.add(A.mul(dx, dx), A.mul(dy, dy)))
        r = A.mul(tan(A.mul(dist_r, K(c.d[0]))), K(c.tans_inv)) if c.distorted else dist_r
        if dist_r > 0.01:
            d_factor, br = A.div(r, dist_r), "atan"
        else:
            d_factor, br = K(1.0), "atan_inner"
        br += "" if c.distorted else "_s0"
        x, y = A.mul(d_factor, dx), A.mul(d_factor, dy)
    n = A.sqrt(A.add(A.add(A.mul(x, x), A.mul(y, y)), K(1.0)))
    return A.div(x, n), A.div(y, n), A.div(K(1.0), n), br


# ---- the device's candidates --------------------------------------------------------------------------------------------
def _rn_mp(v) -> float:
    """An mpf rounded once to the nearest double."""
    if not mp.isfinite(v):
        return float(v)
    if v < 0:
        return -_rn_mp(-v)
    man, e = v.man_exp
    return dhp.rnd(Fraction(int(man)) * Fraction(2) ** int(e), "d") if man else 0.0


def _step(v: float, k: int) -> float:
    x = np.float64(v)
    for _ in range(abs(k)):
        x = np.nextafter(x, np.inf if k > 0 else -np.inf)
    return float(x)


def rn_atan(a: float) -> float:
    """atan(a) rounded to the nearest double (40 digits; glibc's for +-inf and NaN, where it is exact)."""
    return _rn_mp(mp.atan(mpf(a))) if math.isfinite(a) else math.atan(a)


def rn_tan(a: float) -> float:
    return _rn_mp(mp.tan(mpf(a))) if math.isfinite(a) else math.nan


def _near(rn, n_ulp):
    """The functions returning rn(a) + k ulp, |k| <= n_ulp (k = 0 first)."""
    def fn(a, k):
        r = rn(a)
        return _step(r, k) if math.isfinite(r) else r
    return [lambda a, k=k: fn(a, k) for k in _KS[:2 * n_ulp + 1]]


_KS = sorted(range(-8, 9), key=abs)  # ulp offsets, smallest first


def _candidates(results):
    """[(k, result)] of distinct results, each with the smallest |k| that gives it."""
    out = []
    for k, r in results:
        if not any(same_tuple(r, o) for _, o in out):
            out.append((k, r))
    return out


def world2cam_candidates(c: CamConst, xyz):
    """Every (k, (u, v)) the device may compute, k the ulp offset of its atan from the correctly rounded one: one for a
    pinhole camera, up to 2 ATAN_ULP + 1 for ATAN."""
    fns = _near(rn_atan, ATAN_ULP) if c.model == ATAN and c.distorted else [rn_atan]
    return _candidates((k, world2cam(c, xyz, fn)[:2]) for k, fn in zip(_KS, fns))


def cam2world_candidates(c: CamConst, px):
    """Every (k, (f0, f1, f2)) the device may compute, k the ulp offset of its tan."""
    fns = _near(rn_tan, TAN_ULP) if c.model == ATAN and c.distorted else [rn_tan]
    return _candidates((k, cam2world(c, px[0], px[1], fn)[:3]) for k, fn in zip(_KS, fns))


def same_tuple(a, b) -> bool:
    """Bit for bit, zeros by value and NaNs by class."""
    return all(dhp.same(float(x), float(y)) for x, y in zip(a, b))
