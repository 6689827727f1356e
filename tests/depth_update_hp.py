"""An exactly rounded statement of DepthFilter::updateSeed (svo/src/depth_filter.cpp:309-332) and an enclosure of the
tau2 that DepthFilter::computeTau (:334-350) hands it, for the tests of depth_filter_kernel and of the CPU oracle.

`update_seed` restates the update operation by operation, in the order and the formats the kernel and the oracle spell
it: every float or double result is computed exactly (Fraction) and rounded once to nearest-even in its format, fmaf
included (never through a double); subnormals, +-inf and NaN follow IEEE.  The value of exp(exponent) is a parameter:
it is the one operation of the update that is not correctly rounded (CUDA's expf is documented at <= 2 ulp, glibc's
expf is its own function), so everything else the update computes is determined bit for bit by its inputs.

The inputs of the update are x = (float)(1./z) and tau2 = (float)(tau_inverse^2).  x comes exactly from the depth z the
kernel reports.  tau2 goes through a pose product, acos, sin and atan, none of them correctly rounded; `tau2_enclosure`
evaluates computeTau at 40 digits over intervals that hold every value the device may have computed:
  - T_ref_cur's translation within POSE_ULP u of the exact product of the caller's [R|t] (the kernel's [R|t] ->
    quaternion -> product path; tests/world_frame_cases.py bounds the round trip at 8 u per entry),
  - every double operation within half an ulp, acos, sin and atan within the maximum ulp error the CUDA C++ Programming
    Guide lists for them (double precision: acos 2, sin 2, atan 2; single precision expf 2),
  - fmax(1e-7, z - tau) and the sign of sin(gamma_plus) evaluated over the interval: a clamp or a sign change inside the
    enclosure yields both outcomes (the enclosure is a union of intervals).
The admissible tau2 are the floats of the enclosure.  `candidates` returns every (a, b, mu, sigma2, status) the update
may produce from those tau2 and exp(exponent) in {RN(e^t) + k ulp, |k| <= 2}.

`triangulation` restates depthFromTriangulation (svo/src/matcher.cpp:109-122) at 40 digits from the pixel the kernel
reports, with a bound on the device depth and the margin of its `det < 1e-6` decision.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import math
from fractions import Fraction

import numpy as np
from mpmath import mp, mpf

mp.dps = 40

U = 2.0 ** -53
POSE_ULP = 8           # tests/world_frame_cases.py: ROUNDTRIP_ULP
ACOS_ULP = 2           # CUDA C++ Programming Guide, double-precision functions: acos(x) 2 ulp (full range)
SIN_ULP = 2            # sin(x) 2 ulp (full range)
ATAN_ULP = 2           # atan(x) 2 ulp (full range)
EXPF_ULP = 2           # single-precision functions: expf(x) 2 ulp (full range)
MAX_TAU2 = 16          # more admissible tau2 than this: only the update's decisive decisions are checked
PI_TRUNC = 3.14159265  # svo/include/svo/global.h:78
UPDATED, CONVERGED, NAN_STATUS = 5, 6, 7

_FMT = {"s": (24, -126, 127), "d": (53, -1022, 1023)}
_libm = ctypes.CDLL(ctypes.util.find_library("m"))
for _n, _t in (("expf", ctypes.c_float), ("acos", ctypes.c_double), ("sin", ctypes.c_double), ("atan", ctypes.c_double)):
    getattr(_libm, _n).restype = _t
    getattr(_libm, _n).argtypes = [_t]


def c_expf(t: float) -> float:
    """glibc's expf, as the oracle calls it."""
    return float(_libm.expf(t))


def c_acos(x: float) -> float:
    return float(_libm.acos(x))


def c_sin(x: float) -> float:
    return float(_libm.sin(x))


def c_atan(x: float) -> float:
    return float(_libm.atan(x))


# ---- exact rounding ------------------------------------------------------------------------------------------------
def rnd(x: Fraction, fmt: str) -> float:
    """x rounded once to nearest-even in binary32 ("s") or binary64 ("d"), overflow to +-inf; returned as the Python
    float that holds that value exactly."""
    if x == 0:
        return 0.0
    p, emin, emax = _FMT[fmt]
    neg = x < 0
    x = -x if neg else x
    n, d = x.numerator, x.denominator
    e = n.bit_length() - d.bit_length()
    if (n << -e if e < 0 else n) < (d << e if e > 0 else d):
        e -= 1
    q = max(e, emin) - (p - 1)
    num, den = (n, d << q) if q >= 0 else (n << -q, d)
    m, r = divmod(num, den)
    if 2 * r > den or (2 * r == den and m & 1):
        m += 1
    v = math.inf if m.bit_length() - 1 + q > emax else math.ldexp(m, q)  # m < 2^(p+1): exact in a double
    return -v if neg else v


def _fr(x: float) -> Fraction:
    return Fraction(x)


def _fin(*xs) -> bool:
    return all(math.isfinite(x) for x in xs)


def _np(fmt):
    return np.float32 if fmt == "s" else np.float64


def add(x, y, fmt):
    if _fin(x, y):
        return rnd(_fr(x) + _fr(y), fmt)
    return float(_np(fmt)(x) + _np(fmt)(y))


def sub(x, y, fmt):
    if _fin(x, y):
        return rnd(_fr(x) - _fr(y), fmt)
    return float(_np(fmt)(x) - _np(fmt)(y))


def mul(x, y, fmt):
    if _fin(x, y):
        return rnd(_fr(x) * _fr(y), fmt)
    with np.errstate(all="ignore"):
        return float(_np(fmt)(x) * _np(fmt)(y))


def div(x, y, fmt):
    if _fin(x, y) and y != 0:
        return rnd(_fr(x) / _fr(y), fmt)
    with np.errstate(all="ignore"):
        return float(_np(fmt)(x) / _np(fmt)(y))


def fma(a, b, c, fmt):
    """a * b + c rounded once."""
    if _fin(a, b, c):
        return rnd(_fr(a) * _fr(b) + _fr(c), fmt)
    with np.errstate(all="ignore"):  # a non-finite operand: the product of two floats is exact in a double
        return float(_np(fmt)(np.float64(a) * np.float64(b) + np.float64(c)))


def sqrt(x, fmt):
    if not math.isfinite(x) or x <= 0:
        with np.errstate(all="ignore"):
            return float(np.sqrt(_np(fmt)(x)))
    f = _fr(x)
    k = 200 + max(0, -(f.numerator.bit_length() - f.denominator.bit_length()))  # r = isqrt(x 4^k) has >= 100 bits
    s = (f.numerator << (2 * k)) // f.denominator
    r = math.isqrt(s)
    exact = r * r == s and (f.numerator << (2 * k)) % f.denominator == 0
    return rnd((Fraction(r) if exact else Fraction(2 * r + 1, 2)) / (1 << k), fmt)


def f32(x: float) -> float:
    """(float) of a double."""
    return rnd(_fr(x), "s") if math.isfinite(x) else x


def same(x: float, y: float) -> bool:
    """Bit for bit, zeros by value and NaNs by class (the oracle is built with -fno-signed-zeros)."""
    return (math.isnan(x) and math.isnan(y)) or x == y


# ---- updateSeed ---------------------------------------------------------------------------------------------------------
SQRT_2PI_F = sqrt(mul(2.0, f32(3.14159265358979323846264338327950288), "s"), "s")


def pdf_exponent(x, mu, sigma2, tau2):
    """norm_scale and the exponent normal_pdf_f hands to exp (None when updateSeed returns early or x is infinite)."""
    norm_scale = sqrt(add(sigma2, tau2, "s"), "s")
    if math.isnan(norm_scale) or math.isinf(x):
        return norm_scale, None
    e = sub(x, mu, "s")
    e = mul(e, -e, "s")
    return norm_scale, div(e, mul(mul(2.0, norm_scale, "s"), norm_scale, "s"), "s")


def update_seed(x, tau2, a, b, mu, z_range, sigma2, expv):
    """(a, b, mu, sigma2) after updateSeed, with exp(exponent) = expv (a float, or a function of the exponent)."""
    norm_scale, t = pdf_exponent(x, mu, sigma2, tau2)
    if math.isnan(norm_scale):
        return a, b, mu, sigma2
    s2 = f32(div(1.0, add(div(1.0, sigma2, "d"), div(1.0, tau2, "d"), "d"), "d"))
    m = mul(s2, add(div(mu, sigma2, "s"), div(x, tau2, "s"), "s"), "s")
    if t is None:
        pdf = 0.0
    else:
        pdf = expv(t) if callable(expv) else expv
        pdf = div(pdf, mul(norm_scale, SQRT_2PI_F, "s"), "s")
    apb = add(a, b, "s")
    C1 = mul(div(a, apb, "s"), pdf, "s")
    C2 = f32(div(div(b, apb, "s"), z_range, "d"))  # ((double)(b / (a + b)) * 1.) / (double)z_range
    nc = add(C1, C2, "s")
    C1 = div(C1, nc, "s")
    C2 = div(C2, nc, "s")
    ab1 = add(apb, 1.0, "d")
    ab2 = add(apb, 2.0, "d")
    f = f32(add(div(mul(C1, add(a, 1.0, "d"), "d"), ab1, "d"), div(mul(C2, a, "s"), ab1, "d"), "d"))
    e = f32(add(div(mul(mul(C1, add(a, 1.0, "d"), "d"), add(a, 2.0, "d"), "d"), mul(ab1, ab2, "d"), "d"),
                div(mul(mul(C2, a, "s"), add(a, 1.0, "s"), "s"),
                    mul(add(apb, 1.0, "s"), add(apb, 2.0, "s"), "s"), "s"), "d"))
    mu_new = fma(C1, m, mul(C2, mu, "s"), "s")
    sigma2_new = fma(-mu_new, mu_new, fma(C1, fma(m, m, s2, "s"), mul(C2, fma(mu, mu, sigma2, "s"), "s"), "s"), "s")
    a_new = div(sub(e, f, "s"), sub(f, div(e, f, "s"), "s"), "s")
    b_new = div(mul(a_new, sub(1.0, f, "s"), "s"), f, "s")
    return a_new, b_new, mu_new, sigma2_new


def status(sigma2_new, z_range, thresh, mu_old, sigma2_old):
    """updateSeeds' verdict after the update (:261-287): converged when (double)sqrtf(sigma2) < (double)z_range / thresh
    (strict), NaN when z_inv_min = mu + sqrtf(sigma2) of the seed before the update is NaN, else updated."""
    if sqrt(sigma2_new, "s") < div(z_range, thresh, "d"):
        return CONVERGED
    if math.isnan(add(mu_old, sqrt(sigma2_old, "s"), "s")):
        return NAN_STATUS
    return UPDATED


def rn_exp(t: float) -> float:
    """e^t rounded to the nearest float (40 digits: e^t of a nonzero float is never a tie)."""
    if math.isnan(t):
        return math.nan
    man, e = mp.exp(mpf(t)).man_exp
    return rnd(Fraction(int(man)) * Fraction(2) ** int(e), "s") if man else 0.0


def _f32_step(v: float, k: int) -> float:
    x = np.float32(v)
    for _ in range(abs(k)):
        x = np.nextafter(x, np.float32(np.inf if k > 0 else 0.0), dtype=np.float32)
    return float(x)


def exp_values(t):
    """{k: RN(e^t) + k ulp} for |k| <= EXPF_ULP (never below 0)."""
    if t is None:
        return {0: None}
    r = rn_exp(t)
    if math.isnan(r):
        return {0: math.nan}
    return {k: _f32_step(r, k) for k in range(-EXPF_ULP, EXPF_ULP + 1) if not (k < 0 and r == 0.0)}


# ---- computeTau ---------------------------------------------------------------------------------------------------------
def compute_tau(t, f, z, px_error_angle, acos=c_acos, sin=c_sin):
    """computeTau in IEEE double, operation by operation (the oracle's and the kernel's order)."""
    ax, ay, az = f[0] * z - t[0], f[1] * z - t[1], f[2] * z - t[2]
    t_norm = math.sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2])
    a_norm = math.sqrt(ax * ax + ay * ay + az * az)
    alpha = acos((f[0] * t[0] + f[1] * t[1] + f[2] * t[2]) / t_norm)
    beta = acos((ax * -t[0] + ay * -t[1] + az * -t[2]) / (t_norm * a_norm))
    beta_plus = beta + px_error_angle
    gamma_plus = PI_TRUNC - alpha - beta_plus
    with np.errstate(all="ignore"):
        z_plus = float(np.float64(t_norm * sin(beta_plus)) / np.float64(sin(gamma_plus)))
    return z_plus - z


def px_error_angle(fx: float, atan=c_atan) -> float:
    return atan(1.0 / (2.0 * abs(fx))) * 2.0


# Interval evaluation at 40 digits.  A value is a list of closed intervals (lo, hi) of mpf, or None when NaN is possible.
_INF = mpf("inf")


def _widen(iv, n_half_ulp):
    out = []
    for lo, hi in iv:
        w = lambda v: n_half_ulp * U * abs(v) + mpf(2) ** -1074 if mp.isfinite(v) else 0
        out.append((lo - w(lo), hi + w(hi)))
    return out


def _binop(x, y, op, n=1):
    if x is None or y is None:
        return None
    out = []
    for a in x:
        for b in y:
            if op == "+":
                out.append((a[0] + b[0], a[1] + b[1]))
            elif op == "-":
                out.append((a[0] - b[1], a[1] - b[0]))
            elif op == "*":
                ps = [p * q for p in a for q in b]
                if any(mp.isnan(v) for v in ps):
                    return None
                out.append((min(ps), max(ps)))
            else:  # "/": a divisor interval holding 0 splits into its two signs
                parts = []
                if b[0] < 0:
                    parts.append((b[0], min(b[1], -mpf(2) ** -1074)))
                if b[1] > 0:
                    parts.append((max(b[0], mpf(2) ** -1074), b[1]))
                if b[0] == 0 and b[1] == 0:
                    return None
                for c in parts:
                    qs = [p / q for p in a for q in c]
                    if any(mp.isnan(v) for v in qs):
                        return None
                    out.append((min(qs), max(qs)))
    return _widen(out, n)


def _pt(v):
    return [(mpf(v), mpf(v))]


def _sqrt(x):
    if x is None or any(lo < 0 for lo, _ in x):
        return None
    return _widen([(mp.sqrt(lo), mp.sqrt(hi)) for lo, hi in x], 1)


def _acos(x):
    if x is None or any(lo < -1 or hi > 1 for lo, hi in x):
        return None
    return _widen([(mp.acos(hi), mp.acos(lo)) for lo, hi in x], 2 * ACOS_ULP)


def _sin(x):
    if x is None:
        return None
    out = []
    for lo, hi in x:
        if not (mp.isfinite(lo) and mp.isfinite(hi)):
            return None
        vals = [mp.sin(lo), mp.sin(hi)]
        k0, k1 = int(mp.ceil((lo - mp.pi / 2) / mp.pi)), int(mp.floor((hi - mp.pi / 2) / mp.pi))
        for k in range(k0, min(k1, k0 + 2) + 1):  # extrema inside
            vals.append(mp.sin(mp.pi / 2 + k * mp.pi))
        out.append((min(vals), max(vals)))
    return _widen(out, 2 * SIN_ULP)


def pose_t(T_ref_w, T_cur_w):
    """T_ref_cur's translation at 40 digits and the radius the device's pose product may be off by: 2 POSE_ULP u of
    |t_ref| + 3 |t_cur| (the rotation's round trip applied to t_cur, then the products' own roundings)."""
    A, B = [[mpf(float(v)) for v in row] for row in np.asarray(T_ref_w).reshape(3, 4)], \
           [[mpf(float(v)) for v in row] for row in np.asarray(T_cur_w).reshape(3, 4)]
    Rrc = [[sum(A[i][k] * B[j][k] for k in range(3)) for j in range(3)] for i in range(3)]
    t = [A[i][3] - sum(Rrc[i][j] * B[j][3] for j in range(3)) for i in range(3)]
    scale = float(max(abs(A[i][3]) for i in range(3)) + 3 * max(abs(B[i][3]) for i in range(3)))
    # An input rotation that is not orthonormal to working precision (a float32-rounded R) comes back from the round trip
    # as a nearby rotation, about its orthonormality defect away per entry rather than POSE_ULP u.
    defect = sum(float(np.max(np.abs(R @ R.T - np.eye(3)))) for R in (np.asarray(T_ref_w)[:, :3], np.asarray(T_cur_w)[:, :3]))
    return t, 2 * POSE_ULP * U * scale + 2 * defect * 3 * float(max(abs(B[i][3]) for i in range(3)))


def tau2_enclosure(t, t_rad, f, z, fx):
    """(intervals of tau_inverse^2, branch record): computeTau and tau_inverse over every input and rounding the device
    may have seen.  None in place of the intervals: a NaN is possible (an acos argument past +-1)."""
    T = [[(ti - t_rad, ti + t_rad)] for ti in t]
    F = [_pt(v) for v in f]
    Z = _pt(z)
    mul_, add_, sub_, div_ = (lambda a, b: _binop(a, b, "*")), (lambda a, b: _binop(a, b, "+")), \
                             (lambda a, b: _binop(a, b, "-")), (lambda a, b: _binop(a, b, "/"))
    A = [sub_(mul_(F[i], Z), T[i]) for i in range(3)]
    dot = lambda p, q: add_(add_(mul_(p[0], q[0]), mul_(p[1], q[1])), mul_(p[2], q[2]))
    t_norm = _sqrt(dot(T, T))
    a_norm = _sqrt(dot(A, A))
    negT = [[(-hi, -lo) for lo, hi in ti] for ti in T]
    alpha = _acos(div_(dot(F, T), t_norm))
    beta = _acos(div_(dot(A, negT), mul_(t_norm, a_norm)))
    pea_x = 2 * mp.atan(1 / (2 * abs(mpf(fx))))
    pea = _widen(_widen([(pea_x, pea_x)], 2 * ATAN_ULP), 2)  # atan, then 1/(2|fx|) and * 2
    rec = {}
    if alpha is None or beta is None:
        return None, dict(nan=True)
    beta_plus = add_(beta, pea)
    gamma_plus = sub_(sub_(_pt(PI_TRUNC), alpha), beta_plus)
    glo, ghi = min(lo for lo, _ in gamma_plus), max(hi for _, hi in gamma_plus)
    rec["gamma"] = "pos" if glo > 0 else "neg" if ghi < 0 else "both"
    s_g = _sin(gamma_plus)
    rec["sin_gamma"] = "pos" if s_g and min(lo for lo, _ in s_g) > 0 else "neg" if s_g and max(hi for _, hi in s_g) < 0 \
        else "both"
    z_plus = div_(mul_(t_norm, _sin(beta_plus)), s_g)
    if z_plus is None:
        return None, dict(rec, nan=True)
    tau = sub_(z_plus, Z)
    d1 = sub_(Z, tau)
    lim = mpf(0.0000001)
    clamp = set()
    d1c = []
    for lo, hi in d1:
        if hi <= lim:
            clamp.add(True)
            d1c.append((lim, lim))
        elif lo >= lim:
            clamp.add(False)
            d1c.append((lo, hi))
        else:
            clamp |= {True, False}
            d1c.append((lim, hi))
    rec["clamp"] = "yes" if clamp == {True} else "no" if clamp == {False} else "both"
    ti = _binop(_pt(0.5), sub_(div_(_pt(1), d1c), div_(_pt(1), add_(Z, tau))), "*")
    if ti is None:
        return None, dict(rec, nan=True)
    sq = []
    for lo, hi in ti:
        c = [lo * lo, hi * hi]
        sq.append((mpf(0) if lo <= 0 <= hi else min(c), max(c)))
    return _widen(sq, 1), rec


def _rn32(v) -> float:
    """An mpf rounded once to the nearest float (not through a double)."""
    if not mp.isfinite(v):
        return float(v)
    man, e = v.man_exp
    return rnd(Fraction(int(man)) * Fraction(2) ** int(e), "s") if man else 0.0


def _f32_bits_range(lo, hi):
    """[first, last] uint32 patterns of the floats in [RN(lo), RN(hi)] (lo clipped at 0): tau2 is the double
    tau_inverse^2, which the enclosure holds, rounded to the nearest float, and rounding is monotone."""
    a, b = np.float32(_rn32(max(lo, mpf(0)))), np.float32(_rn32(hi))
    return int(np.array(a, np.float32).view(np.uint32)), int(np.array(b, np.float32).view(np.uint32))


def tau2_values(enc):
    """The admissible float tau2 of an enclosure: (list of floats or None when there are more than MAX_TAU2, count)."""
    if enc is None:
        return None, math.inf
    ranges = sorted(_f32_bits_range(lo, hi) for lo, hi in enc)
    merged = []
    for a, b in ranges:
        if merged and a <= merged[-1][1] + 1:
            merged[-1][1] = max(merged[-1][1], b)
        else:
            merged.append([a, b])
    n = sum(b - a + 1 for a, b in merged)
    if n > MAX_TAU2:
        return None, n
    vals = [float(np.array(v, np.uint32).view(np.float32)) for a, b in merged for v in range(a, b + 1)]
    return vals, n


def oracle_tau2(t, f, z, fx) -> float:
    """tau2 = (float)(tau_inverse^2) as the oracle computes it from its own T_ref_cur translation t: computeTau with
    glibc's acos / sin / atan, std::max(1e-7, z - tau) (1e-7 for a NaN), every double operation IEEE."""
    with np.errstate(all="ignore"):
        tau = np.float64(compute_tau(t, f, z, px_error_angle(fx)))
        zt = np.float64(z) - tau
        d1 = zt if np.float64(0.0000001) < zt else np.float64(0.0000001)
        ti = np.float64(0.5) * (np.float64(1.0) / d1 - np.float64(1.0) / (np.float64(z) + tau))
        return f32(float(ti * ti))


def x_of(z: float) -> float:
    """x = (float)(1. / z), exactly."""
    return f32(1.0 / z) if z != 0 else f32(math.copysign(math.inf, z))


# ---- candidates ---------------------------------------------------------------------------------------------------------
def candidates(z, t, t_rad, f, fx, seed, thresh, exp="device", tau2_exact=None):
    """Every (a, b, mu, sigma2, status) updateSeed and the convergence test may produce for the seed `seed` (a, b, mu,
    z_range, sigma2 before the update) matched at depth z.  exp: "device" (RN(e^t) + k ulp, |k| <= 2) or "glibc".
    tau2_exact: the one tau2 of a host computation restated in IEEE double (`oracle_tau2`) in place of the enclosure's
    floats; it must lie among them when they are few enough to list (`outside` is set otherwise).
    Returns dict(cands = {(tau2, k): tuple}, n_tau2, ill (the enclosure holds more than MAX_TAU2 floats), rec, samples:
    for an ill-conditioned seed, the outputs at up to 9 tau2 across the enclosure (k = 0))."""
    a, b, mu, zr, s2 = (float(np.float32(v)) for v in seed)
    x = x_of(z)
    enc, rec = tau2_enclosure(t, t_rad, f, z, fx)
    vals, n = tau2_values(enc)
    out = dict(n_tau2=n, ill=vals is None, rec=rec, cands={}, x=x, outside=False)
    if tau2_exact is not None:
        out["outside"] = vals is not None and not any(same(tau2_exact, v) for v in vals)
        vals, out["n_tau2"], out["ill"] = [tau2_exact], 1, False

    def one(tau2, ev):
        r = update_seed(x, tau2, a, b, mu, zr, s2, ev)
        return r + (status(r[3], zr, thresh, mu, s2),)

    def exps(tau2):
        _, t_ = pdf_exponent(x, mu, s2, tau2)
        if exp == "glibc":
            return {0: (c_expf(t_) if t_ is not None else None)}
        return exp_values(t_)

    if vals is not None:
        for tau2 in vals:
            for k, ev in exps(tau2).items():
                out["cands"][(tau2, k)] = one(tau2, ev)
    else:
        pts = []
        if enc is not None:
            for lo, hi in enc:
                lo = max(lo, mpf(0))
                pts += [lo, hi] + ([mp.sqrt(lo * hi)] if lo > 0 and mp.isfinite(hi) else [])
        pts = [f32(float(p)) if p < mpf("3.5e38") else math.inf for p in pts][:9] + ([math.nan] if enc is None else [])
        out["samples"] = [one(tau2, exps(tau2).get(0)) for tau2 in pts]
    return out


def matches(g, cands):
    """The key of the candidate the tuple g = (a, b, mu, sigma2, status) equals (zeros by value, NaNs by class), or None."""
    for key, c in cands.items():
        if g[4] == c[4] and all(same(float(np.float32(u)), v) for u, v in zip(g[:4], c[:4])):
            return key
    return None


def decisive_check(g, samples):
    """An ill-conditioned seed: every output the sampled tau2 agree on -- the status, and which fields are NaN -- must be
    the kernel's.  This is a heuristic, not a bound: a decision could flip between two samples, so callers also compare
    such seeds with the oracle numerically.  Returns the list of disagreements."""
    bad = []
    if not samples:
        return bad
    st = {s[4] for s in samples}
    if len(st) == 1 and g[4] not in st:
        bad.append(("status", g[4], st))
    for j, name in enumerate(("a", "b", "mu", "sigma2")):
        cls = {math.isnan(s[j]) for s in samples}
        if len(cls) == 1 and math.isnan(float(g[j])) not in cls:
            bad.append((name, float(g[j])))
    return bad


# ---- depthFromTriangulation ---------------------------------------------------------------------------------------------
# TRI_K is not derived: it covers the first-order estimate in `triangulation`'s docstring with a margin (the worst seed
# of the tests sits at ~0.07 of the bound).
TRI_K = 64


def pinhole_bearing(cam, u, v):
    """vk::PinholeCamera::cam2world of an undistorted camera, at 40 digits."""
    x, y = (mpf(float(u)) - mpf(cam.cx)) / mpf(cam.fx), (mpf(float(v)) - mpf(cam.cy)) / mpf(cam.fy)
    n = mp.sqrt(x * x + y * y + 1)
    return [x / n, y / n, 1 / n]


def triangulation(T_cur_ref, f_ref, f_cur):
    """depthFromTriangulation at 40 digits: (depth, det, depth bound, det uncertainty).  The device forms R f_ref and t from
    its quaternion pose (POSE_ULP u per entry) and f_cur from the pixel (a few u); each perturbs det and the two dot
    products by ~delta = 16 u, so |depth - exact| <= TRI_K u (|t| + |depth|) / det."""
    T = [[mpf(float(v)) for v in row] for row in np.asarray(T_cur_ref).reshape(3, 4)]
    fr = [mpf(float(v)) for v in f_ref]
    a0 = [sum(T[i][j] * fr[j] for j in range(3)) for i in range(3)]
    a1 = list(f_cur)
    d = lambda p, q: p[0] * q[0] + p[1] * q[1] + p[2] * q[2]
    m00, m01, m11 = d(a0, a0), d(a0, a1), d(a1, a1)
    det = m00 * m11 - m01 * m01
    t = [T[i][3] for i in range(3)]
    depth = abs(-(m11 / det * d(a0, t) - m01 / det * d(a1, t))) if det != 0 else mpf("inf")
    tn = mp.sqrt(d(t, t))
    bound = float(TRI_K * U * (tn + depth) / det) if det > 0 else math.inf
    det_unc = float(TRI_K * U * (m00 * m11 + m01 * m01))
    return float(depth), float(det), bound, det_unc


# ---- one launch -------------------------------------------------------------------------------------------------------
def check_launch(out, seeds, kf_T, ref_index, T_cur_w, ftr_f, fx, thresh=200.0, exp="device", only=None, oracle=None):
    """Every seed of one depth filter launch that reached updateSeed (status UPDATED, CONVERGED or NAN), from the depth z
    the launch reported: its (a, b, mu, sigma2, status) must be one of `candidates`, or, where more than MAX_TAU2 floats
    are admissible for tau2, agree with every decision the sampled tau2 agree on (`only`: a mask of the seeds to check).
    oracle (the oracle binding, with exp="glibc"): the launch is the oracle's; tau2 is pinned to `oracle_tau2` of the
    oracle's own T_ref_cur, so every seed has a single candidate.
    Returns a report: n (seeds checked), single (one admissible tau2), ill and ill_idx, k (histogram of the exp offset of
    the matching candidate; candidates of several k that give the same tuple count at the smallest |k|), rec (branch
    counts over the candidate-checked seeds) and bad (the seeds that failed)."""
    rep = dict(n=0, single=0, ill=0, ill_idx=[], k={}, rec={}, bad=[])
    poses = {}
    sel = np.asarray(out["status"]) >= UPDATED
    for i in np.flatnonzero(sel if only is None else sel & only):
        r_ix = int(ref_index[i])
        if r_ix not in poses:
            poses[r_ix] = pose_t(kf_T[r_ix], T_cur_w)
            if oracle is not None:
                poses[r_ix] += ([float(v) for v in oracle.se3_mul(kf_T[r_ix], oracle.se3_inv(T_cur_w))[:, 3]],)
        t, rad = poses[r_ix][:2]
        seed = tuple(float(np.float32(seeds[k][i])) for k in ("a", "b", "mu", "z_range", "sigma2"))
        f = [float(v) for v in ftr_f[i]]
        z = float(out["z"][i])
        t2 = oracle_tau2(poses[r_ix][2], f, z, fx) if oracle is not None else None
        r = candidates(z, t, rad, f, fx, seed, thresh, exp, tau2_exact=t2)
        g = tuple(float(np.float32(out[k][i])) for k in ("a", "b", "mu", "sigma2")) + (int(out["status"][i]),)
        rep["n"] += 1
        if r["ill"]:
            rep["ill"] += 1
            rep["ill_idx"].append(int(i))
            bad = decisive_check(g, r.get("samples"))
            if bad:
                rep["bad"].append((int(i), "decisive", bad))
            continue
        for name, v in r["rec"].items():
            rep["rec"][f"{name}={v}"] = rep["rec"].get(f"{name}={v}", 0) + 1
        rep["single"] += r["n_tau2"] == 1
        if r["outside"]:
            rep["bad"].append((int(i), "tau2 outside the enclosure", t2))
        keys = [k for k, c in r["cands"].items() if matches(g, {k: c}) is not None]
        if not keys:
            rep["bad"].append((int(i), g, seed, z, sorted(set(r["cands"].values()))[:6]))
            continue
        k = min((key[1] for key in keys), key=abs)
        rep["k"][k] = rep["k"].get(k, 0) + 1
    return rep


def assert_seed_updates(g, o, seeds, kf_T, ref_index, T_cur_w, ftr_f, fx, oracle, thresh=200.0, oracle_statement=True):
    """The seed check of a depth filter launch g (the kernel's) against the oracle's o of the same inputs: seeds that
    never reach updateSeed bit-identical (NaNs by class); every updated seed of the kernel one of the statement's
    candidates (`check_launch`), and, where its tau2 enclosure is too wide to list, within 2e-5 of the oracle as well;
    with oracle_statement, every updated seed of the oracle bit for bit its own statement (tau2 pinned, glibc's expf).
    Returns the kernel's report."""
    upd = np.asarray(o["status"]) >= UPDATED
    for k in ("a", "b", "mu", "sigma2"):
        x, y = np.asarray(g[k], np.float32)[~upd], np.asarray(o[k], np.float32)[~upd]
        assert np.all((x.view(np.uint32) == y.view(np.uint32)) | (np.isnan(x) & np.isnan(y))), k
    rep = check_launch(g, seeds, kf_T, ref_index, T_cur_w, ftr_f, fx, thresh, "device")
    assert not rep["bad"], ("kernel", rep["bad"][:3])
    ill = np.asarray(rep["ill_idx"], int)
    for k in ("a", "b", "mu", "sigma2"):
        assert np.allclose(np.asarray(g[k])[ill], np.asarray(o[k])[ill], rtol=2e-5, atol=1e-7, equal_nan=True), k
    if oracle_statement:
        ro = check_launch(o, seeds, kf_T, ref_index, T_cur_w, ftr_f, fx, thresh, "glibc", oracle=oracle)
        assert not ro["bad"], ("oracle", ro["bad"][:3])
    return rep
