"""A high-precision statement of pose_optimizer::optimizeGaussNewton (svo/src/pose_optimizer.cpp:28-161, with
Frame::jacobian_xyz2uv of svo/include/svo/frame.h:116-138) for the tests of pose_opt_kernel.

Working precision.  Every double quantity is computed from the double inputs in mpmath at `dps` (40) significant digits,
so against a double implementation it is exact.  The pose is applied as the kernel applies it: T_f_w goes through its
quaternion (the matrix-to-quaternion conversion of pose_from_rt12, then the quaternion's rotation matrix), at working
precision; an update is the exact SE(3) exponential left-multiplied onto the pose.  Non-finite values follow IEEE rules
(x/0 = +-inf, 0/0 = NaN, 0 * inf = NaN, comparisons with NaN false).

Float steps as candidate sets.  Four steps of the reference round to float: errors.push_back(e.norm()), 1.48f * median,
(float)(e.norm() / scale) and the Tukey weight (b = 4.6851f, evaluated in float).  Each exact value maps to the set of
floats that a double computation within its error bound can round to (rounding is monotone, so the set is the floats
between the roundings of the bound's two ends); the float arithmetic on those candidates is numpy float32, which is IEEE
and equals the kernel's __fmul_rn / __fdiv_rn.  The median (vk::getMedian: element n/2 of nth_element) of values known
as intervals is an interval, [n/2-th lower end, n/2-th upper end].  NaN sorts above +inf (the kernel's order_key); the
reference leaves a NaN's place to libstdc++'s nth_element, which this statement does not emulate.

Decisions, each with a margin.  Roll back on `iter > 0 && new_chi2 > chi2` or a NaN dT[0]; stop when max|dT| <= EPS
(1e-10); switch to scale = 0.85 / fx at iteration 5; cull when sqrt(e^2) > fl(reproj_thresh / fx).  A decision is decisive
when its margin exceeds TIE_REL relative and the kernel's own uncertainty in the compared quantities; a near-tie may go
either way, and `branches` follows both.  A scale whose candidate set holds more than one float is a tie between those
floats: `branches` runs each.  A culling test within the uncertainty of the error it compares leaves that observation's
flag open (`cull_open`).

Bound on the pose.  Iteration i forms A = sum w J^T J and b = -sum w J^T e as double sums over the frame's n
observations and solves the 6x6 system; then it applies exp(dT) to the pose.  With lam the smallest eigenvalue of A:
  * each residual is known to de_j ~ K u (1 + |project2d| + |X| / z) (scaled by sqrt_inv_cov).  Since A = J^T W J,
    |A^-1 J^T W^1/2|_2 = lam^-1/2 exactly, so the residual rounding moves the step by at most sqrt(sum w de_j^2 / lam);
  * the sums carry a relative (n + 1) u each: through A that moves the step by (n + 1) u cond(A) |dT|, through b by
    (n + 1) u sum w |J| |e| / lam;
  * the LDL^T solve is backward stable (inside the cond(A) |dT| term) and the pose update rounds at u (1 + |t|).
The per-iteration errors add (Gauss-Newton corrects an error in the pose it starts from, so adding them overstates it):

    |T_kernel - T_exact| <= sum_i K [sqrt(sum w de^2 / lam_i) + (n + 1) u (cond(A_i) |dT_i| + sum w |J| |e| / lam_i)
                                     + u (1 + |t|)]   (+ a weight term, below)

K = 8, as in tests/point_hp.py.  The older form K u cond(A)(n + 1)(s + |dT|) charges every iteration the whole scale s of
the scene, ~1e-9 on a 120-observation frame: fed back into the float candidate sets of the next iteration's weights, that
spread every weight and made the bound grow without end.  Where a Tukey weight still has more than one float candidate,
the spread dw of that weight moves the step by at most dw |J| (|J| |dT| + |e|) / lam; that is added.
The bound is on the largest entry of the 3x4 [R | t] (scaled by 1 + |t| for the translation column).

Covariance.  Cov = (A fx^2)^-1 with the A of the last iteration computed -- the rejected one after a roll-back -- known to
a relative ~K u (n + 1) cond(A) in any implementation.
"""
from __future__ import annotations

import math

import numpy as np
from mpmath import mp, mpf

DPS = 40
mp.dps = DPS

U = 2.0 ** -53
K = 8.0
TIE_REL = 1e-9
EPS = 0.0000000001            # the double constant EPS of global.h:77
NAN, INF = mpf("nan"), mpf("inf")
B_TUKEY = np.float32(4.6851)


# ---- scalar helpers ------------------------------------------------------------------------------------------------
def _div(a, b):
    """a / b with IEEE semantics for b == 0 (mpmath raises there); a zero divisor counts as +0 (mpmath has no -0)."""
    if mp.isnan(a) or mp.isnan(b):
        return NAN
    if b == 0:
        if a == 0:
            return NAN
        return INF if a > 0 else -INF
    if mp.isinf(a) and mp.isinf(b):
        return NAN
    return a / b


def _mul(a, b):
    if (a == 0 and mp.isinf(b)) or (b == 0 and mp.isinf(a)):
        return NAN
    return a * b


def _add(a, b):
    if mp.isinf(a) and mp.isinf(b) and (a > 0) != (b > 0):
        return NAN
    return a + b


def _isnan(x) -> bool:
    return bool(mp.isnan(x))


def _fin(x) -> bool:
    return bool(mp.isfinite(x))


def _f32(x) -> np.float32:
    """Round a working-precision value to float through double, as the kernel casts (monotone: used on interval ends)."""
    with np.errstate(over="ignore"):
        return np.float32(float(x))


def f32_interval(lo, hi, cap=64):
    """Every float a double in [lo, hi] can round to (NaN: {NaN}).  Capped at `cap` entries (a wider set is returned as
    its two ends, which still brackets every candidate)."""
    if _isnan(lo) or _isnan(hi):
        return [np.float32(np.nan)]
    a, b = _f32(min(lo, hi)), _f32(max(lo, hi))
    out = [a]
    while out[-1] < b and len(out) < cap:
        out.append(np.nextafter(out[-1], np.float32(np.inf), dtype=np.float32))
    if out[-1] != b:
        out = [a, b]
    return out


def tukey(x: np.float32) -> np.float32:
    """vk::robust_cost::TukeyWeightFunction::value in float (b = 4.6851f)."""
    with np.errstate(all="ignore"):
        b2 = B_TUKEY * B_TUKEY
        x2 = np.float32(x) * np.float32(x)
        if x2 <= b2:
            t = np.float32(1) - x2 / b2
            return np.float32(t * t)
        return np.float32(0)


def order_key(v):
    """Sort key with NaN above +inf (the kernel's order_key on IEEE bits)."""
    v = float(v)
    return (1, 0.0) if math.isnan(v) else (0, v)


def kth(vals, k):
    return sorted(vals, key=order_key)[k]


# ---- pose at working precision -------------------------------------------------------------------------------------
def qfrommatrix(R):
    """pose_from_rt12's matrix -> quaternion (the branch on the trace and the largest diagonal)."""
    t = R[0][0] + R[1][1] + R[2][2]
    if t > 0:
        t = mp.sqrt(t + 1)
        w = t / 2
        t = mpf(0.5) / t
        return w, (R[2][1] - R[1][2]) * t, (R[0][2] - R[2][0]) * t, (R[1][0] - R[0][1]) * t
    if R[0][0] >= R[1][1] and R[0][0] >= R[2][2]:
        t = mp.sqrt(R[0][0] - R[1][1] - R[2][2] + 1)
        x = t / 2
        t = mpf(0.5) / t
        return (R[2][1] - R[1][2]) * t, x, (R[1][0] + R[0][1]) * t, (R[2][0] + R[0][2]) * t
    if R[1][1] >= R[2][2]:
        t = mp.sqrt(R[1][1] - R[2][2] - R[0][0] + 1)
        y = t / 2
        t = mpf(0.5) / t
        return (R[0][2] - R[2][0]) * t, (R[1][0] + R[0][1]) * t, y, (R[2][1] + R[1][2]) * t
    t = mp.sqrt(R[2][2] - R[0][0] - R[1][1] + 1)
    z = t / 2
    t = mpf(0.5) / t
    return (R[1][0] - R[0][1]) * t, (R[2][0] + R[0][2]) * t, (R[2][1] + R[1][2]) * t, z


def qmatrix(q):
    w, x, y, z = q
    return [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
            [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
            [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]


def start_pose(T):
    """(R, t) of T_f_w after the quaternion round trip, at working precision."""
    T = np.asarray(T, np.float64).reshape(3, 4)
    R = [[mpf(float(T[r, c])) for c in range(3)] for r in range(3)]
    t = [mpf(float(T[r, 3])) for r in range(3)]
    if not all(_fin(v) for row in R for v in row):
        return [[NAN] * 3 for _ in range(3)], t
    return qmatrix(qfrommatrix(R)), t


def _hat(w):
    return [[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]


def _mm(A, B):
    return [[sum(A[r][k] * B[k][c] for k in range(3)) for c in range(3)] for r in range(3)]


def se3_exp(u):
    """SE(3) exponential of u = [v, omega] (Sophus::SE3::exp): (R, t)."""
    v, w = u[:3], u[3:]
    th2 = w[0] ** 2 + w[1] ** 2 + w[2] ** 2
    th = mp.sqrt(th2)
    W = _hat(w)
    W2 = _mm(W, W)
    if th2 == 0:
        a, b, s = mpf(0.5), mpf(1) / 6, mpf(1)
        c1 = mpf(0.5)
    else:
        s = mp.sin(th) / th
        c1 = (1 - mp.cos(th)) / th2
        a, b = c1, (th - mp.sin(th)) / (th2 * th)
    I = [[mpf(int(r == c)) for c in range(3)] for r in range(3)]
    R = [[I[r][c] + s * W[r][c] + c1 * W2[r][c] for c in range(3)] for r in range(3)]
    V = [[I[r][c] + a * W[r][c] + b * W2[r][c] for c in range(3)] for r in range(3)]
    t = [sum(V[r][k] * v[k] for k in range(3)) for r in range(3)]
    return R, t


def compose(A, B):
    (Ra, ta), (Rb, tb) = A, B
    return _mm(Ra, Rb), [sum(Ra[r][k] * tb[k] for k in range(3)) + ta[r] for r in range(3)]


# ---- 6x6 solve -----------------------------------------------------------------------------------------------------
TINY = mpf(1.0 / 1.7976931348623157e308)


def ldlt_solve(A, b):
    """The symmetric-pivoting LDL^T solve of ldlt6_factor / Eigen::LDLT at working precision (largest remaining diagonal
    first, a zero first pivot ends the factorisation, the solve zeroes the components whose |pivot| <= 1/DBL_MAX)."""
    n = len(b)
    if not all(_fin(v) for row in A for v in row) or not all(_fin(v) for v in b):
        return [NAN] * n
    A = [row[:] for row in A]
    tr = list(range(n))
    for k in range(n):
        big, bigv = k, abs(A[k][k])
        for i in range(k + 1, n):
            if abs(A[i][i]) > bigv:
                bigv, big = abs(A[i][i]), i
        tr[k] = big
        if big != k:
            for j in range(k):
                A[k][j], A[big][j] = A[big][j], A[k][j]
            for i in range(big + 1, n):
                A[i][k], A[i][big] = A[i][big], A[i][k]
            A[k][k], A[big][big] = A[big][big], A[k][k]
            for i in range(k + 1, big):
                A[i][k], A[big][i] = A[big][i], A[i][k]
        if k > 0:
            temp = [A[j][j] * A[k][j] for j in range(k)]
            A[k][k] -= sum(A[k][j] * temp[j] for j in range(k))
            for i in range(k + 1, n):
                A[i][k] -= sum(A[i][j] * temp[j] for j in range(k))
        akk = A[k][k]
        if k == 0 and akk == 0:
            tr = list(range(n))
            break
        if akk != 0:
            for i in range(k + 1, n):
                A[i][k] = A[i][k] / akk
    x = list(b)
    for i in range(n):
        j = tr[i]
        x[i], x[j] = x[j], x[i]
    for i in range(1, n):
        for j in range(i):
            x[i] -= A[i][j] * x[j]
    for i in range(n):
        x[i] = x[i] / A[i][i] if abs(A[i][i]) > TINY else mpf(0)
    for i in range(n - 2, -1, -1):
        for j in range(i + 1, n):
            x[i] -= A[j][i] * x[j]
    for i in range(n - 1, -1, -1):
        j = tr[i]
        x[i], x[j] = x[j], x[i]
    return x


def eig_range(A):
    """(largest |eigenvalue|, smallest |eigenvalue| above 1e-35 of it) of the symmetric A; (nan, nan) if not finite."""
    if not all(_fin(v) for row in A for v in row):
        return math.nan, math.nan
    ev = [abs(e) for e in mp.eigsy(mp.matrix(A), eigvals_only=True)]
    top = max(ev)
    if top == 0:
        return 0.0, 0.0
    live = [e for e in ev if e > top * mpf("1e-35")]
    return float(top), float(min(live))


def cond(A) -> float:
    """2-norm condition number of the symmetric A, counting eigenvalues that are 40-digit rounding of 0 (inf then)."""
    if not all(_fin(v) for row in A for v in row):
        return math.nan
    ev = [abs(e) for e in mp.eigsy(mp.matrix(A), eigvals_only=True)]
    top, bot = max(ev), min(ev)
    if top == 0:
        return 1.0
    return math.inf if bot <= top * mpf("1e-35") else float(top / bot)


# ---- the observations --------------------------------------------------------------------------------------------
class Frame:
    """The frame's observations with has_point set, at working precision."""

    def __init__(self, reproj_thresh, fx, f, pos, level, has_point, exact=False):
        hp = np.asarray(has_point).astype(bool)
        self.exact = exact  # every residual is computed without a rounding (the case says why)
        self.idx = np.flatnonzero(hp)
        self.fx = float(fx)
        self.thresh = float(np.float64(reproj_thresh) / np.float64(fx))    # reproj_thresh / errorMultiplier2(), in double
        f, pos = np.asarray(f, np.float64), np.asarray(pos, np.float64)
        lv = np.asarray(level)
        self.obs = []
        for i in self.idx:
            fi = [mpf(float(v)) for v in f[i]]
            self.obs.append(dict(ox=_div(fi[0], fi[2]), oy=_div(fi[1], fi[2]), X=[mpf(float(v)) for v in pos[i]],
                                 sic=mpf(1) / (1 << int(lv[i]))))

    def residuals(self, R, t, jac=True):
        """Per observation: e (2), |e|^2, J (2x6, scaled by sqrt_inv_cov) and the residual uncertainty de."""
        out = []
        for o in self.obs:
            X = o["X"]
            p = [_add(_add(_add(_mul(R[r][0], X[0]), _mul(R[r][1], X[1])), _mul(R[r][2], X[2])), t[r]) for r in range(3)]
            px, py = _div(p[0], p[2]), _div(p[1], p[2])
            sic = o["sic"]
            ex, ey = _mul(_add(o["ox"], -px), sic), _mul(_add(o["oy"], -py), sic)
            e2 = _add(_mul(ex, ex), _mul(ey, ey))
            size = [abs(v) for v in (o["ox"], o["oy"], px, py) if _fin(v)]
            xs = [abs(v) for v in X + t if _fin(v)]
            de = K * U * float(sic) * (1.0 + float(max(size, default=0)) +
                                       (float(max(xs, default=0)) / float(abs(p[2])) if _fin(p[2]) and p[2] != 0 else 0.0))
            r = dict(e=(ex, ey), e2=e2, de=0.0 if self.exact else de, z=p[2], proj=float(max(size, default=0)))
            if jac:
                zi = _div(mpf(1), p[2])
                zi2 = _mul(zi, zi)
                x, y = p[0], p[1]
                j02 = _mul(x, zi2)
                j12 = _mul(y, zi2)
                J0 = [-zi, mpf(0), j02, _mul(y, j02), -_add(mpf(1), _mul(x, j02)), _mul(y, zi)]
                J1 = [mpf(0), -zi, j12, _add(mpf(1), _mul(y, j12)), -_mul(y, j02), -_mul(x, zi)]
                r["J"] = ([_mul(v, sic) for v in J0], [_mul(v, sic) for v in J1])
            out.append(r)
        return out


def _interval_kth(los, his, k):
    return kth(los, k), kth(his, k)


def scale_candidates(fr: Frame, R, t):
    """(candidate floats of 1.48f * median(errors), the median's candidates, per-observation float error intervals)."""
    res = fr.residuals(R, t, jac=False)
    los, his = [], []
    for r in res:
        en = mp.sqrt(r["e2"]) if not _isnan(r["e2"]) else NAN
        cands = f32_interval(en - r["de"] if _fin(en) else en, en + r["de"] if _fin(en) else en)
        los.append(cands[0])
        his.append(cands[-1])
    k = len(res) // 2
    lo, hi = _interval_kth(los, his, k)
    meds = sorted({float(v) for v in los + his if order_key(lo) <= order_key(v) <= order_key(hi)} |
                  {float(lo), float(hi)}, key=order_key)
    if any(math.isnan(m) for m in meds):
        meds = [m for m in meds if not math.isnan(m)] + [math.nan]
    with np.errstate(all="ignore"):
        scales = sorted({float(np.float32(1.48) * np.float32(m)) for m in meds}, key=order_key)
    if any(math.isnan(s) for s in scales):
        scales = [s for s in scales if not math.isnan(s)] + [math.nan]
    return scales, meds


def normal_system(fr: Frame, R, t, scale, err):
    """A, b, chi2 of one iteration at (R, t) with the double `scale`; per-observation squared errors; the weight spread
    term; chi2's uncertainty; max |J| for culling.  `err`: bound on the kernel's pose distance from (R, t)."""
    res = fr.residuals(R, t)
    A = [[mpf(0)] * 6 for _ in range(6)]
    b = [mpf(0)] * 6
    chi2 = mpf(0)
    spread = []  # (dw, |J|, |e|) of the observations whose float weight is not unique
    rsum, jes, jw = 0.0, 0.0, 0.0  # sum w de^2 (residual rounding), sum w |J| |e| (b's summation error), max |J| at w > 0
    n = len(res)
    max_de, max_j = 0.0, 0.0
    sc = mpf(scale)
    for r in res:
        J0, J1 = r["J"]
        ex, ey = r["e"]
        en = mp.sqrt(r["e2"]) if not _isnan(r["e2"]) else NAN
        jn = max((float(abs(v)) for v in J0 + J1 if _fin(v)), default=0.0)
        de = r["de"] + jn * err
        max_j = max(max_j, jn)
        if _fin(en):
            cands = f32_interval(_div(en - de, sc), _div(en + de, sc))
        else:
            cands = [_f32(_div(en, sc))]
        ws = [tukey(c) for c in cands]
        x_nom = _f32(_div(en, sc))
        w = tukey(x_nom)
        dw = max(abs(float(v) - float(w)) for v in ws)
        if dw > 0:
            spread.append((dw, jn, float(en) if _fin(en) else math.inf))
        wm = mpf(float(w))
        wf = float(max(ws))
        if wf > 0:   # an observation of weight 0 adds exact zeros to chi2 and A
            max_de, jw = max(max_de, de), max(jw, jn)
        rsum += wf * r["de"] ** 2
        if wf > 0:
            jes += wf * jn * (float(en) if _fin(en) else math.inf)
        for rr in range(6):
            for c in range(6):
                A[rr][c] = _add(A[rr][c], _mul(_add(_mul(J0[rr], J0[c]), _mul(J1[rr], J1[c])), wm))
            b[rr] = _add(b[rr], -_mul(_add(_mul(J0[rr], ex), _mul(J1[rr], ey)), wm))
        chi2 = _add(chi2, _mul(r["e2"], wm))
    c2 = float(chi2) if _fin(chi2) else math.inf
    unc = 2.0 * math.sqrt(n * abs(c2)) * max_de + n * max_de ** 2 + K * n * U * abs(c2) if math.isfinite(c2) else math.inf
    unc += sum(dw * (en * en if math.isfinite(en) else math.inf) for dw, _, en in spread)
    return A, b, chi2, [r["e2"] for r in res], spread, unc, (rsum, jes, jw)


def optimize(reproj_thresh, n_iter, fx, T_init, f, pos, level, has_point, force=None, scale_pick=0, cache=None, exact=False):
    """optimizeGaussNewton at working precision.  `force` maps an iteration to the branch to take there regardless of the
    exact comparison ("rollback" / "accept" at the chi2 test, "stop" / "continue" at the EPS test); `scale_pick` picks one
    of the MAD scale's float candidates.  Returns a dict with the final pose, its bound, the trace and every output's
    exact value or candidate set."""
    force = force or {}
    cache = {} if cache is None else cache
    if "fr" not in cache:
        cache["fr"] = Frame(reproj_thresh, fx, f, pos, level, has_point, exact)
        cache["T0"] = start_pose(T_init)
        cache["ns"] = {}
    fr = cache["fr"]
    N = len(np.asarray(has_point))
    n = len(fr.obs)
    T_in = np.asarray(T_init, np.float64).reshape(3, 4)
    run = dict(n=n, N=N, force=force, scale_pick=scale_pick, trace=[], T_init=T_in)
    if n == 0:  # errors.empty() -> return: pose, flags untouched, outputs zero
        run.update(empty=True, untouched=True, T=None, bound=0.0, scale_cands=[0.0], scale=0.0, n_iter_done=0,
                   has_point=np.asarray(has_point, np.uint8).copy(), num_obs=0, cull_open=np.zeros(N, bool),
                   error_init=(0.0, 0.0), error_final=(0.0, 0.0), A=None, ties=[])
        return run
    run["empty"] = False
    R, t = cache["T0"]
    T_old = (R, t)
    if "scale" not in cache:
        cache["scale"] = scale_candidates(fr, R, t)
    scales, meds = cache["scale"]
    est = scales[min(scale_pick, len(scales) - 1)]
    run["scale_cands"] = scales
    run["median_cands"] = meds
    run["scale"] = est
    ties = ["scale"] if len(scales) > 1 else []
    scale = est
    chi2, chi2_unc = mpf(0), 0.0
    # the kernel's rotation matrix of the start pose, rounded from its quaternion (exact for the identity)
    err = 0.0 if np.array_equal(T_in[:, :3], np.eye(3)) else 4 * U
    err_old = err
    e2_init = None
    A_last, spread_last, jw_last = None, [], 0.0
    untouched = True
    iters = 0
    for it in range(n_iter):
        if it == 5:
            scale = float(np.float64(0.85) / np.float64(fx))
        key = (it >= 5, scale, tuple(map(tuple, R)), tuple(t))
        if key not in cache["ns"]:
            A, b, new_chi2, e2s, spread, unc, sums = normal_system(fr, R, t, scale, err)
            dT = ldlt_solve(A, b)
            top, bot = eig_range(A)
            cache["ns"][key] = (A, b, new_chi2, e2s, spread, unc, dT, top, bot, sums)
        A, b, new_chi2, e2s, spread, unc, dT, top, bot, (rsum, jes, jw) = cache["ns"][key]
        if it == 0:
            e2_init = e2s
        A_last, spread_last, jw_last = A, spread, jw
        iters += 1
        c = (top / bot if bot > 0 else math.inf) if not math.isnan(top) else math.nan
        nan_step = _isnan(dT[0])
        max_dT = max(abs(v) for v in dT) if not any(_isnan(v) for v in dT) else NAN
        step = float(mp.sqrt(sum(v * v for v in dT))) if not nan_step else math.nan
        tnorm = max((float(abs(v)) for v in t if _fin(v)), default=0.0)
        if top > 0:
            term = K * (math.sqrt(rsum / bot) + (n + 1) * U * (c * step + jes / bot) + U * (1.0 + tnorm)) if bot > 0 else math.inf
        else:
            term = 0.0
        if spread and bot > 0:
            term += sum(dw * jn * (jn * step + en) for dw, jn, en in spread) / bot
        singular = not math.isnan(top) and top > 0 and cond(A) > 1e30   # rank-deficient: its null-space pivots are noise
        rec = dict(it=it, chi2=chi2, new_chi2=new_chi2, dT=dT, max_dT=max_dT, cond=math.inf if singular else c, scale=scale, tie=None,
                   n_spread=len(spread))
        run["trace"].append(rec)
        increased = False
        if it > 0 and not nan_step:
            u_all = unc + chi2_unc
            rec["chi2_margin"] = float(abs(_div(new_chi2 - chi2, chi2))) if chi2 != 0 else (math.inf if new_chi2 != 0 else 0.0)
            if not (abs(float(new_chi2 - chi2)) > TIE_REL * abs(float(chi2)) + u_all) or not math.isfinite(u_all):
                rec["tie"] = "chi2"
            increased = new_chi2 > chi2
            if force.get(it) in ("rollback", "accept"):
                increased = force[it] == "rollback"
        if (it > 0 and increased) or nan_step:
            rec["decision"] = "nan" if nan_step else "rollback"
            R, t = T_old
            err = err_old
            untouched = T_old is cache["T0"]
            break
        T_new = compose(se3_exp(dT), (R, t))
        T_old, err_old = (R, t), err
        R, t = T_new
        untouched = False
        err = err + term
        chi2, chi2_unc = new_chi2, unc
        rec["eps_margin"] = float((max_dT - EPS) / EPS)
        if not (abs(float(max_dT) - EPS) > TIE_REL * EPS + term + err_old):
            rec["tie"] = "eps" if rec["tie"] is None else "chi2+eps"
        stop = max_dT <= EPS
        if force.get(it) in ("stop", "continue"):
            stop = force[it] == "stop"
        if stop:
            rec["decision"] = "stop"
            break
        rec["decision"] = "step"
    else:
        if run["trace"]:
            run["trace"][-1]["decision"] = "out_of_iterations"
    tmax = max((float(abs(v)) for v in t if _fin(v)), default=0.0)
    run["bound"] = (err + 16 * U) * (1.0 + tmax)
    run["R"], run["t"] = R, t
    run["untouched"] = untouched
    run["n_iter_done"] = iters
    run["A"] = A_last
    run["A_spread"], run["A_jmax"] = spread_last, jw_last
    run["ties"] = ties
    # culling at the final pose, and the two medians over the pre-culling set
    res = fr.residuals(R, t, jac=True)
    hp_out = np.asarray(has_point, np.uint8).copy()
    cull_open = np.zeros(N, bool)
    n_del, n_open = 0, 0
    thresh = mpf(fr.thresh)
    los_f, his_f = [], []
    for i, r in zip(fr.idx, res):
        en = mp.sqrt(r["e2"]) if not _isnan(r["e2"]) else NAN
        jn = max((float(abs(v)) for v in r["J"][0] + r["J"][1] if _fin(v)), default=0.0)
        de = r["de"] + jn * err
        de2 = 2 * float(en) * de + de * de if _fin(en) else 0.0
        los_f.append(r["e2"] - de2 if _fin(r["e2"]) else r["e2"])
        his_f.append(r["e2"] + de2 if _fin(r["e2"]) else r["e2"])
        if _isnan(en):
            continue
        if en > thresh:
            hp_out[i] = 0
            n_del += 1
        if _fin(en) and abs(float(en - thresh)) <= de and not (err == 0 and r["de"] == 0):
            cull_open[i] = True
            n_open += 1
    run["has_point"], run["cull_open"] = hp_out, cull_open
    run["num_obs"] = n - n_del
    run["num_obs_range"] = (n - n_del - n_open, n - n_del + n_open)
    k = n // 2
    fx64 = np.float64(fx)

    def med_interval(lo_vals, hi_vals):
        lo, hi = kth(lo_vals, k), kth(hi_vals, k)
        if _isnan(lo) or _isnan(hi):
            return (math.nan, math.nan) if _isnan(lo) and _isnan(hi) else (float(mp.sqrt(max(lo, 0)) * fx) if not _isnan(lo) else math.nan, math.nan)
        return (float(mp.sqrt(max(lo, 0))) * fx * (1 - 4 * U), float(mp.sqrt(max(hi, 0))) * fx * (1 + 4 * U))

    if e2_init is None:
        run["error_init"] = (0.0, 0.0)
    else:
        lo_i = [v - (2 * mp.sqrt(v) * r["de"] + r["de"] ** 2) if _fin(v) else v for v, r in zip(e2_init, fr.residuals(*cache["T0"], jac=False))]
        hi_i = [v + (2 * mp.sqrt(v) * r["de"] + r["de"] ** 2) if _fin(v) else v for v, r in zip(e2_init, fr.residuals(*cache["T0"], jac=False))]
        run["error_init"] = med_interval(lo_i, hi_i)
    run["error_final"] = med_interval(los_f, his_f)
    run["est_out"] = float(np.float64(est) * fx64)
    run["fx"] = float(fx64)
    return run


def branches(reproj_thresh, n_iter, fx, T_init, f, pos, level, has_point, max_forks=6, exact=False):
    """Every run the kernel may legitimately take: for each candidate of the MAD scale, the exact run and, at each
    near-tie decision, both of its branches (depth-first, at most max_forks forks per scale).  The exact run first."""
    cache = {}
    args = (reproj_thresh, n_iter, fx, T_init, f, pos, level, has_point)
    first = optimize(*args, cache=cache, exact=exact)
    runs = []
    for pick in range(1 if len(first.get("scale_cands", [0])) > 4 else len(first.get("scale_cands", [0]))):
        todo, mine = [dict()], []
        while todo:
            force = todo.pop()
            r = first if (pick == 0 and not force) else optimize(*args, force=force, scale_pick=pick, cache=cache, exact=exact)
            mine.append(r)
            for rec in r["trace"]:
                it = rec["it"]
                if rec["tie"] is None or it in force or len(mine) + len(todo) > max_forks:
                    continue
                if rec["tie"] in ("chi2", "chi2+eps"):
                    todo.append({**force, it: "accept" if rec["decision"] == "rollback" else "rollback"})
                if rec["tie"] in ("eps", "chi2+eps") and rec["decision"] in ("stop", "step", "out_of_iterations"):
                    todo.append({**force, it: "continue" if rec["decision"] == "stop" else "stop"})
        runs += mine
    return runs


def decisive(r) -> bool:
    """Every loop decision and every culling test decided beyond its uncertainty.  (A MAD scale with several float
    candidates is not a decision: `branches` runs each candidate, and each run is decisive or not on its own.)"""
    return all(rec["tie"] is None for rec in r["trace"]) and not r["cull_open"].any()


def pose_matrix(r):
    """The run's final [R | t] as doubles (the untouched start when no step was kept)."""
    return np.array([[float(v) for v in row] + [float(tv)] for row, tv in zip(r["R"], r["t"])])


def pose_error(T, r) -> float:
    T = np.asarray(T, np.float64).reshape(3, 4)
    ex = [abs(mpf(float(T[i, j])) - (r["R"][i][j] if j < 3 else r["t"][i])) for i in range(3) for j in range(4)]
    return float(max(ex))


def defined(r) -> bool:
    return math.isfinite(r["bound"]) and r["bound"] <= 1e-3


def cov_exact(r, fx):
    """(A fx^2)^-1 of the run's last A at working precision, or None when A is singular or not finite."""
    A = r["A"]
    if A is None or not all(_fin(v) for row in A for v in row):
        return None
    M = mp.matrix(A) * (mpf(fx) ** 2)
    try:
        return mp.inverse(M)
    except ZeroDivisionError:
        return None


def matches(g, r, fx):
    """(ok, error / bound, why) of the kernel's output dict g against the run r."""
    if r["empty"]:
        ok = (np.array_equal(np.asarray(g["T"]).view(np.int64), r["T_init"].view(np.int64)) and g["num_obs"] == 0
              and g["n_iter_done"] == 0 and g["estimated_scale"] == 0 and g["error_init"] == 0 and g["error_final"] == 0)
        return ok, 0.0, "empty"
    if g["n_iter_done"] != r["n_iter_done"]:
        return False, math.inf, "n_iter_done"
    est = float(g["estimated_scale"])
    cands = [float(np.float64(v) * np.float64(fx)) for v in r["scale_cands"]]
    if len(cands) > 1:  # rounding is monotone: every candidate lies between the set's ends
        ok = any(math.isnan(v) for v in cands) if math.isnan(est) else min(v for v in cands if not math.isnan(v)) <= est <= max(v for v in cands if not math.isnan(v))
    else:
        ok = est == r["est_out"] or (math.isnan(est) and math.isnan(r["est_out"]))
    if not ok:
        return False, math.inf, "estimated_scale"
    open_ = r["cull_open"]
    if not np.array_equal(np.asarray(g["has_point"])[~open_], r["has_point"][~open_]):
        return False, math.inf, "has_point"
    lo, hi = r["num_obs_range"]
    if not lo <= g["num_obs"] <= hi:
        return False, math.inf, "num_obs"
    for k in ("error_init", "error_final"):
        a, b = r[k]
        v = float(g[k])
        if math.isnan(a) or math.isnan(b):
            if not (math.isnan(v) or (not math.isnan(a) and v >= a)):
                return False, math.inf, k
        elif not a <= v <= b:
            return False, math.inf, k
    T = np.asarray(g["T"], np.float64)
    fin = np.array([[_fin(v) for v in row] + [_fin(tv)] for row, tv in zip(r["R"], r["t"])])
    if not np.array_equal(np.isfinite(T), fin):
        return False, math.inf, "finite"
    if not fin.all() or not defined(r) or any(not rec["cond"] < 1e12 for rec in r["trace"] if not _isnan(rec["dT"][0])):
        return True, 0.0, ""   # the step divided by a pivot that is rounding noise: no bound on the pose
    e = pose_error(T, r)
    ratio = e / r["bound"] if r["bound"] > 0 else (0.0 if e == 0 else math.inf)
    return ratio <= 1.0, ratio, "pose"


def cov_check(g, r, fx):
    """(ok, relative error / bound, checked) of the kernel's covariance against (A fx^2)^-1 of the run's last A.
    The bound: A's sums carry (n + 1) u relative, and a weight with several float candidates moves A by dw |J|^2; through
    the inverse that is cond(A) times A's relative error.  `checked` is False where no bound is defined: A singular or
    not finite, cond(A) > 1e12, or no bound on the pose A was formed at."""
    C = cov_exact(r, fx)
    cov = np.asarray(g["cov"], np.float64)
    if r["A"] is not None and all(v == 0 for row in r["A"] for v in row):
        return (not np.isfinite(cov).any()), 0.0, True      # a zero A: Gauss-Jordan divides by 0 everywhere
    if C is None or not defined(r):
        return True, 0.0, False
    top, bot = eig_range(r["A"])
    c = cond(r["A"])
    if not math.isfinite(c) or c > 1e12:
        return True, 0.0, False
    n = r["n"]
    # A is formed at the kernel's pose, within the bound of the exact one: each J moves by <= |J|^2 err (J ~ 1/z, its
    # derivative along the pose ~ 1/z^2), so A = sum w J J^T moves by <= 2 |J| err relative
    dA = (K * (n + 1) * U + 2 * K * r["A_jmax"] * r["bound"]) * top + sum(6 * dw * jn * jn for dw, jn, _ in r["A_spread"])
    cmax = max(abs(C[i, j]) for i in range(6) for j in range(6))
    err = max(abs(mpf(float(cov[i, j])) - C[i, j]) for i in range(6) for j in range(6))
    bound = c * dA / top * float(cmax) + 1e-300
    ratio = float(err) / bound
    return ratio <= 1.0, ratio, True


def match_any(g, runs, fx):
    ok, ratio, why = matches(g, runs[0], fx)
    if ok:
        return runs[0], ratio, why
    for r in runs[1:]:
        ok2, ratio2, _ = matches(g, r, fx)
        if ok2:
            return r, ratio2, ""
    return None, ratio, why


def assert_rank_deficient(g, r):
    """What a frame with a rank-deficient A pins: iteration 0's MAD scale and median, the culling flags and num_obs (its
    residuals stay at the observations' rounding noise whichever null-space step is taken)."""
    assert r["scale_cands"][0] * r["fx"] <= g["estimated_scale"] <= r["scale_cands"][-1] * r["fx"], g["estimated_scale"]
    a, b = r["error_init"]
    assert a <= g["error_init"] <= b, (g["error_init"], a, b)
    assert np.array_equal(np.asarray(g["has_point"]), r["has_point"]) and g["num_obs"] == r["num_obs"]
