"""A high-precision statement of Point::optimize (svo/src/point.cpp:119-177, with Point::jacobian_xyz2uv of
svo/include/svo/point.h:88-104) for the tests of point_optimize_kernel.

Every quantity is computed from the double inputs in mpmath at 40 significant digits, so against a double implementation
it is exact: the difference between the kernel and this reference is the kernel's rounding alone.  The iteration takes the
reference's decisions -- roll back and stop when `i > 0 && new_chi2 > chi2` or when dp[0] is NaN, stop after a step with
max|dp| <= EPS = 1e-10 -- and solves A dp = b by the symmetric-pivoting LDL^T that ldlt3_solve and Eigen's LDLT share
(largest remaining diagonal first, a pivot of exactly 0 leaves its column unscaled, the solve zeroes the component whose
|pivot| <= 1/DBL_MAX), here at working precision.  Non-finite values follow IEEE rules (x/0 = +-inf, 0/0 = NaN, every
comparison with NaN false), as they do in the kernel.

For each iteration the trace records the exact chi2, step, max|dp|, cond(A), the decision, and each decision's margin:
(new_chi2 - chi2) / chi2 against the roll-back test and (max|dp| - EPS) / EPS against the stop test.

Bound on the kernel's position.  Iteration i forms A and b as serial double sums over the point's n observations and
solves a 3x3 system; the kernel then adds the step to the position.  The sums have a relative backward error of at most
gamma_n ~ n u (u = 2^-53, recursive summation) and each term carries a few roundings of its own: the residual
e = project2d(f) - project2d(T p) is known to ~u |project2d| absolutely, which through A^-1 J^T moves the step by
~cond(A) u z ~ cond(A) u s, with s = |pos| + max |t_f_w| the scale of the point's coordinates in its observing frames; the
LDL^T solve is backward stable, moving the step by ~cond(A) u |dp_i|.  Gauss-Newton forgets an error in the position it
starts an iteration from (the next step corrects it, up to second order), so the per-iteration errors add:

    |pos_kernel - pos_exact| <= K u sum_i cond(A_i) (n + 1) (s + |dp_i|)

K = 8 covers the constant factors of the terms above (3 coordinates per row of R p + t, two quotients per residual, the
two normal-equation terms per observation) with a factor ~2 to spare.  It is tight where it matters: on a well-conditioned
two-view point 3 m away (cond ~1e2, n = 2) it is ~1e-12 m, five orders below the 1e-7 m a wrong sum or sign produces.

A decision is decisive when its margin exceeds TIE_REL = 1e-9 relative and the kernel's own uncertainty in the compared
quantities: the bound above for max|dp| against EPS, and for chi2 the residual uncertainty
de = K u (1 + max |project2d|) + |J| |pos error| propagated into sum |e|^2.  Near a tie either branch is legitimate:
`branches` follows both and returns every final position the kernel may end at, each with its own bound.
"""
from __future__ import annotations

import math

import numpy as np
from mpmath import mp, mpf

mp.dps = 40

U = 2.0 ** -53
K = 8.0
TIE_REL = 1e-9
EPS = mpf(0.0000000001)                      # the double constant EPS of global.h:77
TINY = mpf(1.0 / 1.7976931348623157e308)     # Eigen's 1 / NumTraits<double>::highest()
NAN, INF = mpf("nan"), mpf("inf")


def _div(a, b):
    """a / b with IEEE semantics for b == 0 (mpmath raises there).  mpmath has no -0: a zero divisor counts as +0."""
    if b == 0:
        if a == 0 or mp.isnan(a):
            return NAN
        return INF if a > 0 else -INF
    return a / b


def _isnan(x) -> bool:
    return bool(mp.isnan(x))


def jacobian_xyz2uv(p, R):
    """Point::jacobian_xyz2uv: J = -[[z^-1, 0, -x z^-2], [0, z^-1, -y z^-2]] R."""
    z_inv = _div(mpf(1), p[2])
    z_inv_sq = z_inv * z_inv
    pj = ((z_inv, mpf(0), -p[0] * z_inv_sq), (mpf(0), z_inv, -p[1] * z_inv_sq))
    return [[-(pj[r][0] * R[0][c] + pj[r][1] * R[1][c] + pj[r][2] * R[2][c]) for c in range(3)] for r in range(2)]


def ldlt3_solve(A, b):
    """The symmetric-pivoting LDL^T solve of ldlt3_solve / Eigen::LDLT at working precision.  Returns (x, pivots)."""
    A = [row[:] for row in A]
    tr = [0, 1, 2]
    for k in range(3):
        big, bigv = k, abs(A[k][k])
        for i in range(k + 1, 3):
            if abs(A[i][i]) > bigv:
                bigv, big = abs(A[i][i]), i
        tr[k] = big
        if big != k:
            for j in range(k):
                A[k][j], A[big][j] = A[big][j], A[k][j]
            for i in range(big + 1, 3):
                A[i][k], A[i][big] = A[i][big], A[i][k]
            A[k][k], A[big][big] = A[big][big], A[k][k]
            for i in range(k + 1, big):
                A[i][k], A[big][i] = A[big][i], A[i][k]
        if k > 0:
            temp = [A[j][j] * A[k][j] for j in range(k)]
            acc = mpf(0)
            for j in range(k):
                acc += A[k][j] * temp[j]
            A[k][k] -= acc
            for i in range(k + 1, 3):
                a2 = mpf(0)
                for j in range(k):
                    a2 += A[i][j] * temp[j]
                A[i][k] -= a2
        akk = A[k][k]
        ok = abs(akk) > 0
        if k == 0 and not ok:
            tr = [0, 1, 2]
            break
        if ok:
            for i in range(k + 1, 3):
                A[i][k] = A[i][k] / akk
    x = list(b)
    for i in range(3):
        j = tr[i]
        x[i], x[j] = x[j], x[i]
    for i in range(1, 3):
        for j in range(i):
            x[i] -= A[i][j] * x[j]
    for i in range(3):
        x[i] = x[i] / A[i][i] if abs(A[i][i]) > TINY else mpf(0)
    for i in (1, 0):
        for j in range(i + 1, 3):
            x[i] -= A[j][i] * x[j]
    for i in (2, 1, 0):
        j = tr[i]
        x[i], x[j] = x[j], x[i]
    return x, [A[i][i] for i in range(3)]


def normal_system(pos, Ts, fs):
    """A, b, chi2 of one iteration at pos, plus max |project2d| and max |J| (for the residual uncertainty)."""
    A = [[mpf(0)] * 3 for _ in range(3)]
    b = [mpf(0)] * 3
    chi2 = mpf(0)
    max_proj, max_j = mpf(0), mpf(0)
    for T, f in zip(Ts, fs):
        R = (T[0:3], T[4:7], T[8:11])
        p = [R[r][0] * pos[0] + R[r][1] * pos[1] + R[r][2] * pos[2] + T[4 * r + 3] for r in range(3)]
        J = jacobian_xyz2uv(p, R)
        ox, oy = _div(f[0], f[2]), _div(f[1], f[2])
        px, py = _div(p[0], p[2]), _div(p[1], p[2])
        ex, ey = ox - px, oy - py
        chi2 += ex * ex + ey * ey
        for r in range(3):
            for c in range(3):
                A[r][c] += J[0][r] * J[0][c] + J[1][r] * J[1][c]
            b[r] -= J[0][r] * ex + J[1][r] * ey
        max_proj = max(max_proj, abs(ox), abs(oy), abs(px), abs(py))
        max_j = max(max_j, *(abs(v) for row in J for v in row))
    return A, b, chi2, max_proj, max_j


def cond(A) -> float:
    """2-norm condition number of the symmetric A (inf when singular, NaN when A is not finite).  Eigenvalues below
    1e-35 of the largest are 40-digit rounding of an exact zero: a component the solve zeroes, left out."""
    if any(not mp.isfinite(v) for row in A for v in row):
        return math.nan
    ev = [abs(e) for e in mp.eigsy(mp.matrix(A), eigvals_only=True)]
    top = max(ev)
    if top == 0:
        return 1.0
    live = [e for e in ev if e > top * mpf("1e-35")]
    return float(top / min(live))


def _mp(v):
    return [mpf(float(x)) for x in v]


def optimize(n_iter, pos, Ts, fs, force=None, cache=None):
    """Point::optimize at working precision.  Ts: the observing poses (each 12 doubles, [R | t] row-major), fs: the
    bearings.  `force` maps an iteration to the branch to take there regardless of the exact comparison ("rollback" or
    "accept" at the chi2 test, "stop" or "continue" at the EPS test).  Returns the final position (mpf), its bound, and
    the trace (one dict per iteration)."""
    force = force or {}
    cache = {} if cache is None else cache  # shared by the runs of `branches`: inputs and normal systems by position
    if "Ts" not in cache:
        cache["Ts"], cache["fs"], cache["ns"] = [_mp(T) for T in Ts], [_mp(f) for f in fs], {}
    Ts, fs = cache["Ts"], cache["fs"]
    n = len(Ts)
    start_f = np.array(pos, np.float64).reshape(3)  # the start's own bits (mpmath turns every NaN into -NaN)
    pos = _mp(pos)
    start = pos
    s = float(max(abs(v) for v in pos) if all(mp.isfinite(v) for v in pos) else math.inf)
    s += max((float(abs(v)) for T in Ts for v in (T[3], T[7], T[11]) if mp.isfinite(v)), default=0.0)
    old_point = pos
    chi2, chi2_unc = mpf(0), 0.0
    err = 0.0         # bound on the kernel's distance from the exact position reached so far
    err_old = 0.0
    trace = []
    for i in range(n_iter):
        key = tuple(pos)
        if key not in cache["ns"]:
            A, b, new_chi2, max_proj, max_j = normal_system(pos, Ts, fs)
            cache["ns"][key] = (A, b, new_chi2, max_proj, max_j, ldlt3_solve(A, b), cond(A))
        A, b, new_chi2, max_proj, max_j, (dp, piv), c = cache["ns"][key]
        max_dp = max(abs(dp[0]), abs(dp[1]), abs(dp[2])) if not any(_isnan(v) for v in dp) else NAN
        de = K * U * (1.0 + float(max_proj)) + float(max_j) * err
        new_unc = (2.0 * math.sqrt(n * abs(float(new_chi2))) * de + n * de * de + K * n * U * abs(float(new_chi2))
                   if mp.isfinite(new_chi2) else math.inf)
        step = float(mp.sqrt(dp[0] ** 2 + dp[1] ** 2 + dp[2] ** 2)) if not _isnan(max_dp) else math.nan
        term = K * U * c * (n + 1) * (s + step)
        rec = dict(it=i, chi2=chi2, new_chi2=new_chi2, dp=dp, max_dp=max_dp, cond=c, pivots=piv, n=n, tie=None)
        trace.append(rec)
        nan_step = _isnan(dp[0])
        if i > 0 and not nan_step:
            margin = float(abs(_div(new_chi2 - chi2, chi2))) if chi2 != 0 else (math.inf if new_chi2 != 0 else 0.0)
            rec["chi2_margin"] = margin
            unc = new_unc + chi2_unc
            tie = not (abs(float(new_chi2 - chi2)) > TIE_REL * abs(float(chi2)) + unc) or not math.isfinite(unc)
            increased = new_chi2 > chi2
            if tie:
                rec["tie"] = "chi2"
            if i in force and force[i] in ("rollback", "accept"):
                increased = force[i] == "rollback"
        else:
            increased = False
        if (i > 0 and increased) or nan_step:
            rec["decision"] = "nan" if nan_step and not (i > 0 and increased) else "rollback"
            pos = old_point
            err = err_old
            break
        new_point = [pos[k] + dp[k] for k in range(3)]
        old_point, err_old = pos, err
        pos = new_point
        err = err + term
        chi2, chi2_unc = new_chi2, new_unc
        eps_margin = float(_div(max_dp - EPS, EPS))
        rec["eps_margin"] = eps_margin
        d_unc = term + err_old
        if not (abs(float(max_dp - EPS)) > TIE_REL * float(EPS) + d_unc):
            rec["tie"] = rec["tie"] or "eps"
            if rec["tie"] == "chi2":
                rec["tie"] = "chi2+eps"
        stop = max_dp <= EPS
        if i in force and force[i] in ("stop", "continue"):
            stop = force[i] == "stop"
        if stop:
            rec["decision"] = "stop"
            break
        rec["decision"] = "step"
    else:
        if trace:
            trace[-1]["decision"] = "out_of_iterations"
    final_err = err + 2 * U * float(max((abs(v) for v in pos), default=0)) if all(mp.isfinite(v) for v in pos) else math.nan
    return dict(pos=pos, start=start_f, untouched=pos is start, bound=final_err, trace=trace, scale=s)


def branches(n_iter, pos, Ts, fs, max_forks=6):
    """Every run of `optimize` the kernel may legitimately take: the exact run and, at each near-tie decision, both of
    its branches (depth-first, at most max_forks forks).  Returns the list of runs, the exact one first."""
    runs, todo, cache = [], [dict()], {}
    while todo:
        force = todo.pop()
        r = optimize(n_iter, pos, Ts, fs, force, cache)
        r["force"] = force
        runs.append(r)
        for rec in r["trace"]:
            it = rec["it"]
            if rec["tie"] is None or it in force or len(runs) + len(todo) > max_forks:
                continue
            if rec["tie"] in ("chi2", "chi2+eps"):
                other = "accept" if rec["decision"] in ("rollback",) else "rollback"
                todo.append({**force, it: other})
            if rec["tie"] in ("eps", "chi2+eps") and rec["decision"] in ("stop", "step", "out_of_iterations"):
                todo.append({**force, it: "continue" if rec["decision"] == "stop" else "stop"})
    return runs


def error(g, r) -> float:
    """max |g - exact| over the coordinates (g: the kernel's double result)."""
    return float(max(abs(mpf(float(x)) - y) for x, y in zip(g, r["pos"])))


def decisive(r) -> bool:
    return all(rec["tie"] is None for rec in r["trace"])


def defined(r) -> bool:
    """The bound says something: finite and below 1e-3 of the final position's size (past that the step divided by a
    pivot that is rounding noise, and any finite result is as good as another)."""
    size = max((abs(float(v)) for v in r["pos"]), default=0.0)
    return math.isfinite(r["bound"]) and r["bound"] <= 1e-3 * max(1.0, size)


def matches(g, r):
    """(ok, error / bound) of the double result g against the run r: a run that ends at its untouched start (no step
    taken, or every step rolled back) must be returned bit for bit; any other must agree on which coordinates are
    finite and, where its bound is defined, lie within it."""
    g = [float(x) for x in g]
    if r["untouched"]:
        return np.array_equal(np.array(g).view(np.int64), r["start"].view(np.int64)), 0.0
    fin = [bool(mp.isfinite(v)) for v in r["pos"]]
    if [math.isfinite(x) for x in g] != fin:
        return False, math.inf
    if not all(fin) or not math.isfinite(r["bound"]):
        return True, 0.0
    e = error(g, r)
    ratio = e / r["bound"] if r["bound"] > 0 else (0.0 if e == 0 else math.inf)
    return ratio <= 1.0, ratio


def match_any(g, runs):
    """The run of `branches` the kernel's result g matches (the exact one when it does), with its error / bound ratio;
    (None, ratio against the exact run) when it matches none."""
    ok, ratio = matches(g, runs[0])
    if ok:
        return runs[0], ratio
    for r in runs[1:]:
        ok2, ratio2 = matches(g, r)
        if ok2:
            return r, ratio2
    return None, ratio


def as_float(r):
    return [float(v) for v in r["pos"]]
