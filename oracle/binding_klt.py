"""ctypes binding of the KLT oracle (oracle/libsvo_oracle_klt.so, built by oracle/klt.mk) and the reference wrappers around
OpenCV's own pyramidal Lucas-Kanade (`ref_klt_*`, the calls svo/src/initialization.cpp:127-169 makes) -- TEST
INFRASTRUCTURE ONLY.

Import this module only from tests/.  The product package (rpg_svo_b200) must never import it.  The `ref_klt_*` functions
need OpenCV's Python module (cv2); the tests replay their recorded outputs (tests/ref_golden.py) wherever it is absent."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.binding import MAX_LEVELS, _p

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libsvo_oracle_klt.so")
WIN = 30  # the reference's klt_win_size (initialization.cpp:136)
# how a point's tracking ended at a level (SVO_B200_KLT_* of include/svo_b200.h); -1 = level not run
CONVERGED, HALF_STEP, MAX_ITER, OUT_OF_BOUNDS, SMALL_EIG = 0, 1, 2, 3, 4


def build() -> str:
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "klt.mk"])
    return _LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_klt_track.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def level_sizes(w, h, max_level=4, win=WIN):
    """[(w, h)] of the LK pyramid's levels: buildOpticalFlowPyramid's level cut."""
    ws, hs = np.zeros(MAX_LEVELS, np.int32), np.zeros(MAX_LEVELS, np.int32)
    n = lib().orc_klt_levels(w, h, max_level, win, _p(ws), _p(hs))
    return [(int(ws[i]), int(hs[i])) for i in range(n)]


def pyramid(img, max_level=4, win=WIN):
    """The oracle's LK pyramid: dict(images=[h x w uint8], derivs=[h x w x 2 int16])."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    sizes = level_sizes(w, h, max_level, win)
    tot = sum(a * b for a, b in sizes)
    out, der = np.zeros(tot, np.uint8), np.zeros(tot * 2, np.int16)
    lib().orc_klt_pyramid(_p(img), w, h, max_level, win, _p(out), _p(der))
    images, derivs, o = [], [], 0
    for a, b in sizes:
        images.append(out[o:o + a * b].reshape(b, a))
        derivs.append(der[2 * o:2 * (o + a * b)].reshape(b, a, 2))
        o += a * b
    return dict(images=images, derivs=derivs)


def track(prev, nxt, prev_pts, next_pts, max_level=4, max_iter=30, eps=0.001, win=WIN):
    """calcOpticalFlowPyrLK restated.  dict(next_pts (N x 2 f32), status, reason, level_reason / iters (N x MAX_LEVELS),
    margins (N x MAX_LEVELS x 5: eps, half-step, eigenvalue, determinant, bounds; see orc_klt_track), n_levels)."""
    prev, nxt = np.ascontiguousarray(prev, np.uint8), np.ascontiguousarray(nxt, np.uint8)
    h, w = prev.shape
    p0 = np.ascontiguousarray(prev_pts, np.float32).reshape(-1, 2)
    p1 = np.ascontiguousarray(next_pts, np.float32).reshape(-1, 2).copy()
    n = len(p0)
    st = np.zeros(n, np.uint8)
    reason = np.zeros(n, np.int32)
    lr = np.zeros((n, MAX_LEVELS), np.int32)
    it = np.zeros((n, MAX_LEVELS), np.int32)
    mg = np.zeros((n, MAX_LEVELS, 5))
    nl = lib().orc_klt_track(_p(prev), _p(nxt), w, h, max_level, win, max_iter, eps, n, _p(p0), _p(p1), _p(st), _p(reason),
                             _p(lr), _p(it), _p(mg))
    return dict(next_pts=p1, status=st, reason=reason, level_reason=lr, iters=it, margins=mg, n_levels=nl)


# ---- the reference: OpenCV's calcOpticalFlowPyrLK as initialization.cpp calls it ----
def ref_klt_track(prev, nxt, prev_pts, next_pts, max_level=4, max_iter=30, eps=0.001):
    """cv::calcOpticalFlowPyrLK(prev, next, prev_pts, next_pts, status, err, Size(30, 30), max_level,
    TermCriteria(COUNT + EPS, max_iter, eps), OPTFLOW_USE_INITIAL_FLOW).  dict(next_pts (N x 2 f32), status (N uint8))."""
    import cv2

    p0 = np.ascontiguousarray(prev_pts, np.float32).reshape(-1, 1, 2)
    p1 = np.ascontiguousarray(next_pts, np.float32).reshape(-1, 1, 2).copy()
    if len(p0) == 0:
        return dict(next_pts=np.zeros((0, 2), np.float32), status=np.zeros(0, np.uint8))
    crit = (cv2.TERM_CRITERIA_COUNT | cv2.TERM_CRITERIA_EPS, int(max_iter), float(eps))
    p1, st, _ = cv2.calcOpticalFlowPyrLK(prev, nxt, p0, p1, winSize=(WIN, WIN), maxLevel=int(max_level), criteria=crit,
                                         flags=cv2.OPTFLOW_USE_INITIAL_FLOW)
    return dict(next_pts=p1.reshape(-1, 2).astype(np.float32), status=st.reshape(-1).astype(np.uint8))


def ref_klt_pyramid(img, max_level=4):
    """cv::buildOpticalFlowPyramid(img, pyr, Size(30, 30), max_level, true): dict(n_levels (its return value + 1),
    images, derivs (interleaved dx, dy int16))."""
    import cv2

    ret, pyr = cv2.buildOpticalFlowPyramid(np.ascontiguousarray(img, np.uint8), (WIN, WIN), int(max_level), withDerivatives=True)
    return dict(n_levels=int(ret) + 1, images=[np.ascontiguousarray(pyr[2 * i]) for i in range(ret + 1)],
                derivs=[np.ascontiguousarray(pyr[2 * i + 1]).astype(np.int16) for i in range(ret + 1)])
