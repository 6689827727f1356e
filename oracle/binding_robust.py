"""ctypes binding of the robust-cost oracle (oracle/libsvo_oracle_robust.so) and of the reference's own SparseImgAlign with
the robust cost set (oracle/_ref/libsvo_ref_robust.so) -- TEST INFRASTRUCTURE ONLY, built by oracle/robust.mk.

Import this module only from tests/.  The product package (rpg_svo_b200) must never import it."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.binding import MAX_LEVELS, SiaIter, _cam4, _level_ptrs, _p, c64, cam_struct

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libsvo_oracle_robust.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libsvo_ref_robust.so")


def build() -> str:
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "robust.mk"])
    return _LIB_PATH


def build_ref() -> str | None:
    """Only where the original project's sources are; elsewhere the tests replay its recorded outputs."""
    if os.path.isdir("/root/reference/svo/src"):
        subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "robust.mk", "ref"])
    return _REF_PATH if os.path.exists(_REF_PATH) else None


_lib = None
_ref_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_sparse_img_align_robust.restype = C.c_int64
    return _lib


def ref_lib():
    """CDLL of oracle/_ref/libsvo_ref_robust.so or None when it has not been built."""
    global _ref_lib
    if _ref_lib is None:
        if not os.path.exists(_REF_PATH):
            build_ref()
        if os.path.exists(_REF_PATH):
            _ref_lib = C.CDLL(_REF_PATH)
            _ref_lib.ref_sparse_img_align_robust.restype = C.c_longlong
    return _ref_lib


def sparse_img_align_robust(ref_pyr, cur_pyr, cam, T_init, px, f, pos, has_point, ref_pos, max_level, min_level,
                            weight, n_iter=30, eps=1e-6):
    """svo::SparseImgAlign::run restated with setRobustCostFunction(MADScale, weight) (weight: 0 unit, 2 Tukey, 3 Huber).
    Returns dict(T, n_tracked, visible, H, scales (MAX_LEVELS float32, NaN for the levels not run), trace)."""
    L = lib()
    n = int(px.shape[0])
    rp, cols, rows = _level_ptrs(ref_pyr)
    cp, _, _ = _level_ptrs(cur_pyr)
    T = c64(T_init).copy().reshape(12)
    visible = np.zeros(max(n, 1), dtype=np.uint8)
    H = np.zeros(36)
    scales = np.zeros(MAX_LEVELS, np.float32)
    cap = (max_level - min_level + 1) * max(n_iter, 1) + 8
    trace = (SiaIter * cap)()
    ntr = C.c_int(0)
    cs = cam_struct(cam)
    px, f, pos = c64(px), c64(f), c64(pos)
    hp = np.ascontiguousarray(has_point, dtype=np.uint8)
    ret = L.orc_sparse_img_align_robust(rp, cp, _p(cols), _p(rows), len(ref_pyr), C.byref(cs), _p(T), _p(px), _p(f), _p(pos),
                                        _p(hp), _p(c64(ref_pos)), n, max_level, min_level, n_iter, C.c_double(eps), int(weight),
                                        _p(visible), _p(H), _p(scales), trace, cap, C.byref(ntr))
    tr = [dict(level=r.level, iter=r.iter, accepted=r.accepted, n_meas=r.n_meas, chi2=r.chi2, x=np.array(r.x[:]),
               T=np.array(r.T[:]).reshape(3, 4)) for r in trace[:min(ntr.value, cap)]]
    return dict(T=T.reshape(3, 4), n_tracked=int(ret), visible=visible[:n], H=H.reshape(6, 6), scales=scales, trace=tr)


def ref_sparse_img_align_robust(ref_l0, cur_l0, n_levels, cam, T_ref_w, T_cur_w, px, f, pos, has_point, max_level, min_level,
                                weight, n_iter=30):
    """The compiled reference's SparseImgAlign(max, min, n_iter, GaussNewton, false, false) with the robust cost set
    (MADScale, weight: 0 unit, 2 Tukey, 3 Huber), run(ref, cur); pyramids by the reference's createImgPyramid.  `scales`
    (MAX_LEVELS float32, NaN for the levels not run): scale_ after each level's pre-call computeResiduals(model, false, true)."""
    h, w = ref_l0.shape
    T = c64(T_cur_w).copy().reshape(12)
    px, f, pos = c64(px), c64(f), c64(pos)
    hp = np.ascontiguousarray(has_point, np.uint8)
    n = len(hp)
    vis = np.zeros(max(n, 1), np.uint8)
    H = np.zeros(36)
    scales = np.zeros(MAX_LEVELS, np.float32)
    ret = ref_lib().ref_sparse_img_align_robust(_p(np.ascontiguousarray(ref_l0)), _p(np.ascontiguousarray(cur_l0)), w, h, n_levels,
                                                _p(_cam4(cam)), _p(c64(T_ref_w).reshape(12)), _p(T), _p(px), _p(f), _p(pos), _p(hp),
                                                n, max_level, min_level, n_iter, int(weight), _p(vis), _p(H), _p(scales))
    return dict(T_cur_w=T.reshape(3, 4), n_tracked=int(ret), visible=vis[:n], H=H.reshape(6, 6), scales=scales)
