"""ctypes binding of the epipolar-options oracle (oracle/libsvo_oracle_epipolar.so) and of the reference's own Matcher and
DepthFilter with Matcher::options_ set (oracle/_ref/libsvo_ref_epipolar.so) -- TEST INFRASTRUCTURE ONLY, built by
oracle/epipolar.mk.

`opt` everywhere is a dict with the keys of svo_b200_epipolar_options' Python form (align_1d, subpix_refinement,
edgelet_filtering, edgelet_max_angle); missing keys take the reference's defaults.

Import this module only from tests/.  The product package (rpg_svo_b200) must never import it."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle.binding import EpiResult, RefMatchOut, _cam4, _level_ptrs, _p, c64, cam_struct

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libsvo_oracle_epipolar.so")
_REF_PATH = os.path.join(_HERE, "_ref", "libsvo_ref_epipolar.so")

DEFAULTS = dict(align_1d=False, subpix_refinement=True, edgelet_filtering=True, edgelet_max_angle=0.7)


class EpiOptions(C.Structure):  # svo_b200_epipolar_options
    _fields_ = [("align_1d", C.c_int), ("subpix_refinement", C.c_int), ("epi_search_edgelet_filtering", C.c_int),
                ("epi_search_edgelet_max_angle", C.c_double)]


def options(opt=None) -> EpiOptions:
    o = dict(DEFAULTS, **(opt or {}))
    return EpiOptions(int(o["align_1d"]), int(o["subpix_refinement"]), int(o["edgelet_filtering"]), float(o["edgelet_max_angle"]))


def build() -> str:
    subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "epipolar.mk"])
    return _LIB_PATH


def build_ref() -> str | None:
    """Only where the original project's sources are; elsewhere the tests replay its recorded outputs."""
    if os.path.isdir("/root/reference/svo/src"):
        subprocess.check_call(["make", "-s", "-C", _HERE, "-f", "epipolar.mk", "ref"])
    return _REF_PATH if os.path.exists(_REF_PATH) else None


_lib = None
_ref_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
    return _lib


def ref_lib():
    """CDLL of oracle/_ref/libsvo_ref_epipolar.so or None when it has not been built."""
    global _ref_lib
    if _ref_lib is None:
        if not os.path.exists(_REF_PATH):
            build_ref()
        if os.path.exists(_REF_PATH):
            _ref_lib = C.CDLL(_REF_PATH)
    return _ref_lib


def find_epipolar_match_direct(ref_pyr, cur_pyr, cam, T_cur_ref, ref_px, ref_f, ref_level, ftr_type, ref_grad, d_est, d_min,
                               d_max, max_search_level, align_max_iter=10, max_epi_search_steps=1000, opt=None):
    """oracle.binding.find_epipolar_match_direct under Matcher::Options `opt`, plus ran_1d (align1D ran and set h_inv)."""
    rp, cols, rows = _level_ptrs(ref_pyr)
    cp, _, _ = _level_ptrs(cur_pyr)
    out = EpiResult()
    ran = C.c_int(0)
    cs = cam_struct(cam)
    eo = options(opt)
    lib().orc_find_epipolar_match_direct_opt(rp, cp, _p(cols), _p(rows), len(ref_pyr), C.byref(cs), _p(c64(T_cur_ref).reshape(12)),
                                             _p(c64(ref_px)), _p(c64(ref_f)), int(ref_level), int(ftr_type), _p(c64(ref_grad)),
                                             C.c_double(d_est), C.c_double(d_min), C.c_double(d_max), int(max_search_level),
                                             int(align_max_iter), int(max_epi_search_steps), C.byref(eo), C.byref(out),
                                             C.byref(ran))
    return dict(success=bool(out.success), reject=bool(out.reject), search_level=out.search_level, n_zmssd=out.n_zmssd_evals,
                epi_length=out.epi_length, px_cur=np.array(out.px_cur[:]), depth=out.depth, h_inv=out.h_inv,
                ran_1d=bool(ran.value), A_cur_ref=np.array(out.A_cur_ref[:]).reshape(2, 2))


def depth_filter_update(ref_pyrs, ref_T_f_w, cur_pyr, cur_T_f_w, cam, ref_index, ftr_px, ftr_f, ftr_level, ftr_type, ftr_grad,
                        batch_id, batch_counter, seeds, max_n_kfs=3, sigma2_thresh=200.0, max_search_level=2, align_max_iter=10,
                        max_epi_search_steps=1000, opt=None):
    """oracle.binding.depth_filter_update with DepthFilter::matcher_.options_ = `opt`."""
    n_ref = len(ref_pyrs)
    nl = len(cur_pyr)
    flat = (C.c_void_p * (n_ref * nl))()
    for r, pyr in enumerate(ref_pyrs):
        for lv, im in enumerate(pyr):
            flat[r * nl + lv] = im.ctypes.data
    cp, cols, rows = _level_ptrs(cur_pyr)
    M = len(ref_index)
    out = {k: np.ascontiguousarray(seeds[k], np.float32).copy() for k in ("a", "b", "mu", "z_range", "sigma2")}
    status = np.zeros(M, np.uint8)
    pxc, z, nz = np.zeros((M, 2)), np.zeros(M), np.zeros(M, np.int32)
    cs = cam_struct(cam)
    eo = options(opt)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    refT = c64(np.asarray(ref_T_f_w)).reshape(-1)
    ri, fl, ft, bi = i32(ref_index), i32(ftr_level), i32(ftr_type), i32(batch_id)
    fpx, ff, fg = c64(ftr_px), c64(ftr_f), c64(ftr_grad)
    lib().orc_depth_filter_update_opt(flat, _p(refT), n_ref, cp, _p(c64(cur_T_f_w).reshape(12)), _p(cols), _p(rows), nl,
                                      C.byref(cs), M, _p(ri), _p(fpx), _p(ff), _p(fl), _p(ft), _p(fg), _p(bi), int(batch_counter),
                                      int(max_n_kfs), C.c_double(sigma2_thresh), int(max_search_level), int(align_max_iter),
                                      int(max_epi_search_steps), C.byref(eo), _p(out["a"]), _p(out["b"]), _p(out["mu"]),
                                      _p(out["z_range"]), _p(out["sigma2"]), _p(status), _p(pxc), _p(z), _p(nz))
    out.update(status=status, px_cur=pxc, z=z, n_zmssd=nz)
    return out


def ref_matcher_epipolar(ref_l0, cur_l0, n_levels, cam, T_ref_w, T_cur_w, ref_px, ref_f, ref_level, ftr_type, ref_grad, d_est,
                         d_min, d_max, opt=None, n_pyr_levels=3):
    """The compiled reference's Matcher::findEpipolarMatchDirect(ref, cur, ftr, d_est, d_min, d_max) with options_ = `opt`
    on a fresh Matcher; ran_1d: align1D ran (h_inv is the h_inv_ it set, 0 otherwise)."""
    h, w = ref_l0.shape
    out = RefMatchOut()
    ran = C.c_int(0)
    eo = options(opt)
    ref_lib().ref_matcher_epipolar(_p(np.ascontiguousarray(ref_l0)), _p(np.ascontiguousarray(cur_l0)), w, h, n_levels,
                                   _p(_cam4(cam)), _p(c64(T_ref_w).reshape(12)), _p(c64(T_cur_w).reshape(12)), _p(c64(ref_px)),
                                   _p(c64(ref_f)), int(ref_level), int(ftr_type), _p(c64(ref_grad)), C.c_double(d_est),
                                   C.c_double(d_min), C.c_double(d_max), int(n_pyr_levels), C.byref(eo), C.byref(out),
                                   C.byref(ran))
    return dict(success=bool(out.success), search_level=out.search_level, reject=bool(out.reject),
                px_cur=np.array(out.px_cur[:]), A_cur_ref=np.array(out.A[:]).reshape(2, 2), h_inv=out.h_inv,
                ran_1d=bool(ran.value), epi_length=out.epi_length, depth=out.depth)


def ref_depth_filter_update_epipolar(ref_l0s, ref_T_f_w, cur_l0, cur_T_f_w, n_levels, cam, ref_index, ftr_px, ftr_f, ftr_level,
                                     ftr_type, ftr_grad, batch_id, batch_counter, seeds, opt=None, n_pyr_levels=3):
    """The compiled reference's DepthFilter::updateSeeds with matcher_.options_ = `opt`.  status: 0 kept, 1 converged,
    2 erased."""
    imgs = np.ascontiguousarray(np.stack(ref_l0s))
    h, w = cur_l0.shape
    M = len(ref_index)
    out = {k: np.ascontiguousarray(seeds[k], np.float32).copy() for k in ("a", "b", "mu", "z_range", "sigma2")}
    status = np.zeros(M, np.uint8)
    xyz = np.zeros((M, 3))
    eo = options(opt)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    ref_lib().ref_depth_filter_update_epipolar(_p(imgs), _p(c64(np.asarray(ref_T_f_w)).reshape(-1)), len(ref_l0s),
                                               _p(np.ascontiguousarray(cur_l0)), _p(c64(cur_T_f_w).reshape(12)), w, h, n_levels,
                                               _p(_cam4(cam)), M, _p(i32(ref_index)), _p(c64(ftr_px)), _p(c64(ftr_f)),
                                               _p(i32(ftr_level)), _p(i32(ftr_type)), _p(c64(ftr_grad)), _p(i32(batch_id)),
                                               int(batch_counter), int(n_pyr_levels), C.byref(eo), _p(out["a"]), _p(out["b"]),
                                               _p(out["mu"]), _p(out["z_range"]), _p(out["sigma2"]), _p(status), _p(xyz))
    out.update(status=status, xyz_world=xyz)
    return out
