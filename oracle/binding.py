"""ctypes binding of the CPU oracle (oracle/libsvo_oracle.so) -- TEST INFRASTRUCTURE ONLY.

Import this module only from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs.  The product package (rpg_svo_b200) must never import it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libsvo_oracle.so")
MAX_LEVELS = 8


def build_ref() -> str | None:
    """oracle/_ref: the reference's own hot-path sources (feature_alignment, sparse_img_align, matcher,
    pose_optimizer, point, frame, config .cpp) compiled where they lie against oracle/shim (only where
    /root/reference exists; the GPU box uses the prebuilt .so that travels with the snapshot)."""
    out = os.path.join(_HERE, "_ref", "libsvo_ref.so")
    if os.path.isdir("/root/reference/svo/src"):
        subprocess.check_call(["make", "-s", "-C", _HERE, "ref"])
    return out if os.path.exists(out) else None


def build(force: bool = False) -> str:
    srcs = ["svo_oracle.cpp", "svo_oracle_align.inc", "svo_oracle_depth.inc", "svo_oracle_pose.inc", "svo_oracle_reproject.inc", "svo_oracle_detect.inc", "fast_ext.h",
            "oracle_math.h", "svo_oracle.h", "Makefile"]
    stale = force or not os.path.exists(_LIB_PATH) or any(
        os.path.getmtime(os.path.join(_HERE, s)) > os.path.getmtime(_LIB_PATH) for s in srcs)
    if stale:
        subprocess.check_call(["make", "-s", "-C", _HERE] + (["-B"] if force else []))
    return _LIB_PATH


class Camera(C.Structure):
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("width", C.c_int), ("height", C.c_int), ("model", C.c_int), ("reserved_", C.c_int), ("d", C.c_double * 5)]


class SiaIter(C.Structure):
    _fields_ = [("level", C.c_int), ("iter", C.c_int), ("accepted", C.c_int), ("n_meas", C.c_int),
                ("chi2", C.c_double), ("x", C.c_double * 6), ("T", C.c_double * 12)]


class MatchResult(C.Structure):
    _fields_ = [("success", C.c_int), ("search_level", C.c_int), ("px_cur", C.c_double * 2),
                ("A_cur_ref", C.c_double * 4), ("h_inv", C.c_double)]


class EpiResult(C.Structure):
    _fields_ = [("success", C.c_int), ("reject", C.c_int), ("search_level", C.c_int),
                ("n_zmssd_evals", C.c_int), ("n_align_iter", C.c_int), ("epi_length", C.c_double),
                ("px_cur", C.c_double * 2), ("depth", C.c_double), ("h_inv", C.c_double),
                ("A_cur_ref", C.c_double * 4)]


class PoseOptResult(C.Structure):
    _fields_ = [("estimated_scale", C.c_double), ("error_init", C.c_double),
                ("error_final", C.c_double), ("num_obs", C.c_int64), ("n_iter_done", C.c_int),
                ("cov", C.c_double * 36)]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_sparse_img_align_run.restype = C.c_int64
        _lib.orc_sparse_img_align_batch.restype = None
        _lib.orc_compute_tau.restype = C.c_double
        _lib.orc_compute_tau.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double]
        _lib.orc_update_seed.argtypes = [C.c_float, C.c_float] + [C.c_void_p] * 5
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def cam_struct(cam) -> Camera:
    d = (C.c_double * 5)(*([float(x) for x in getattr(cam, "d", ())] + [0.0] * 5)[:5])
    return Camera(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height, int(getattr(cam, "model", 0)), 0, d)


def _level_ptrs(pyr, n=None):
    arr = (C.c_void_p * (len(pyr) if n is None else n))()  # entries past the pyramid's depth stay NULL
    for i, im in enumerate(pyr):
        assert im.dtype == np.uint8 and im.flags.c_contiguous
        arr[i] = im.ctypes.data
    cols = np.array([im.shape[1] for im in pyr], dtype=np.int32)
    rows = np.array([im.shape[0] for im in pyr], dtype=np.int32)
    return arr, cols, rows


def c64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def sparse_img_align(ref_pyr, cur_pyr, cam, T_init, px, f, pos, has_point, ref_pos, max_level,
                     min_level, n_iter=30, eps=1e-6, want_trace=True):
    """svo::SparseImgAlign::run restated.  Returns dict(T, n_tracked, visible, H, residuals, trace)."""
    L = lib()
    n = int(px.shape[0])
    rp, cols, rows = _level_ptrs(ref_pyr)
    cp, _, _ = _level_ptrs(cur_pyr)
    T = c64(T_init).copy().reshape(12)
    visible = np.zeros(max(n, 1), dtype=np.uint8)
    H = np.zeros(36)
    res = np.zeros((max(n, 1), 16), dtype=np.float32)
    # a negative n_iter is the reference's size_t n_iter_ wrapped around: no limit (room for 100 per level)
    cap = (max_level - min_level + 1) * (max(n_iter, 1) if n_iter >= 0 else 100) + 8
    trace = (SiaIter * cap)()
    ntr = C.c_int(0)
    cs = cam_struct(cam)
    px, f, pos = c64(px), c64(f), c64(pos)
    hp = np.ascontiguousarray(has_point, dtype=np.uint8)
    rpos = c64(ref_pos)
    ret = L.orc_sparse_img_align_run(rp, cp, _p(cols), _p(rows), len(ref_pyr), C.byref(cs), _p(T),
                                     _p(px), _p(f), _p(pos), _p(hp), _p(rpos), n, max_level,
                                     min_level, n_iter, C.c_double(eps), _p(visible), _p(H), _p(res),
                                     trace if want_trace else None, cap, C.byref(ntr))
    tr = []
    if want_trace:
        for k in range(min(ntr.value, cap)):
            r = trace[k]
            tr.append(dict(level=r.level, iter=r.iter, accepted=r.accepted, n_meas=r.n_meas,
                           chi2=r.chi2, x=np.array(r.x[:]), T=np.array(r.T[:]).reshape(3, 4)))
    return dict(T=T.reshape(3, 4), n_tracked=int(ret), visible=visible[:n], H=H.reshape(6, 6),
                residuals=res[:n], trace=tr)


def sparse_img_align_batch(ref_pyrs, cur_pyrs, cam, T_init, feat_offset, px, f, pos, has_point, ref_pos,
                           max_level, min_level, n_iter=30, eps=1e-6, n_threads=1):
    """B independent runs on n_threads host threads (no Python in the loop).  Returns (T [B,3,4], n_tracked [B])."""
    L = lib()
    B = len(ref_pyrs)
    nl = len(ref_pyrs[0])
    rp = (C.c_void_p * (B * nl))()
    cp = (C.c_void_p * (B * nl))()
    for b in range(B):
        for l in range(nl):
            rp[b * nl + l] = ref_pyrs[b][l].ctypes.data
            cp[b * nl + l] = cur_pyrs[b][l].ctypes.data
    cols = np.array([im.shape[1] for im in ref_pyrs[0]], dtype=np.int32)
    rows = np.array([im.shape[0] for im in ref_pyrs[0]], dtype=np.int32)
    T = c64(T_init).copy().reshape(B, 12)
    fo = np.ascontiguousarray(feat_offset, np.int32)
    px, f, pos, rpos = c64(px), c64(f), c64(pos), c64(ref_pos)
    hp = np.ascontiguousarray(has_point, np.uint8)
    ntr = np.zeros(B, np.int64)
    cs = cam_struct(cam)
    L.orc_sparse_img_align_batch(B, rp, cp, _p(cols), _p(rows), nl, C.byref(cs), _p(T), _p(fo), _p(px), _p(f),
                                 _p(pos), _p(hp), _p(rpos), max_level, min_level, n_iter, C.c_double(eps),
                                 _p(ntr), int(n_threads))
    return T.reshape(B, 3, 4), ntr


def sparse_residuals(ref_img, cur_img, level, cam, T, px, f, pos, has_point, ref_pos, visible_in=None):
    L = lib()
    n = int(px.shape[0])
    rows, cols = ref_img.shape
    vis = np.zeros(n, dtype=np.uint8) if visible_in is None else np.ascontiguousarray(visible_in, np.uint8).copy()
    ref_patch = np.zeros((n, 16), np.float32)
    jac = np.zeros((n, 16, 6))
    res = np.zeros((n, 16), np.float32)
    inimg = np.zeros(n, np.uint8)
    H = np.zeros(36)
    Jres = np.zeros(6)
    chi2 = C.c_double(0)
    nm = C.c_int64(0)
    cs = cam_struct(cam)
    px, f, pos = c64(px), c64(f), c64(pos)
    hp = np.ascontiguousarray(has_point, dtype=np.uint8)
    T = c64(T).reshape(12)
    rpos = c64(ref_pos)
    L.orc_sparse_residuals(_p(ref_img), _p(cur_img), cols, rows, level, C.byref(cs), _p(T), _p(px),
                           _p(f), _p(pos), _p(hp), _p(rpos), n, _p(vis), _p(ref_patch), _p(jac),
                           _p(res), _p(inimg), _p(H), _p(Jres), C.byref(chi2), C.byref(nm))
    return dict(visible=vis, ref_patch=ref_patch, jac=jac, residuals=res, in_image=inimg,
                H=H.reshape(6, 6), Jres=Jres, chi2=chi2.value, n_meas=nm.value)


def camera_world2cam(cam, xyz):
    xyz = c64(xyz).reshape(-1, 3)
    out = np.zeros((len(xyz), 2))
    cs = cam_struct(cam)
    lib().orc_camera_world2cam(C.byref(cs), _p(xyz), len(xyz), _p(out))
    return out


def camera_cam2world(cam, px):
    px = c64(px).reshape(-1, 2)
    out = np.zeros((len(px), 3))
    cs = cam_struct(cam)
    lib().orc_camera_cam2world(C.byref(cs), _p(px), len(px), _p(out))
    return out


PYR_SCALAR, PYR_X86 = 0, 1


def half_sample(img, rule=PYR_X86):
    """[EXT] vk::halfSample: rule PYR_X86 = the reference's x86 build (SSE2 branch for widths % 16 == 0), PYR_SCALAR."""
    out = np.zeros((img.shape[0] // 2, img.shape[1] // 2), np.uint8)
    lib().orc_half_sample_rule(_p(np.ascontiguousarray(img)), img.shape[1], img.shape[0], _p(out), int(rule))
    return out


def se3_exp(x):
    T = np.zeros(12)
    lib().orc_se3_exp(_p(c64(x)), _p(T))
    return T.reshape(3, 4)


def se3_mul(A, B):
    Cm = np.zeros(12)
    lib().orc_se3_mul(_p(c64(A).reshape(12)), _p(c64(B).reshape(12)), _p(Cm))
    return Cm.reshape(3, 4)


def se3_inv(A):
    Cm = np.zeros(12)
    lib().orc_se3_inv(_p(c64(A).reshape(12)), _p(Cm))
    return Cm.reshape(3, 4)


def ldlt6_solve(H, b):
    x = np.zeros(6)
    lib().orc_ldlt6_solve(_p(c64(H).reshape(36)), _p(c64(b)), _p(x))
    return x


ALIGN_EXITS = {1: "border_first", 2: "border", 3: "converged", 4: "max_iter", 5: "rollback", 6: "nan"}  # ORC_ALIGN_EXIT_*


def align2d(cur_img, pwb, ref_patch, n_iter, px, want_exit=False):
    """(converged, px); with want_exit, (converged, px, exit, n_iter_done) where exit is a name of ALIGN_EXITS."""
    px = c64(px).copy()
    a = (_p(cur_img), cur_img.shape[1], cur_img.shape[0], cur_img.strides[0], _p(np.ascontiguousarray(pwb, np.uint8)),
         _p(np.ascontiguousarray(ref_patch, np.uint8)), int(n_iter), _p(px))
    if not want_exit:
        return bool(lib().orc_align2d(*a)), px
    it, ex = C.c_int(0), C.c_int(0)
    ok = lib().orc_align2d_ex(*a, C.byref(it), C.byref(ex))
    return bool(ok), px, ALIGN_EXITS[ex.value], it.value


def align1d(cur_img, direction, pwb, ref_patch, n_iter, px, want_exit=False):
    """(converged, px, h_inv); with want_exit, (converged, px, h_inv, exit, n_iter_done)."""
    px = c64(px).copy()
    d = np.ascontiguousarray(direction, np.float32)
    h = C.c_double(0)
    a = (_p(cur_img), cur_img.shape[1], cur_img.shape[0], cur_img.strides[0], _p(d), _p(np.ascontiguousarray(pwb, np.uint8)),
         _p(np.ascontiguousarray(ref_patch, np.uint8)), int(n_iter), _p(px), C.byref(h))
    if not want_exit:
        ok = lib().orc_align1d(*a)
        return bool(ok), px, h.value
    it, ex = C.c_int(0), C.c_int(0)
    ok = lib().orc_align1d_ex(*a, C.byref(it), C.byref(ex))
    return bool(ok), px, h.value, ALIGN_EXITS[ex.value], it.value


def warp_matrix_affine(cam, px_ref, f_ref, depth, T_cur_ref, level_ref):
    A = np.zeros(4)
    cs = cam_struct(cam)
    lib().orc_get_warp_matrix_affine(C.byref(cs), C.byref(cs), _p(c64(px_ref)), _p(c64(f_ref)),
                                     C.c_double(depth), _p(c64(T_cur_ref).reshape(12)), level_ref, _p(A))
    return A.reshape(2, 2)


def best_search_level(A, max_level):
    return lib().orc_get_best_search_level(_p(c64(A).reshape(4)), max_level)


def warp_affine(A, img_ref, px_ref, level_ref, search_level, halfpatch_size):
    patch = np.zeros((2 * halfpatch_size, 2 * halfpatch_size), np.uint8)
    ok = lib().orc_warp_affine(_p(c64(A).reshape(4)), _p(img_ref), img_ref.shape[1], img_ref.shape[0],
                               _p(c64(px_ref)), level_ref, search_level, halfpatch_size, _p(patch))
    return bool(ok), patch


def depth_from_triangulation(T, f_ref, f_cur):
    d = C.c_double(0)
    ok = lib().orc_depth_from_triangulation(_p(c64(T).reshape(12)), _p(c64(f_ref)), _p(c64(f_cur)), C.byref(d))
    return bool(ok), d.value


def find_match_direct(ref_pyr, cur_pyr, cam, T_cur_ref, ref_px, ref_f, ref_level, ftr_type, ref_grad,
                      depth_ref, max_search_level, align_max_iter, px_cur):
    """The two pyramids share their level sizes but may differ in depth; the levels one of them lacks are passed as NULL
    (the matcher reads ref_pyr[ref_level] and cur_pyr[search level] only)."""
    n = max(len(ref_pyr), len(cur_pyr))
    rp, _, _ = _level_ptrs(ref_pyr, n)
    cp, _, _ = _level_ptrs(cur_pyr, n)
    deeper = ref_pyr if len(ref_pyr) >= len(cur_pyr) else cur_pyr
    cols = np.array([im.shape[1] for im in deeper], dtype=np.int32)
    rows = np.array([im.shape[0] for im in deeper], dtype=np.int32)
    out = MatchResult()
    cs = cam_struct(cam)
    lib().orc_find_match_direct(rp, cp, _p(cols), _p(rows), n, C.byref(cs),
                                _p(c64(T_cur_ref).reshape(12)), _p(c64(ref_px)), _p(c64(ref_f)),
                                ref_level, ftr_type, _p(c64(ref_grad)), C.c_double(depth_ref),
                                max_search_level, align_max_iter, _p(c64(px_cur)), C.byref(out))
    return dict(success=bool(out.success), search_level=out.search_level,
                px_cur=np.array(out.px_cur[:]), A_cur_ref=np.array(out.A_cur_ref[:]).reshape(2, 2),
                h_inv=out.h_inv)


def find_epipolar_match_direct(ref_pyr, cur_pyr, cam, T_cur_ref, ref_px, ref_f, ref_level, ftr_type,
                               ref_grad, d_est, d_min, d_max, max_search_level, align_max_iter=10,
                               max_epi_search_steps=1000, align_1d=False):
    rp, cols, rows = _level_ptrs(ref_pyr)
    cp, _, _ = _level_ptrs(cur_pyr)
    out = EpiResult()
    cs = cam_struct(cam)
    lib().orc_find_epipolar_match_direct(rp, cp, _p(cols), _p(rows), len(ref_pyr), C.byref(cs),
                                         _p(c64(T_cur_ref).reshape(12)), _p(c64(ref_px)),
                                         _p(c64(ref_f)), ref_level, ftr_type, _p(c64(ref_grad)),
                                         C.c_double(d_est), C.c_double(d_min), C.c_double(d_max),
                                         max_search_level, align_max_iter, max_epi_search_steps,
                                         int(align_1d), C.byref(out))
    return dict(success=bool(out.success), reject=bool(out.reject), search_level=out.search_level,
                n_zmssd=out.n_zmssd_evals, epi_length=out.epi_length, px_cur=np.array(out.px_cur[:]),
                depth=out.depth, h_inv=out.h_inv, A_cur_ref=np.array(out.A_cur_ref[:]).reshape(2, 2))


def update_seed(x, tau2, a, b, mu, z_range, sigma2):
    """Returns the updated (a, b, mu, z_range, sigma2) as float32 scalars."""
    s = np.array([a, b, mu, z_range, sigma2], dtype=np.float32)
    base = s.ctypes.data
    lib().orc_update_seed(C.c_float(x), C.c_float(tau2), base, base + 4, base + 8, base + 12, base + 16)
    return s


def compute_tau(T_ref_cur, f, z, px_error_angle):
    return lib().orc_compute_tau(_p(c64(T_ref_cur).reshape(12)), _p(c64(f)), z, px_error_angle)


def depth_filter_update(ref_pyrs, ref_T_f_w, cur_pyr, cur_T_f_w, cam, ref_index, ftr_px, ftr_f,
                        ftr_level, ftr_type, ftr_grad, batch_id, batch_counter, seeds, max_n_kfs=3,
                        sigma2_thresh=200.0, max_search_level=2, align_max_iter=10, max_epi_search_steps=1000):
    """seeds: dict of float32 arrays a,b,mu,z_range,sigma2 (updated copies are returned)."""
    n_ref = len(ref_pyrs)
    nl = len(cur_pyr)
    flat = (C.c_void_p * (n_ref * nl))()
    for r, pyr in enumerate(ref_pyrs):
        for l, im in enumerate(pyr):
            flat[r * nl + l] = im.ctypes.data
    cp, cols, rows = _level_ptrs(cur_pyr)
    M = len(ref_index)
    out = {k: np.ascontiguousarray(seeds[k], np.float32).copy() for k in ("a", "b", "mu", "z_range", "sigma2")}
    status = np.zeros(M, np.uint8)
    pxc = np.zeros((M, 2))
    z = np.zeros(M)
    nz = np.zeros(M, np.int32)
    cs = cam_struct(cam)
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    refT = c64(np.asarray(ref_T_f_w)).reshape(-1)
    ri, fl, ft, bi = i32(ref_index), i32(ftr_level), i32(ftr_type), i32(batch_id)
    fpx, ff, fg = c64(ftr_px), c64(ftr_f), c64(ftr_grad)
    lib().orc_depth_filter_update(flat, _p(refT), n_ref, cp, _p(c64(cur_T_f_w).reshape(12)), _p(cols),
                                  _p(rows), nl, C.byref(cs), M, _p(ri), _p(fpx), _p(ff), _p(fl),
                                  _p(ft), _p(fg), _p(bi), batch_counter, max_n_kfs,
                                  C.c_double(sigma2_thresh), max_search_level, int(align_max_iter),
                                  int(max_epi_search_steps), _p(out["a"]),
                                  _p(out["b"]), _p(out["mu"]), _p(out["z_range"]), _p(out["sigma2"]),
                                  _p(status), _p(pxc), _p(z), _p(nz))
    out.update(status=status, px_cur=pxc, z=z, n_zmssd=nz)
    return out


def pose_optimize(reproj_thresh, n_iter, fx, T_f_w, f, pos, level, has_point):
    T = c64(T_f_w).copy().reshape(12)
    hp = np.ascontiguousarray(has_point, np.uint8).copy()
    out = PoseOptResult()
    lv = np.ascontiguousarray(level, np.int32)
    f, pos = c64(f), c64(pos)
    lib().orc_pose_optimize(C.c_double(reproj_thresh), n_iter, C.c_double(fx), _p(T), _p(f), _p(pos),
                            _p(lv), _p(hp), len(hp), C.byref(out))
    return dict(T=T.reshape(3, 4), has_point=hp, estimated_scale=out.estimated_scale,
                error_init=out.error_init, error_final=out.error_final, num_obs=out.num_obs,
                n_iter_done=out.n_iter_done, cov=np.array(out.cov[:]).reshape(6, 6))


def point_optimize(n_iter, pos, obs_T_f_w, obs_f):
    p = c64(pos).copy()
    T = c64(np.asarray(obs_T_f_w)).reshape(-1)
    f = c64(obs_f)
    lib().orc_point_optimize(int(n_iter), _p(p), len(f), _p(T), _p(f))
    return p


# ---- oracle/_ref: the reference's own classes (compiled from /root/reference with stand-in headers) ----
_ref_lib = None


def ref_lib():
    """CDLL of oracle/_ref/libsvo_ref.so or None when it has not been built."""
    global _ref_lib
    if _ref_lib is None:
        path = os.path.join(_HERE, "_ref", "libsvo_ref.so")
        if not os.path.exists(path):
            build_ref()
        if os.path.exists(path):
            _ref_lib = C.CDLL(path)
            _ref_lib.ref_sparse_img_align.restype = C.c_longlong
    return _ref_lib


def _cam4(cam):
    """[fx fy cx cy model d0..d4] for the ref_* wrappers (oracle/ref_wrap.cpp: make_camera)."""
    d = ([float(x) for x in getattr(cam, "d", ())] + [0.0] * 5)[:5]
    return c64([cam.fx, cam.fy, cam.cx, cam.cy, float(getattr(cam, "model", 0))] + d)


def ref_sparse_img_align(ref_l0, cur_l0, n_levels, cam, T_ref_w, T_cur_w, px, f, pos, has_point, max_level, min_level,
                         n_iter=30):
    """svo::SparseImgAlign(max, min, n_iter, GaussNewton, false, false).run(ref, cur) of the compiled reference; the
    frames' pyramids are built by the reference's own frame_utils::createImgPyramid."""
    h, w = ref_l0.shape
    T = c64(T_cur_w).copy().reshape(12)
    px, f, pos = c64(px), c64(f), c64(pos)
    hp = np.ascontiguousarray(has_point, np.uint8)
    n = len(hp)
    vis = np.zeros(n, np.uint8)
    H = np.zeros(36)
    cache = np.zeros((n, 16), np.float32)
    ret = ref_lib().ref_sparse_img_align(_p(np.ascontiguousarray(ref_l0)), _p(np.ascontiguousarray(cur_l0)), w, h, n_levels,
                                         _p(_cam4(cam)), _p(c64(T_ref_w).reshape(12)), _p(T), _p(px), _p(f), _p(pos), _p(hp),
                                         n, max_level, min_level, n_iter, _p(vis), _p(H), _p(cache))
    return dict(T_cur_w=T.reshape(3, 4), n_tracked=int(ret), visible=vis, H=H.reshape(6, 6), ref_patch=cache)


def ref_sparse_residuals(ref_l0, cur_l0, n_levels, cam, T_ref_w, T_cur_w, px, f, pos, has_point, level):
    """svo::SparseImgAlign::computeResiduals(T_cur_from_ref, true, true) of the compiled reference at one level and one
    pose (fresh object, precomputeReferencePatches included): visibility mask, patch cache, H_, Jres_, chi2, n_meas_ and
    |res| of every pixel of every in-image patch in feature order (`abs_res`, n_meas values)."""
    h, w = ref_l0.shape
    px, f, pos = c64(px), c64(f), c64(pos)
    hp = np.ascontiguousarray(has_point, np.uint8)
    n = len(hp)
    vis = np.zeros(n, np.uint8)
    cache = np.zeros((n, 16), np.float32)
    H, Jres = np.zeros(36), np.zeros(6)
    chi2 = C.c_double(0)
    absres = np.zeros(16 * max(n, 1), np.float32)
    L = ref_lib()
    L.ref_sparse_residuals.restype = C.c_longlong
    nm = L.ref_sparse_residuals(_p(np.ascontiguousarray(ref_l0)), _p(np.ascontiguousarray(cur_l0)), w, h, n_levels,
                                _p(_cam4(cam)), _p(c64(T_ref_w).reshape(12)), _p(c64(T_cur_w).reshape(12)), _p(px), _p(f),
                                _p(pos), _p(hp), n, int(level), _p(vis), _p(cache), _p(H), _p(Jres), C.byref(chi2), _p(absres),
                                C.c_longlong(len(absres)))
    return dict(visible=vis, ref_patch=cache, H=H.reshape(6, 6), Jres=Jres, chi2=chi2.value, n_meas=int(nm),
                abs_res=absres[:int(nm)].reshape(-1, 16))


def ref_image_pyramid(img, n_levels):
    """frame_utils::createImgPyramid of the compiled reference (svo/src/frame.cpp:156-165 over the shim's vk::halfSample,
    real SSE2 intrinsics on this x86 host)."""
    h, w = img.shape
    sizes = [((h >> l), (w >> l)) for l in range(n_levels)]
    out = np.zeros(sum(a * b for a, b in sizes), np.uint8)
    ref_lib().ref_image_pyramid(_p(np.ascontiguousarray(img, np.uint8)), w, h, n_levels, _p(out))
    pyr, o = [], 0
    for a, b in sizes:
        pyr.append(out[o:o + a * b].reshape(a, b).copy())
        o += a * b
    return pyr


def ref_last_seconds() -> float:
    """Seconds the reference algorithm itself took inside the most recent ref_* call (setup / copies excluded)."""
    L = ref_lib()
    L.ref_last_seconds.restype = C.c_double
    return float(L.ref_last_seconds())


def ref_align2d_batch(level0, n_levels, level, pwb, patch, n_iter, px):
    """feature_alignment::align2D of the compiled reference for M problems in one C loop."""
    lv = np.ascontiguousarray(level, np.int32)
    M = len(lv)
    p = c64(px).copy().reshape(M, 2)
    conv = np.zeros(M, np.uint8)
    h, w = level0.shape
    ref_lib().ref_align2d_batch(_p(np.ascontiguousarray(level0, np.uint8)), w, h, n_levels, M, _p(lv),
                                _p(np.ascontiguousarray(pwb, np.uint8)), _p(np.ascontiguousarray(patch, np.uint8)), int(n_iter), _p(p),
                                _p(conv))
    return conv.astype(bool), p


def ref_pose_optimize(reproj_thresh, n_iter, cam, T_f_w, f, pos, level, has_point):
    T = c64(T_f_w).copy().reshape(12)
    hp = np.ascontiguousarray(has_point, np.uint8).copy()
    sc = np.zeros(4)
    cov = np.zeros(36)
    ref_lib().ref_pose_optimize(C.c_double(reproj_thresh), n_iter, _p(_cam4(cam)), cam.width, cam.height, _p(T), _p(c64(f)),
                                _p(c64(pos)), _p(np.ascontiguousarray(level, np.int32)), _p(hp), len(hp), _p(sc), _p(cov))
    return dict(T=T.reshape(3, 4), has_point=hp, estimated_scale=sc[0], error_init=sc[1], error_final=sc[2],
                num_obs=int(sc[3]), cov=cov.reshape(6, 6))


def ref_point_optimize(n_iter, pos, obs_T_f_w, obs_f):
    p = c64(pos).copy()
    f = c64(obs_f)
    ref_lib().ref_point_optimize(int(n_iter), _p(p), len(f), _p(c64(np.asarray(obs_T_f_w)).reshape(-1)), _p(f))
    return p


class RefMatchOut(C.Structure):
    _fields_ = [("success", C.c_int), ("search_level", C.c_int), ("reject", C.c_int), ("px_cur", C.c_double * 2),
                ("A", C.c_double * 4), ("h_inv", C.c_double), ("epi_length", C.c_double), ("depth", C.c_double)]


def ref_matcher(mode, ref_l0, cur_l0, n_levels, cam, T_ref_w, T_cur_w, ref_px, ref_f, ref_level, ftr_type, ref_grad,
                point_pos, px_cur=(0, 0), d_est=0.0, d_min=0.0, d_max=0.0, n_pyr_levels=3):
    """mode 0: svo::Matcher::findMatchDirect(pt, cur, px_cur); mode 1: findEpipolarMatchDirect(ref, cur, ftr, d_est,
    d_min, d_max) of the compiled reference (default Matcher::Options)."""
    h, w = ref_l0.shape
    out = RefMatchOut()
    ref_lib().ref_matcher(mode, _p(np.ascontiguousarray(ref_l0)), _p(np.ascontiguousarray(cur_l0)), w, h, n_levels,
                          _p(_cam4(cam)), _p(c64(T_ref_w).reshape(12)), _p(c64(T_cur_w).reshape(12)), _p(c64(ref_px)),
                          _p(c64(ref_f)), ref_level, ftr_type, _p(c64(ref_grad)), _p(c64(point_pos)), _p(c64(px_cur)),
                          C.c_double(d_est), C.c_double(d_min), C.c_double(d_max), n_pyr_levels, C.byref(out))
    return dict(success=bool(out.success), search_level=out.search_level, reject=bool(out.reject),
                px_cur=np.array(out.px_cur[:]), A_cur_ref=np.array(out.A[:]).reshape(2, 2), h_inv=out.h_inv,
                epi_length=out.epi_length, depth=out.depth)


def ref_align2d(cur_img, pwb, ref_patch, n_iter, px):
    px = c64(px).copy()
    pwb, ref_patch = np.ascontiguousarray(pwb, np.uint8).copy(), np.ascontiguousarray(ref_patch, np.uint8).copy()
    ok = ref_lib().ref_align2d(_p(cur_img), cur_img.shape[1], cur_img.shape[0], cur_img.strides[0], _p(pwb), _p(ref_patch),
                               n_iter, _p(px))
    return bool(ok), px


def ref_align1d(cur_img, direction, pwb, ref_patch, n_iter, px):
    px = c64(px).copy()
    d = np.ascontiguousarray(direction, np.float32)
    pwb, ref_patch = np.ascontiguousarray(pwb, np.uint8).copy(), np.ascontiguousarray(ref_patch, np.uint8).copy()
    h = C.c_double(0)
    ok = ref_lib().ref_align1d(_p(cur_img), cur_img.shape[1], cur_img.shape[0], cur_img.strides[0], _p(d), _p(pwb),
                               _p(ref_patch), n_iter, _p(px), C.byref(h))
    return bool(ok), px, h.value


def ref_update_seed(x, tau2, a, b, mu, z_range, sigma2):
    s = np.array([a, b, mu, z_range, sigma2], dtype=np.float32)
    base = s.ctypes.data
    ref_lib().ref_update_seed(C.c_float(x), C.c_float(tau2), base, base + 4, base + 8, base + 12, base + 16)
    return s


def ref_compute_tau(T_ref_cur, f, z, px_error_angle):
    fn = ref_lib().ref_compute_tau
    fn.restype = C.c_double
    return fn(_p(c64(T_ref_cur).reshape(12)), _p(c64(f)), C.c_double(z), C.c_double(px_error_angle))


def ref_depth_filter_update(ref_l0s, ref_T_f_w, cur_l0, cur_T_f_w, n_levels, cam, ref_index, ftr_px, ftr_f, ftr_level,
                            ftr_type, ftr_grad, batch_id, batch_counter, seeds, n_pyr_levels=3):
    """svo::DepthFilter::updateSeeds of the compiled reference.  status: 0 kept, 1 converged, 2 erased."""
    imgs = np.ascontiguousarray(np.stack(ref_l0s))
    h, w = cur_l0.shape
    M = len(ref_index)
    out = {k: np.ascontiguousarray(seeds[k], np.float32).copy() for k in ("a", "b", "mu", "z_range", "sigma2")}
    status = np.zeros(M, np.uint8)
    xyz = np.zeros((M, 3))
    i32 = lambda a: np.ascontiguousarray(a, np.int32)
    ref_lib().ref_depth_filter_update(_p(imgs), _p(c64(np.asarray(ref_T_f_w)).reshape(-1)), len(ref_l0s),
                                      _p(np.ascontiguousarray(cur_l0)), _p(c64(cur_T_f_w).reshape(12)), w, h, n_levels,
                                      _p(_cam4(cam)), M, _p(i32(ref_index)), _p(c64(ftr_px)), _p(c64(ftr_f)),
                                      _p(i32(ftr_level)), _p(i32(ftr_type)), _p(c64(ftr_grad)), _p(i32(batch_id)),
                                      batch_counter, n_pyr_levels, _p(out["a"]), _p(out["b"]), _p(out["mu"]),
                                      _p(out["z_range"]), _p(out["sigma2"]), _p(status), _p(xyz))
    out.update(status=status, xyz_world=xyz)
    return out


class RefStream:
    """B frame pairs (frame k, frame k+1) held by the compiled reference; run() times svo::SparseImgAlign::run alone."""

    def __init__(self, level0s, cam, n_levels, T_f_w, feat_offset, px, f, pos, has_point):
        L = ref_lib()
        L.ref_stream_create.restype = C.c_void_p
        L.ref_stream_run.restype = C.c_double
        imgs = self._imgs = np.ascontiguousarray(level0s, np.uint8)  # level 0 of the frames aliases this memory
        self.B = imgs.shape[0] - 1
        h, w = imgs.shape[1:]
        self._h = C.c_void_p(L.ref_stream_create(_p(imgs), self.B, w, h, n_levels, _p(_cam4(cam)),
                                                 _p(c64(np.asarray(T_f_w)).reshape(-1)),
                                                 _p(np.ascontiguousarray(feat_offset, np.int32)), _p(c64(px)), _p(c64(f)),
                                                 _p(c64(pos)), _p(np.ascontiguousarray(has_point, np.uint8))))

    def run(self, n_threads, max_level, min_level, n_iter=30, want_poses=False):
        T = np.zeros((self.B, 3, 4)) if want_poses else None
        nt = np.zeros(self.B, np.int64)
        sec = ref_lib().ref_stream_run(self._h, int(n_threads), max_level, min_level, n_iter, _p(T) if want_poses else None,
                                       _p(nt))
        return dict(seconds=sec, T=T, n_tracked=nt)

    def destroy(self):
        if self._h:
            ref_lib().ref_stream_destroy(self._h)
            self._h = None


# ---- Reprojector::reprojectMap on a flat map view ----
class MapView(C.Structure):
    _fields_ = [("n_kfs", C.c_int), ("kf_T_f_w", C.c_void_p), ("kf_keypt_pos", C.c_void_p), ("kf_keypt_valid", C.c_void_p),
                ("kf_fts_offset", C.c_void_p), ("kf_fts", C.c_void_p), ("n_ftrs", C.c_int), ("ftr_kf", C.c_void_p),
                ("ftr_px", C.c_void_p), ("ftr_f", C.c_void_p), ("ftr_level", C.c_void_p), ("ftr_type", C.c_void_p),
                ("ftr_grad", C.c_void_p), ("ftr_point", C.c_void_p), ("n_points", C.c_int), ("pt_pos", C.c_void_p),
                ("pt_obs_offset", C.c_void_p), ("pt_obs", C.c_void_p), ("n_candidates", C.c_int), ("cand_point", C.c_void_p)]


class ReprojectOptions(C.Structure):
    _fields_ = [("grid_size", C.c_int), ("max_fts", C.c_int), ("max_n_kfs", C.c_int), ("find_match_direct", C.c_int),
                ("max_search_level", C.c_int), ("align_max_iter", C.c_int)]


class ReprojectStats(C.Structure):
    _fields_ = [("n_matches", C.c_int64), ("n_trials", C.c_int64), ("n_new", C.c_int), ("n_overlap", C.c_int),
                ("n_projected", C.c_int), ("n_speculative", C.c_int)]


_MV_DTYPES = dict(kf_T_f_w=np.float64, kf_keypt_pos=np.float64, kf_keypt_valid=np.uint8, kf_fts_offset=np.int32,
                  kf_fts=np.int32, ftr_kf=np.int32, ftr_px=np.float64, ftr_f=np.float64, ftr_level=np.int32,
                  ftr_type=np.int32, ftr_grad=np.float64, ftr_point=np.int32, pt_pos=np.float64, pt_obs_offset=np.int32,
                  pt_obs=np.int32, cand_point=np.int32)


def pack_map_view(view, struct_cls=MapView):
    """dict of arrays -> (ctypes struct, keep-alive list)."""
    mv, keep = struct_cls(), []
    for k, v in view.items():
        if k in _MV_DTYPES:
            a = np.ascontiguousarray(v, _MV_DTYPES[k])
            keep.append(a)
            setattr(mv, k, a.ctypes.data)
        else:
            setattr(mv, k, int(v))
    return mv, keep


def reproject_outputs(view, options, pt_type, pt_n_failed, pt_n_succeeded):
    P, cap = int(view["n_points"]), int(options["max_fts"]) + 1
    return dict(pt_type=np.ascontiguousarray(pt_type, np.int32).copy(), pt_n_failed=np.ascontiguousarray(pt_n_failed, np.int32).copy(),
                pt_n_succeeded=np.ascontiguousarray(pt_n_succeeded, np.int32).copy(), pt_action=np.zeros(P, np.uint8),
                overlap_kf=np.full(int(options["max_n_kfs"]), -1, np.int32), overlap_count=np.zeros(int(options["max_n_kfs"]), np.int64),
                new_point=np.full(cap, -1, np.int32), new_px=np.zeros((cap, 2)), new_level=np.zeros(cap, np.int32),
                new_type=np.zeros(cap, np.int32), new_grad=np.zeros((cap, 2)))


def trim_reproject(o, st):
    n, k = st.n_new, st.n_overlap
    for key in ("new_point", "new_px", "new_level", "new_type", "new_grad"):
        o[key] = o[key][:n]
    o["overlap_kf"], o["overlap_count"] = o["overlap_kf"][:k], o["overlap_count"][:k]
    o.update(n_matches=st.n_matches, n_trials=st.n_trials, n_new=n, n_overlap=k, n_projected=st.n_projected,
             n_speculative=st.n_speculative)
    return o


def reproject_map(case):
    """Reprojector::reprojectMap restated (sequential cell policy)."""
    v = case["view"]
    mv, keep = pack_map_view(v)
    nl = case["n_levels"]
    flat = (C.c_void_p * (v["n_kfs"] * nl))()
    for k, pyr in enumerate(case["kf_pyr"]):
        for l, im in enumerate(pyr):
            flat[k * nl + l] = im.ctypes.data
    cp, cols, rows = _level_ptrs(case["cur_pyr"])
    opt = ReprojectOptions(**case["options"])
    o = reproject_outputs(v, case["options"], case["pt_type"], case["pt_n_failed"], case["pt_n_succeeded"])
    st = ReprojectStats()
    cs = cam_struct(case["cam"])
    co = np.ascontiguousarray(case["cell_order"], np.int32)
    lib().orc_reproject_map(C.byref(mv), flat, cp, _p(cols), _p(rows), nl, C.byref(cs), _p(c64(case["cur_T_f_w"]).reshape(12)),
                            C.byref(opt), _p(co), _p(o["pt_type"]), _p(o["pt_n_failed"]), _p(o["pt_n_succeeded"]),
                            _p(o["pt_action"]), _p(o["overlap_kf"]), _p(o["overlap_count"]), _p(o["new_point"]), _p(o["new_px"]),
                            _p(o["new_level"]), _p(o["new_type"]), _p(o["new_grad"]), C.byref(st))
    return trim_reproject(o, st)


def ref_reproject_map(case):
    """svo::Reprojector::reprojectMap of the compiled reference (oracle/_ref) on the same flat map view."""
    v = case["view"]
    mv, keep = pack_map_view(v)
    kf_l0 = np.ascontiguousarray(np.stack([pyr[0] for pyr in case["kf_pyr"]]))
    cur_l0 = np.ascontiguousarray(case["cur_pyr"][0])
    h, w = cur_l0.shape
    opt = ReprojectOptions(**case["options"])
    o = reproject_outputs(v, case["options"], case["pt_type"], case["pt_n_failed"], case["pt_n_succeeded"])
    st = ReprojectStats()
    co = np.ascontiguousarray(case["cell_order"], np.int32)
    ref_lib().ref_reproject_map(C.byref(mv), _p(kf_l0), _p(cur_l0), w, h, case["n_levels"], _p(_cam4(case["cam"])),
                                _p(c64(case["cur_T_f_w"]).reshape(12)), C.byref(opt), _p(co), _p(o["pt_type"]),
                                _p(o["pt_n_failed"]), _p(o["pt_n_succeeded"]), _p(o["pt_action"]), _p(o["overlap_kf"]),
                                _p(o["overlap_count"]), _p(o["new_point"]), _p(o["new_px"]), _p(o["new_level"]),
                                _p(o["new_type"]), _p(o["new_grad"]), C.byref(st))
    return trim_reproject(o, st)


def fast_detect(pyr, n_pyr_levels, cell_size, detection_threshold, grid_occupancy=None, cap=4096, nonmax_ties_suppress=0,
                fast_threshold=20):
    """FastDetector::detect restated: returns dict(x, y, level, score) in grid-cell order.  fast_threshold is the FAST
    segment-test threshold b, which the reference hard-codes to 20."""
    lp, cols, rows = _level_ptrs(pyr)
    h, w = pyr[0].shape
    x, y, lv = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    sc = np.zeros(cap, np.float32)
    occ = None if grid_occupancy is None else np.ascontiguousarray(grid_occupancy, np.uint8)
    n = lib().orc_fast_detect(lp, _p(cols), _p(rows), n_pyr_levels, w, h, cell_size, _p(occ) if occ is not None else None,
                              C.c_double(detection_threshold), int(fast_threshold), int(nonmax_ties_suppress), _p(x), _p(y),
                              _p(lv), _p(sc), cap)
    assert n <= cap
    return dict(x=x[:n], y=y[:n], level=lv[:n], score=sc[:n])


def ref_fast_detect(l0, n_levels, n_pyr_levels, cell_size, detection_threshold, grid_occupancy=None, cap=4096):
    """feature_detection::FastDetector::detect of the compiled reference (with the [EXT] fast library restated)."""
    h, w = l0.shape
    x, y, lv = np.zeros(cap, np.int32), np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    occ = None if grid_occupancy is None else np.ascontiguousarray(grid_occupancy, np.uint8)
    n = ref_lib().ref_fast_detect(_p(np.ascontiguousarray(l0)), w, h, n_levels, n_pyr_levels, cell_size,
                                  _p(occ) if occ is not None else None, C.c_double(detection_threshold), _p(x), _p(y), _p(lv), cap)
    return dict(x=x[:n], y=y[:n], level=lv[:n])
