"""ctypes binding of libsvo_b200.so -- the thin Python face of the C ABI in include/svo_b200.h.

The product path is the CUDA library.  There is no CPU fallback: `load()` raises if the shared
library has not been built, and `Context()` raises if no CUDA device is usable.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsvo_b200.so")
MAX_LEVELS = 8


class SvoB200Error(RuntimeError):
    pass


class Camera(C.Structure):
    _fields_ = [("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("width", C.c_int), ("height", C.c_int), ("model", C.c_int), ("reserved_", C.c_int),
                ("d", C.c_double * 5)]


class FrameUploadEntry(C.Structure):  # svo_b200_frame_upload_entry
    _fields_ = [("frame", C.c_void_p), ("level0", C.c_void_p)]


class SiaOptions(C.Structure):
    _fields_ = [("max_level", C.c_int), ("min_level", C.c_int), ("n_iter", C.c_int), ("eps", C.c_double)]


class SiaIter(C.Structure):
    _fields_ = [("level", C.c_int), ("iter", C.c_int), ("accepted", C.c_int), ("n_meas", C.c_int),
                ("chi2", C.c_double), ("x", C.c_double * 6), ("T", C.c_double * 12)]


class SiaStats(C.Structure):
    _fields_ = [("n_iters", C.c_int32), ("sum_visible", C.c_int32), ("sum_in_image", C.c_int32),
                ("n_tracked", C.c_int32)]


SIA_STAGE_NAMES = {-1: None, 0: "global", 1: "image", 2: "window"}  # SVO_B200_SIA_STAGE_*
# robust cost (svo_b200_sia_robust): SVO_B200_SCALE_* / SVO_B200_WEIGHT_*, vikit's numbering
SCALE_UNIT, SCALE_TDIST, SCALE_MAD, SCALE_NORMAL = 0, 1, 2, 3
WEIGHT_UNIT, WEIGHT_TDIST, WEIGHT_TUKEY, WEIGHT_HUBER = 0, 1, 2, 3


class SiaLaunch(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("n_pairs", "ctas_per_pair", "threads", "features_per_thread", "min_blocks", "upfront",
                                       "general_camera", "residuals_only", "stage_cap", "smem_bytes", "resident_clusters", "sm_count", "min_level", "max_level")] + \
                [("level_stage", C.c_int * MAX_LEVELS)]


class MatchOptions(C.Structure):
    _fields_ = [("max_search_level", C.c_int), ("align_max_iter", C.c_int)]


class PoseOptResult(C.Structure):
    _fields_ = [("estimated_scale", C.c_double), ("error_init", C.c_double), ("error_final", C.c_double),
                ("num_obs", C.c_int64), ("n_iter_done", C.c_int), ("n_pivoted_solves", C.c_int16),
                ("cov_pivoted", C.c_int16), ("cov", C.c_double * 36)]


# ---- Reprojector::reprojectMap on a flat map view (svo_b200_reproject_map) ----
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


class ReprojectStream(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("map", "kf_frames", "cur", "cur_T_f_w", "cam", "opt", "cell_order", "pt_type_io",
                                          "pt_n_failed_io", "pt_n_succeeded_io", "pt_action_out", "overlap_kf_out",
                                          "overlap_count_out", "new_point_out", "new_px_out", "new_level_out",
                                          "new_type_out", "new_grad_out", "stats")]


class DetectOptions(C.Structure):
    _fields_ = [("cell_size", C.c_int), ("n_pyr_levels", C.c_int), ("fast_threshold", C.c_int),
                ("nonmax_ties_suppress", C.c_int), ("detection_threshold", C.c_double)]


class DetectStream(C.Structure):
    _fields_ = [("frame", C.c_void_p), ("opt", C.c_void_p), ("grid_occupancy", C.c_void_p), ("cap", C.c_int),
                ("x_out", C.c_void_p), ("y_out", C.c_void_p), ("level_out", C.c_void_p), ("score_out", C.c_void_p),
                ("n_out", C.c_void_p)]


class DepthOptions(C.Structure):
    _fields_ = [("max_n_kfs", C.c_int), ("seed_convergence_sigma2_thresh", C.c_double),
                ("max_search_level", C.c_int), ("align_max_iter", C.c_int), ("max_epi_search_steps", C.c_int)]


class EpipolarOptions(C.Structure):  # svo_b200_epipolar_options
    _fields_ = [("align_1d", C.c_int), ("subpix_refinement", C.c_int), ("epi_search_edgelet_filtering", C.c_int),
                ("epi_search_edgelet_max_angle", C.c_double)]


# ------------------------------------------------------------------ KLT tracking of the two-view initialisation
KLT_CONVERGED, KLT_HALF_STEP, KLT_MAX_ITER, KLT_OUT_OF_BOUNDS, KLT_SMALL_EIG = 0, 1, 2, 3, 4  # SVO_B200_KLT_*


class KltBuild(C.Structure):  # svo_b200_klt_build
    _fields_ = [("pyr", C.c_void_p), ("frame", C.c_void_p), ("max_level", C.c_int), ("with_derivatives", C.c_int)]


class KltOptions(C.Structure):
    _fields_ = [("win_size", C.c_int), ("max_level", C.c_int), ("max_iter", C.c_int), ("eps", C.c_double)]


class KltExit(C.Structure):
    _fields_ = [("reason", C.c_int32), ("level_reason", C.c_int32 * MAX_LEVELS), ("iters", C.c_int32 * MAX_LEVELS)]


class KltStream(C.Structure):  # svo_b200_klt_stream
    _fields_ = [("prev", C.c_void_p), ("next", C.c_void_p), ("opt", C.c_void_p), ("N", C.c_int), ("prev_pts", C.c_void_p),
                ("next_pts_io", C.c_void_p), ("status_out", C.c_void_p), ("exit_out", C.c_void_p)]


SIA_STATS_DTYPE = np.dtype([("n_iters", np.int32), ("sum_visible", np.int32),
                            ("sum_in_image", np.int32), ("n_tracked", np.int32)])

# Every function include/svo_b200.h declares, in its order: (name, return type, argument types).  Every pointer is a
# c_void_p, which takes numpy addresses (_p), handles, byref() structs, ctypes arrays and None; every scalar has its exact
# C type, so ctypes converts Python and numpy numbers at each call.
_ptr, _int, _dbl = C.c_void_p, C.c_int, C.c_double
PROTOTYPES = (
    # context
    ("svo_b200_create", _int, (_ptr, _int)),
    ("svo_b200_destroy", None, (_ptr,)),
    ("svo_b200_last_error", C.c_char_p, (_ptr,)),
    ("svo_b200_stream", _ptr, (_ptr,)),
    ("svo_b200_synchronize", _int, (_ptr,)),
    ("svo_b200_last_kernel_ms", _int, (_ptr, _ptr)),
    ("svo_b200_launch_count", C.c_uint64, (_ptr,)),
    ("svo_b200_version", C.c_char_p, ()),
    # frames
    ("svo_b200_frame_create", _int, (_ptr, _int, _int, _int, _ptr)),
    ("svo_b200_set_pyramid_rule", _int, (_ptr, _int)),
    ("svo_b200_frame_upload", _int, (_ptr, _ptr, _ptr, _int)),
    ("svo_b200_frame_upload_streams", _int, (_ptr, _int, _ptr)),
    ("svo_b200_frame_upload_device", _int, (_ptr, _ptr, _ptr)),
    ("svo_b200_frame_download_level", _int, (_ptr, _ptr, _int, _ptr)),
    ("svo_b200_frame_download_level_tiled", _int, (_ptr, _ptr, _int, _ptr)),
    ("svo_b200_frame_destroy", None, (_ptr, _ptr)),
    ("svo_b200_frame_pool_create", _int, (_ptr, _int, _int, _int, _int, _ptr)),
    ("svo_b200_frame_pool_get", _ptr, (_ptr, _int)),
    ("svo_b200_frame_pool_upload", _int, (_ptr, _ptr, _int, _int, _ptr, C.c_size_t)),
    ("svo_b200_frame_pool_destroy", None, (_ptr, _ptr)),
    # SparseImgAlign
    ("svo_b200_sparse_img_align", _int, (_ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _int, _ptr, _ptr,
                                         _ptr, _ptr, _int, _ptr)),
    ("svo_b200_sia_batch_stage", _int, (_ptr, _int, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr)),
    ("svo_b200_sia_batch_run", _int, (_ptr,)),
    ("svo_b200_sia_batch_fetch", _int, (_ptr, _ptr, _ptr, _ptr, _ptr)),
    ("svo_b200_sia_config", _int, (_ptr, _int, _int)),
    ("svo_b200_sia_upfront", _int, (_ptr, _int)),
    ("svo_b200_sia_last_launch", _int, (_ptr, _ptr)),
    ("svo_b200_sia_robust", _int, (_ptr, _int, _int)),
    ("svo_b200_sia_last_scales", _int, (_ptr, _int, _ptr)),
    ("svo_b200_sia_split_create", _int, (_ptr, _int, _int, _int, _ptr, _ptr)),
    ("svo_b200_sia_split_connect", _int, (_ptr, _ptr, _ptr)),
    ("svo_b200_sia_split_destroy", _int, (_ptr,)),
    ("svo_b200_sparse_residuals", _int, (_ptr, _ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _int, _ptr, _ptr,
                                         _ptr, _ptr, _ptr, _ptr, _ptr, _ptr)),
    # feature alignment, direct matcher, pose and point optimizers
    ("svo_b200_align2d_batch", _int, (_ptr, _ptr, _int, _ptr, _ptr, _ptr, _int, _ptr, _ptr)),
    ("svo_b200_align1d_batch", _int, (_ptr, _ptr, _int, _ptr, _ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr)),
    ("svo_b200_find_match_direct", _int, (_ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr, _ptr,
                                          _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr)),
    ("svo_b200_pose_optimize", _int, (_ptr, _dbl, _int, _dbl, _ptr, _ptr, _ptr, _ptr, _ptr, _int, _ptr)),
    ("svo_b200_pose_optimize_batch", _int, (_ptr, _int, _dbl, _int, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr)),
    ("svo_b200_point_optimize_batch", _int, (_ptr, _int, _int, _ptr, _ptr, _ptr, _ptr, _int, _ptr)),
    # reprojector, FAST detector
    ("svo_b200_reproject_map", _int, (_ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr,
                                      _ptr, _ptr, _ptr, _ptr, _ptr)),
    ("svo_b200_reproject_map_streams", _int, (_ptr, _int, _ptr)),
    ("svo_b200_fast_detect", _int, (_ptr, _ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr, _ptr, _ptr)),
    ("svo_b200_fast_detect_streams", _int, (_ptr, _int, _ptr)),
    # depth filter, epipolar matcher
    ("svo_b200_depth_filter_update", _int, (_ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr, _ptr,
                                            _ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr)),
    ("svo_b200_depth_filter_update_streams", _int, (_ptr, _int, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _int, _ptr, _ptr,
                                                    _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr,
                                                    _ptr, _ptr, _ptr)),
    ("svo_b200_find_epipolar_match_direct", _int, (_ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr,
                                                   _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr,
                                                   _ptr, _ptr)),
    ("svo_b200_set_epipolar_options", _int, (_ptr, _ptr)),
    ("svo_b200_get_epipolar_options", _int, (_ptr, _ptr)),
    ("svo_b200_epipolar_last_h_inv", _int, (_ptr, _int, _ptr, _ptr)),
    # KLT tracking
    ("svo_b200_klt_pyramid_create", _int, (_ptr, _ptr)),
    ("svo_b200_klt_pyramid_destroy", None, (_ptr, _ptr)),
    ("svo_b200_klt_pyramid_build", _int, (_ptr, _ptr, _ptr, _int, _int)),
    ("svo_b200_klt_pyramid_levels", _int, (_ptr,)),
    ("svo_b200_klt_pyramid_build_streams", _int, (_ptr, _int, _ptr)),
    ("svo_b200_klt_pyramid_download", _int, (_ptr, _ptr, _int, _ptr, _ptr)),
    ("svo_b200_klt_track", _int, (_ptr, _ptr, _ptr, _ptr, _int, _ptr, _ptr, _ptr, _ptr)),
    ("svo_b200_klt_track_streams", _int, (_ptr, _int, _ptr)),
)

_lib = None


def load() -> C.CDLL:
    """Load the CUDA library; fail loudly if it is missing (no fallback of any kind)."""
    global _lib
    if _lib is None:
        path = os.environ.get("SVO_B200_LIB", LIB_PATH)  # override: instrumented builds of the same library
        if not os.path.exists(path):
            raise SvoB200Error(f"{path} is missing: build it with `python -m rpg_svo_b200.build` "
                               "(there is no CPU fallback)")
        _lib = C.CDLL(path)
        for name, restype, argtypes in PROTOTYPES:
            fn = getattr(_lib, name)
            fn.restype, fn.argtypes = restype, argtypes
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def c64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _u8(a):
    return np.ascontiguousarray(a, dtype=np.uint8)


def _frame_array(frames):
    return (C.c_void_p * len(frames))(*[f.h.value for f in frames])


def _fields(s: C.Structure) -> list:
    """The values of a struct's fields in order: one stream entry as the arguments of the single-stream call."""
    return [getattr(s, name) for name, _ in s._fields_]


CAM_PINHOLE, CAM_ATAN = 0, 1


def cam_struct(cam) -> Camera:
    """`cam` needs fx, fy, cx, cy, width, height; optional `model` (CAM_*) and `d` (up to 5 coefficients)."""
    d = (C.c_double * 5)(*([float(x) for x in getattr(cam, "d", ())] + [0.0] * 5)[:5])
    return Camera(cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height, int(getattr(cam, "model", 0)), 0, d)


def _pose_result(T, has_point, o: PoseOptResult) -> dict:
    """One frame's pose_optimize result, like the oracle's."""
    return dict(T=T.reshape(3, 4), has_point=has_point, estimated_scale=o.estimated_scale, error_init=o.error_init,
                error_final=o.error_final, num_obs=o.num_obs, n_iter_done=o.n_iter_done,
                n_pivoted_solves=o.n_pivoted_solves, cov_pivoted=o.cov_pivoted, cov=np.array(o.cov[:]).reshape(6, 6))


_MV_DTYPES = dict(kf_T_f_w=np.float64, kf_keypt_pos=np.float64, kf_keypt_valid=np.uint8, kf_fts_offset=np.int32,
                  kf_fts=np.int32, ftr_kf=np.int32, ftr_px=np.float64, ftr_f=np.float64, ftr_level=np.int32,
                  ftr_type=np.int32, ftr_grad=np.float64, ftr_point=np.int32, pt_pos=np.float64, pt_obs_offset=np.int32,
                  pt_obs=np.int32, cand_point=np.int32)


def _reproject_prepare(view: dict, kf_frames, cur: Frame, cur_T_f_w, cam, options: dict, cell_order, pt_type, pt_n_failed,
                       pt_n_succeeded):
    """The svo_b200_reproject_stream of one call, its output arrays and the objects the call keeps alive."""
    mv, keep = MapView(), []
    for k, v in view.items():
        if k in _MV_DTYPES:
            a = np.ascontiguousarray(v, _MV_DTYPES[k])
            keep.append(a)
            setattr(mv, k, a.ctypes.data)
        else:
            setattr(mv, k, int(v))
    opt = ReprojectOptions(**options)
    P, cap, nk = int(view["n_points"]), int(options["max_fts"]) + 1, int(options["max_n_kfs"])
    o = dict(pt_type=_i32(pt_type).copy(), pt_n_failed=_i32(pt_n_failed).copy(), pt_n_succeeded=_i32(pt_n_succeeded).copy(),
             pt_action=np.zeros(P, np.uint8), overlap_kf=np.full(nk, -1, np.int32), overlap_count=np.zeros(nk, np.int64),
             new_point=np.full(cap, -1, np.int32), new_px=np.zeros((cap, 2)), new_level=np.zeros(cap, np.int32),
             new_type=np.zeros(cap, np.int32), new_grad=np.zeros((cap, 2)))
    st = ReprojectStats()
    fr = _frame_array(kf_frames)
    cs = cam_struct(cam)
    co = _i32(cell_order)
    cT = c64(cur_T_f_w).reshape(12)
    keep += [mv, opt, st, fr, cs, co, cT]
    rs = ReprojectStream(C.cast(C.pointer(mv), C.c_void_p), C.cast(fr, C.c_void_p), cur.h.value, cT.ctypes.data,
                         C.cast(C.pointer(cs), C.c_void_p), C.cast(C.pointer(opt), C.c_void_p), co.ctypes.data,
                         *[o[k].ctypes.data for k in ("pt_type", "pt_n_failed", "pt_n_succeeded", "pt_action", "overlap_kf",
                                                      "overlap_count", "new_point", "new_px", "new_level", "new_type",
                                                      "new_grad")],
                         C.cast(C.pointer(st), C.c_void_p))
    return rs, o, st, keep


def _reproject_result(o: dict, st: ReprojectStats) -> dict:
    n, k = st.n_new, st.n_overlap
    for key in ("new_point", "new_px", "new_level", "new_type", "new_grad"):
        o[key] = o[key][:n]
    o["overlap_kf"], o["overlap_count"] = o["overlap_kf"][:k], o["overlap_count"][:k]
    o.update(n_matches=st.n_matches, n_trials=st.n_trials, n_new=n, n_overlap=k, n_projected=st.n_projected,
             n_speculative=st.n_speculative)
    return o


def _detect_prepare(frame: Frame, cell_size, n_pyr_levels, detection_threshold, grid_occupancy=None, fast_threshold=20,
                    nonmax_ties_suppress=0, cap=8192):
    """The svo_b200_detect_stream of one fast_detect call, its outputs and the objects the call keeps alive."""
    opt = DetectOptions(int(cell_size), int(n_pyr_levels), int(fast_threshold), int(nonmax_ties_suppress), float(detection_threshold))
    o = dict(x=np.zeros(cap, np.int32), y=np.zeros(cap, np.int32), level=np.zeros(cap, np.int32), score=np.zeros(cap, np.float32))
    occ = None if grid_occupancy is None else _u8(grid_occupancy)
    n = C.c_int(0)
    ds = DetectStream(frame.h.value if frame.h else None, C.cast(C.pointer(opt), C.c_void_p), _p(occ), int(cap),
                      *[o[k].ctypes.data for k in ("x", "y", "level", "score")], C.cast(C.pointer(n), C.c_void_p))
    return ds, o, n, (opt, occ)


def _detect_result(o: dict, n: C.c_int) -> dict:
    k = min(n.value, len(o["x"]))
    return dict(x=o["x"][:k], y=o["y"][:k], level=o["level"][:k], score=o["score"][:k], n=n.value)


def _klt_prepare(prev: KltPyramid | None, nxt: KltPyramid | None, prev_pts, next_pts, max_level=4, max_iter=30, eps=0.001,
                 win_size=30, want_exit=True):
    """The svo_b200_klt_stream of one klt_track call, its outputs and the objects the call keeps alive."""
    p0 = np.ascontiguousarray(prev_pts, np.float32).reshape(-1, 2)
    p1 = np.ascontiguousarray(next_pts, np.float32).reshape(-1, 2).copy()
    n = len(p0)
    st = np.zeros(max(n, 1), np.uint8)
    ex = (KltExit * max(n, 1))() if want_exit else None
    opt = KltOptions(int(win_size), int(max_level), int(max_iter), float(eps))
    ks = KltStream(prev.h.value if prev is not None else None, nxt.h.value if nxt is not None else None,
                   C.cast(C.pointer(opt), C.c_void_p), n, p0.ctypes.data, p1.ctypes.data, st.ctypes.data,
                   C.cast(ex, C.c_void_p) if ex is not None else None)
    return ks, (p1, st, ex, n), (opt, p0)


def _klt_result(o) -> dict:
    p1, st, ex, n = o
    r = dict(next_pts=p1, status=st[:n])
    if ex is not None:
        r["reason"] = np.array([e.reason for e in ex[:n]], np.int32)
        r["level_reason"] = np.array([list(e.level_reason) for e in ex[:n]], np.int32).reshape(n, MAX_LEVELS)
        r["iters"] = np.array([list(e.iters) for e in ex[:n]], np.int32).reshape(n, MAX_LEVELS)
    return r


class Frame:
    """An image pyramid resident in HBM (the image side of svo::Frame)."""

    def __init__(self, ctx: "Context", width: int, height: int, n_levels: int, handle: C.c_void_p | None = None):
        """A new frame, or with `handle` a borrowed one that its owner frees (a frame-pool frame): destroy() leaves it be."""
        self.ctx, self.width, self.height, self.n_levels = ctx, width, height, n_levels
        self.borrowed = handle is not None
        if handle is None:
            handle = C.c_void_p()
            ctx._check(ctx.lib.svo_b200_frame_create(ctx.h, width, height, n_levels, C.byref(handle)))
        self.h = handle

    def upload(self, levels) -> "Frame":
        """levels: list of >=1 contiguous uint8 arrays (level 0 first); missing levels are built on the GPU."""
        arr = (C.c_void_p * len(levels))()
        keep = []
        for i, im in enumerate(levels):
            im = np.ascontiguousarray(im, dtype=np.uint8)
            assert im.shape == (self.height >> i, self.width >> i), (im.shape, i)
            keep.append(im)
            arr[i] = im.ctypes.data
        self.ctx._check(self.ctx.lib.svo_b200_frame_upload(self.ctx.h, self.h, arr, len(levels)))
        self.ctx.synchronize()  # host arrays may be freed by the caller right after
        return self

    def upload_ptrs(self, ptrs) -> None:
        """Asynchronous upload from raw (pinned) host pointers; the caller keeps the memory alive."""
        arr = (C.c_void_p * len(ptrs))(*ptrs)
        self.ctx._check(self.ctx.lib.svo_b200_frame_upload(self.ctx.h, self.h, arr, len(ptrs)))

    def upload_device(self, dev_ptr: int) -> None:
        self.ctx._check(self.ctx.lib.svo_b200_frame_upload_device(self.ctx.h, self.h, dev_ptr))

    def download_level(self, level: int) -> np.ndarray:
        out = np.zeros((self.height >> level, self.width >> level), np.uint8)
        self.ctx._check(self.ctx.lib.svo_b200_frame_download_level(self.ctx.h, self.h, level, _p(out)))
        return out

    def download_level_tiled(self, level: int) -> np.ndarray:
        """The level's block-tiled copy as [ceil(h/4), ceil(w/4), 4 rows, 4 columns]."""
        w, h = self.width >> level, self.height >> level
        out = np.zeros(((h + 3) // 4, (w + 3) // 4, 4, 4), np.uint8)
        self.ctx._check(self.ctx.lib.svo_b200_frame_download_level_tiled(self.ctx.h, self.h, level, _p(out)))
        return out

    def destroy(self):
        if self.h and not self.borrowed:
            self.ctx.lib.svo_b200_frame_destroy(self.ctx.h, self.h)
        self.h = None

    def __del__(self):
        try:
            if self.h and self.ctx.h:
                self.destroy()
        except Exception:
            pass


class FramePool:
    """`count` frames of one geometry in one device slab: one strided H2D copy + one fused pyramid
    kernel per upload (svo_b200_frame_pool_*)."""

    def __init__(self, ctx: "Context", width: int, height: int, n_levels: int, count: int):
        self.ctx, self.width, self.height, self.n_levels, self.count = ctx, width, height, n_levels, count
        h = C.c_void_p()
        ctx._check(ctx.lib.svo_b200_frame_pool_create(ctx.h, width, height, n_levels, count, C.byref(h)))
        self.h = h
        self.frames = [Frame(ctx, width, height, n_levels, C.c_void_p(ctx.lib.svo_b200_frame_pool_get(h, i)))
                       for i in range(count)]

    def upload(self, first: int, count: int, host_ptr: int, host_stride: int) -> None:
        """Asynchronous when `host_ptr` is pinned memory; the caller keeps it alive."""
        self.ctx._check(self.ctx.lib.svo_b200_frame_pool_upload(self.ctx.h, self.h, first, count, host_ptr, host_stride))

    def upload_array(self, imgs: np.ndarray, first: int = 0) -> None:
        imgs = np.ascontiguousarray(imgs, dtype=np.uint8)
        assert imgs.shape[1:] == (self.height, self.width)
        self.upload(first, imgs.shape[0], imgs.ctypes.data, self.height * self.width)
        self.ctx.synchronize()

    def destroy(self):
        if self.h:
            for f in self.frames:
                f.h = None
            self.ctx.lib.svo_b200_frame_pool_destroy(self.ctx.h, self.h)
            self.h = None


class KltPyramid:
    """OpenCV's LK pyramid of one frame's level 0 (and, for the previous image, its Scharr derivatives) in HBM."""

    def __init__(self, ctx: "Context"):
        self.ctx = ctx
        h = C.c_void_p()
        ctx._check(ctx.lib.svo_b200_klt_pyramid_create(ctx.h, C.byref(h)))
        self.h = h

    def build(self, frame: Frame, derivatives: bool, max_level: int = 4) -> "KltPyramid":
        self.ctx._check(self.ctx.lib.svo_b200_klt_pyramid_build(self.ctx.h, self.h, frame.h, max_level, bool(derivatives)))
        self.width, self.height = frame.width, frame.height
        return self

    @property
    def n_levels(self) -> int:
        return int(self.ctx.lib.svo_b200_klt_pyramid_levels(self.h))

    def download(self, level: int, derivatives: bool = False):
        """(image h x w uint8, derivatives h x w x 2 int16 or None) of one level."""
        lib = self.ctx.lib
        w, h = self.width, self.height  # level l is ((w+1)/2, (h+1)/2) of level l-1
        for _ in range(level):
            w, h = (w + 1) // 2, (h + 1) // 2
        img = np.zeros((h, w), np.uint8)
        der = np.zeros((h, w, 2), np.int16) if derivatives else None
        self.ctx._check(lib.svo_b200_klt_pyramid_download(self.ctx.h, self.h, level, _p(img), _p(der)))
        return img, der

    def destroy(self):
        if self.h:
            self.ctx.lib.svo_b200_klt_pyramid_destroy(self.ctx.h, self.h)
            self.h = None


class Context:
    """One GPU + one CUDA stream (use one per calling host thread)."""

    def __init__(self, device: int = 0):
        self.lib = load()
        h = C.c_void_p()
        rc = self.lib.svo_b200_create(C.byref(h), device)
        if rc != 0:
            raise SvoB200Error(f"svo_b200_create(device={device}) failed with {rc}: no usable CUDA device "
                               "(the CUDA path is the only path)")
        self.h = h
        self.device = device

    def close(self):
        if self.h:
            self.lib.svo_b200_destroy(self.h)
            self.h = None

    def _check(self, rc: int):
        if rc != 0:
            raise SvoB200Error(f"svo_b200 error {rc}: {self.lib.svo_b200_last_error(self.h).decode()}")

    @property
    def stream(self) -> int:
        return int(self.lib.svo_b200_stream(self.h))

    def synchronize(self):
        self._check(self.lib.svo_b200_synchronize(self.h))

    def last_kernel_ms(self) -> float:
        """Device time of the kernel(s) of the last entry point (CUDA events inside the library, no copies)."""
        ms = C.c_float(0)
        self._check(self.lib.svo_b200_last_kernel_ms(self.h, C.byref(ms)))
        return float(ms.value)

    def launch_count(self) -> int:
        return int(self.lib.svo_b200_launch_count(self.h))

    # ------------------------------------------------------------------ frames
    def frame(self, pyr) -> Frame:
        """Create + upload a frame from a full host pyramid (list of uint8 arrays)."""
        f = Frame(self, pyr[0].shape[1], pyr[0].shape[0], len(pyr))
        return f.upload(pyr)

    def frame_from_level0(self, img, n_levels: int) -> Frame:
        f = Frame(self, img.shape[1], img.shape[0], n_levels)
        return f.upload([img])

    def set_pyramid_rule(self, rule: int):
        """1 = PYR_X86 (vikit's SSE2 rounding where an x86 build of the reference takes it; default), 0 = PYR_SCALAR."""
        self._check(self.lib.svo_b200_set_pyramid_rule(self.h, rule))

    def frames_upload(self, entries):
        """S frames' level-0 uploads and pyramid builds together (svo_b200_frame_upload_streams: one launch per stage, not
        per frame); each frame ends as Frame.upload([image]) leaves it.  `entries`: (frame, image) pairs, the image a uint8
        array of the frame's size, or the address of one in pinned host memory that the caller keeps alive.  The call waits
        for the device only when an entry is an array.  Returns the frames."""
        keep, arr = [], (FrameUploadEntry * max(len(entries), 1))()
        for i, (f, im) in enumerate(entries):
            if not isinstance(im, int):
                im = np.ascontiguousarray(im, dtype=np.uint8)
                assert im.shape == (f.height, f.width), (im.shape, i)
                keep.append(im)
                im = im.ctypes.data
            arr[i] = FrameUploadEntry(f.h.value if f.h else None, im)
        self._check(self.lib.svo_b200_frame_upload_streams(self.h, len(entries), arr))
        if keep:
            self.synchronize()  # host arrays may be freed by the caller right after
        return [f for f, _ in entries]

    # ------------------------------------------------------------------ SparseImgAlign
    def sparse_img_align(self, ref: Frame, cur: Frame, cam, T_init, px, f, pos, has_point, ref_pos,
                         max_level, min_level, n_iter=30, eps=1e-6, want_trace=False):
        n = int(np.asarray(px).shape[0])
        T = c64(T_init).copy().reshape(12)
        px, f, pos, rpos = c64(px), c64(f), c64(pos), c64(ref_pos)
        hp = np.ascontiguousarray(has_point, dtype=np.uint8)
        visible = np.zeros(max(n, 1), np.uint8)
        H = np.zeros(36)
        stats = SiaStats()
        # a negative n_iter runs up to 1000 iterations per level (the reference's size_t n_iter_: no limit); the trace
        # has room for 100 per level
        cap = ((max_level - min_level + 1) * (max(n_iter, 1) if n_iter >= 0 else 100) + 8) if want_trace else 0
        trace = (SiaIter * cap)() if cap else None
        ntr = C.c_int(0)
        cs = cam_struct(cam)
        opt = SiaOptions(max_level, min_level, n_iter, eps)
        self._check(self.lib.svo_b200_sparse_img_align(
            self.h, ref.h, cur.h, C.byref(cs), C.byref(opt), _p(T), _p(px), _p(f), _p(pos), _p(hp),
            _p(rpos), n, _p(visible), _p(H), C.byref(stats), trace, cap, C.byref(ntr)))
        tr = []
        for k in range(min(ntr.value, cap)):
            r = trace[k]
            tr.append(dict(level=r.level, iter=r.iter, accepted=r.accepted, n_meas=r.n_meas, chi2=r.chi2,
                           x=np.array(r.x[:]), T=np.array(r.T[:]).reshape(3, 4)))
        return dict(T=T.reshape(3, 4), n_tracked=int(stats.n_tracked), visible=visible[:n],
                    H=H.reshape(6, 6), trace=tr,
                    stats=dict(n_iters=stats.n_iters, sum_visible=stats.sum_visible,
                               sum_in_image=stats.sum_in_image, n_tracked=stats.n_tracked))

    def sia_batch_stage(self, refs, curs, cam, T_init, feat_offset, px, f, pos, has_point, ref_pos,
                        max_level, min_level, n_iter=30, eps=1e-6):
        B = len(refs)
        ra = (C.c_void_p * B)(*[r.h.value for r in refs])
        ca = (C.c_void_p * B)(*[c.h.value for c in curs])
        cs = cam_struct(cam)
        opt = SiaOptions(max_level, min_level, n_iter, eps)
        self._batch = dict(B=B, n=int(feat_offset[-1] - feat_offset[0]))
        fo = np.ascontiguousarray(feat_offset, np.int32)
        T, px, f, pos, rpos = c64(T_init), c64(px), c64(f), c64(pos), c64(ref_pos)
        hp = np.ascontiguousarray(has_point, np.uint8)
        self._check(self.lib.svo_b200_sia_batch_stage(self.h, B, ra, ca, C.byref(cs), C.byref(opt), _p(T),
                                                      _p(fo), _p(px), _p(f), _p(pos), _p(hp), _p(rpos)))

    def sia_batch_run(self):
        self._check(self.lib.svo_b200_sia_batch_run(self.h))

    def sia_batch_fetch(self, want_H=False):
        B, n = self._batch["B"], self._batch["n"]
        T = np.zeros((B, 3, 4))
        vis = np.zeros(max(n, 1), np.uint8)
        H = np.zeros((B, 6, 6)) if want_H else None
        stats = np.zeros(B, SIA_STATS_DTYPE)
        self._check(self.lib.svo_b200_sia_batch_fetch(self.h, _p(T), _p(vis), _p(H), _p(stats)))
        return dict(T=T, visible=vis[:n], H=H, stats=stats)

    def sia_config(self, ctas_per_pair=-1, features_per_thread=0):
        """Launch geometry of the alignment kernel (svo_b200_sia_config): -1 / 0 = automatic."""
        self._check(self.lib.svo_b200_sia_config(self.h, ctas_per_pair, features_per_thread))

    def sia_upfront(self, mode=-1):
        """Small-batch cluster geometry: all levels prepared before the first iteration (svo_b200_sia_upfront): -1 auto, 0 off."""
        self._check(self.lib.svo_b200_sia_upfront(self.h, mode))

    def sia_last_launch(self) -> dict:
        """The launch of the most recent alignment / residual / batch call (svo_b200_sia_last_launch): the instantiation's
        parameters, with `stages` = {level: "global" | "image" | "window"} for the levels it ran."""
        L = SiaLaunch()
        self._check(self.lib.svo_b200_sia_last_launch(self.h, C.byref(L)))
        d = {name: getattr(L, name) for name, _ in SiaLaunch._fields_ if name != "level_stage"}
        d["stages"] = {lv: SIA_STAGE_NAMES[L.level_stage[lv]] for lv in range(L.min_level, L.max_level + 1)}
        return d

    def sia_robust(self, scale=SCALE_UNIT, weight=WEIGHT_UNIT):
        """Robust cost of the alignment (svo_b200_sia_robust; vk::NLLSSolver::setRobustCostFunction): SCALE_MAD with
        WEIGHT_UNIT / WEIGHT_TUKEY / WEIGHT_HUBER turns weights on, SCALE_UNIT turns them off."""
        self._check(self.lib.svo_b200_sia_robust(self.h, scale, weight))

    def sia_last_scales(self, B: int = 1) -> np.ndarray:
        """(B, MAX_LEVELS) float32: the scale each pair's iterations used at each level in the last (weighted) alignment
        launch, NaN outside [min_level, max_level] (svo_b200_sia_last_scales)."""
        out = np.zeros((int(B), MAX_LEVELS), np.float32)
        self._check(self.lib.svo_b200_sia_last_scales(self.h, B, _p(out)))
        return out

    # ---- feature split of single pairs over GPUs (svo_b200_sia_split_*)
    def sia_split_create(self, rank: int, world: int, max_pairs: int = 1):
        """Returns (ipc_handle: bytes[64], device_ptr: int) of this rank's exchange buffer."""
        h = (C.c_ubyte * 64)()
        ptr = C.c_void_p()
        self._check(self.lib.svo_b200_sia_split_create(self.h, rank, world, max_pairs, h, C.byref(ptr)))
        return bytes(h), int(ptr.value)

    def sia_split_connect(self, ipc_handles=None, in_process_ptrs=None):
        """ipc_handles: list of `world` 64-byte handles (other processes) or in_process_ptrs: list of `world` device pointers."""
        if in_process_ptrs is not None:
            arr = (C.c_void_p * len(in_process_ptrs))(*[C.c_void_p(p) for p in in_process_ptrs])
            self._check(self.lib.svo_b200_sia_split_connect(self.h, None, arr))
        else:
            blob = b"".join(ipc_handles)
            buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
            self._check(self.lib.svo_b200_sia_split_connect(self.h, buf, None))

    def sia_split_destroy(self):
        self._check(self.lib.svo_b200_sia_split_destroy(self.h))

    def sparse_residuals(self, ref: Frame, cur: Frame, cam, level, T, px, f, pos, has_point, ref_pos,
                         visible_in=None):
        n = int(np.asarray(px).shape[0])
        vis = np.zeros(n, np.uint8) if visible_in is None else np.ascontiguousarray(visible_in, np.uint8).copy()
        ref_patch = np.zeros((n, 16), np.float32)
        res = np.zeros((n, 16), np.float32)
        inimg = np.zeros(n, np.uint8)
        H, Jres = np.zeros(36), np.zeros(6)
        chi2, nm = C.c_double(0), C.c_int64(0)
        cs = cam_struct(cam)
        T, px, f, pos, rpos = c64(T).reshape(12), c64(px), c64(f), c64(pos), c64(ref_pos)
        hp = np.ascontiguousarray(has_point, np.uint8)
        self._check(self.lib.svo_b200_sparse_residuals(
            self.h, ref.h, cur.h, C.byref(cs), level, _p(T), _p(px), _p(f), _p(pos), _p(hp), _p(rpos), n,
            _p(vis), _p(ref_patch), _p(res), _p(inimg), _p(H), _p(Jres), C.byref(chi2), C.byref(nm)))
        return dict(visible=vis, ref_patch=ref_patch, residuals=res, in_image=inimg, H=H.reshape(6, 6),
                    Jres=Jres, chi2=chi2.value, n_meas=nm.value)

    # ------------------------------------------------------------------ feature alignment, matcher
    def align2d_batch(self, cur: Frame, level, pwb, patch, n_iter, px):
        """feature_alignment::align2D for M features; returns (converged[M] bool, px[M,2])."""
        level = _i32(level)
        M = len(level)
        px = c64(px).copy().reshape(M, 2)
        conv = np.zeros(max(M, 1), np.uint8)
        pwb, patch = _u8(pwb).reshape(M, 100), _u8(patch).reshape(M, 64)
        self._check(self.lib.svo_b200_align2d_batch(self.h, cur.h, M, _p(level), _p(pwb), _p(patch), n_iter, _p(px),
                                                    _p(conv)))
        return conv[:M].astype(bool), px

    def align1d_batch(self, cur: Frame, level, direction, pwb, patch, n_iter, px):
        level = _i32(level)
        M = len(level)
        px = c64(px).copy().reshape(M, 2)
        conv = np.zeros(max(M, 1), np.uint8)
        h_inv = np.zeros(max(M, 1))
        d = np.ascontiguousarray(direction, np.float32).reshape(M, 2)
        pwb, patch = _u8(pwb).reshape(M, 100), _u8(patch).reshape(M, 64)
        self._check(self.lib.svo_b200_align1d_batch(self.h, cur.h, M, _p(level), _p(d), _p(pwb), _p(patch), n_iter,
                                                    _p(px), _p(conv), _p(h_inv)))
        return conv[:M].astype(bool), px, h_inv[:M]

    def find_match_direct(self, ref_frames, ref_T_f_w, cur: Frame, cur_T_f_w, cam, ref_index, ref_px, ref_f, ref_level,
                          ftr_type, ref_grad, point_pos, px_cur, max_search_level, align_max_iter=10):
        M = len(ref_index)
        ra = _frame_array(ref_frames)
        refT = c64(np.asarray(ref_T_f_w)).reshape(-1)
        px = c64(px_cur).copy().reshape(M, 2)
        succ = np.zeros(max(M, 1), np.uint8)
        sl = np.zeros(max(M, 1), np.int32)
        A = np.zeros((max(M, 1), 4))
        hinv = np.zeros(max(M, 1))
        cs = cam_struct(cam)
        opt = MatchOptions(max_search_level, align_max_iter)
        ri, lv, ty = _i32(ref_index), _i32(ref_level), _i32(ftr_type)
        rpx, rf, rg, pp, cT = c64(ref_px), c64(ref_f), c64(ref_grad), c64(point_pos), c64(cur_T_f_w).reshape(12)
        self._check(self.lib.svo_b200_find_match_direct(self.h, ra, _p(refT), len(ref_frames), cur.h, _p(cT), C.byref(cs),
                                                        C.byref(opt), M, _p(ri), _p(rpx), _p(rf), _p(lv), _p(ty), _p(rg),
                                                        _p(pp), _p(px), _p(succ), _p(sl), _p(A), _p(hinv)))
        return dict(success=succ[:M].astype(bool), px_cur=px, search_level=sl[:M], A_cur_ref=A[:M].reshape(M, 2, 2),
                    h_inv=hinv[:M])

    # ------------------------------------------------------------------ pose and point optimizers
    def pose_optimize(self, reproj_thresh, n_iter, fx, T_f_w, f, pos, level, has_point):
        """pose_optimizer::optimizeGaussNewton; returns dict like the oracle's."""
        T = c64(T_f_w).copy().reshape(12)
        hp = _u8(has_point).copy()
        out = PoseOptResult()
        lv = _i32(level)
        f, pos = c64(f), c64(pos)
        self._check(self.lib.svo_b200_pose_optimize(self.h, reproj_thresh, n_iter, fx, _p(T), _p(f), _p(pos), _p(lv), _p(hp),
                                                    len(hp), C.byref(out)))
        return _pose_result(T, hp, out)

    def pose_optimize_batch(self, reproj_thresh, n_iter, fx, T_f_w, obs_offset, f, pos, level, has_point):
        """B frames in one launch (svo_b200_pose_optimize_batch); returns a list of dicts like pose_optimize."""
        off = _i32(obs_offset)
        B = len(off) - 1
        T = c64(T_f_w).copy().reshape(B, 12)
        hp = _u8(has_point).copy()
        out = (PoseOptResult * B)()
        fxa = c64(np.broadcast_to(np.asarray(fx, np.float64), (B,)))
        self._check(self.lib.svo_b200_pose_optimize_batch(self.h, B, reproj_thresh, n_iter, _p(fxa), _p(T), _p(off),
                                                          _p(c64(f)), _p(c64(pos)), _p(_i32(level)), _p(hp), out))
        return [_pose_result(T[b], hp[off[b]:off[b + 1]], out[b]) for b in range(B)]

    def point_optimize_batch(self, n_iter, pos, obs_offset, obs_frame, obs_f, frame_T_f_w):
        """Point::optimize for P points; returns the refined positions [P,3]."""
        p = c64(pos).copy().reshape(-1, 3)
        off, fr = _i32(obs_offset), _i32(obs_frame)
        f, T = c64(obs_f), c64(np.asarray(frame_T_f_w)).reshape(-1)
        self._check(self.lib.svo_b200_point_optimize_batch(self.h, len(p), n_iter, _p(off), _p(fr), _p(f), _p(T),
                                                           len(T) // 12, _p(p)))
        return p

    # ------------------------------------------------------------------ reprojector
    def reproject_map(self, view: dict, kf_frames, cur: Frame, cur_T_f_w, cam, options: dict, cell_order, pt_type,
                      pt_n_failed, pt_n_succeeded):
        """Reprojector::reprojectMap: `view` holds the svo_b200_map_view arrays by field name.  Returns the features the
        reference would add to the frame (new_*), the updated point state, per-point actions and the overlap keyframes."""
        rs, o, st, keep = _reproject_prepare(view, kf_frames, cur, cur_T_f_w, cam, options, cell_order, pt_type, pt_n_failed,
                                             pt_n_succeeded)
        self._check(self.lib.svo_b200_reproject_map(self.h, *_fields(rs)))
        return _reproject_result(o, st)

    def reproject_map_streams(self, streams):
        """S streams' Reprojector::reprojectMap with one device launch (svo_b200_reproject_map_streams).  `streams`: one
        dict per stream with the arguments of reproject_map by name (view, kf_frames, cur, cur_T_f_w, cam, options,
        cell_order, pt_type, pt_n_failed, pt_n_succeeded).  Returns one dict per stream, as reproject_map returns."""
        prep = [_reproject_prepare(**s) for s in streams]
        arr = (ReprojectStream * max(len(prep), 1))(*[p[0] for p in prep])
        self._check(self.lib.svo_b200_reproject_map_streams(self.h, len(prep), arr))
        return [_reproject_result(o, st) for _, o, st, _ in prep]

    # ------------------------------------------------------------------ FAST detector
    def fast_detect(self, frame: Frame, cell_size, n_pyr_levels, detection_threshold, grid_occupancy=None, fast_threshold=20,
                    nonmax_ties_suppress=0, cap=8192):
        """FastDetector::detect: dict(x, y, level, score) of the best corner per free grid cell, cell order."""
        ds, o, n, _keep = _detect_prepare(frame, cell_size, n_pyr_levels, detection_threshold, grid_occupancy, fast_threshold,
                                          nonmax_ties_suppress, cap)
        self._check(self.lib.svo_b200_fast_detect(self.h, *_fields(ds)))
        return _detect_result(o, n)

    def fast_detect_streams(self, streams):
        """S streams' FastDetector::detect with one device launch (svo_b200_fast_detect_streams).  `streams`: one dict per
        stream with the arguments of fast_detect by name (frame, cell_size, n_pyr_levels, detection_threshold and the
        optional grid_occupancy, fast_threshold, nonmax_ties_suppress, cap).  Returns one dict per stream, as fast_detect
        returns."""
        prep = [_detect_prepare(**s) for s in streams]
        arr = (DetectStream * max(len(prep), 1))(*[p[0] for p in prep])
        self._check(self.lib.svo_b200_fast_detect_streams(self.h, len(prep), arr))
        return [_detect_result(o, n) for _, o, n, _ in prep]

    # ------------------------------------------------------------------ depth filter, epipolar matcher
    def depth_filter_update(self, ref_frames, ref_T_f_w, cur: Frame, cur_T_f_w, cam, ref_index, ftr_px, ftr_f, ftr_level,
                            ftr_type, ftr_grad, batch_id, batch_counter, seeds, max_n_kfs=3, sigma2_thresh=200.0,
                            max_search_level=2, align_max_iter=10, max_epi_search_steps=1000):
        """DepthFilter::updateSeeds; `seeds` = dict of float32 arrays a,b,mu,z_range,sigma2 (copies are updated)."""
        M = len(ref_index)
        ra = _frame_array(ref_frames)
        refT = c64(np.asarray(ref_T_f_w)).reshape(-1)
        out = {k: np.ascontiguousarray(seeds[k], np.float32).copy() for k in ("a", "b", "mu", "z_range", "sigma2")}
        status = np.zeros(max(M, 1), np.uint8)
        pxc = np.zeros((max(M, 1), 2))
        z = np.zeros(max(M, 1))
        nz = np.zeros(max(M, 1), np.int32)
        cs = cam_struct(cam)
        opt = DepthOptions(max_n_kfs, sigma2_thresh, max_search_level, align_max_iter, max_epi_search_steps)
        ri, fl, ft, bi = _i32(ref_index), _i32(ftr_level), _i32(ftr_type), _i32(batch_id)
        fpx, ff, fg, cT = c64(ftr_px), c64(ftr_f), c64(ftr_grad), c64(cur_T_f_w).reshape(12)
        self._check(self.lib.svo_b200_depth_filter_update(
            self.h, ra, _p(refT), len(ref_frames), cur.h, _p(cT), C.byref(cs), C.byref(opt), M, _p(ri), _p(fpx), _p(ff),
            _p(fl), _p(ft), _p(fg), _p(bi), batch_counter, _p(out["a"]), _p(out["b"]), _p(out["mu"]),
            _p(out["z_range"]), _p(out["sigma2"]), _p(status), _p(pxc), _p(z), _p(nz)))
        out.update(status=status[:M], px_cur=pxc[:M], z=z[:M], n_zmssd=nz[:M])
        return out

    def depth_filter_update_streams(self, streams, ref_frames, ref_T_f_w, max_n_kfs=3, sigma2_thresh=200.0,
                                    max_search_level=2, align_max_iter=10, max_epi_search_steps=1000):
        """S streams' DepthFilter::updateSeeds in one launch (svo_b200_depth_filter_update_streams).  `streams`: one dict
        per stream with cur (Frame), cur_T_f_w, cam, batch_counter and the per-seed arrays of depth_filter_update
        (ref_index, ftr_px, ftr_f, ftr_level, ftr_type, ftr_grad, batch_id, seeds); ref_index indexes the shared keyframe
        table ref_frames / ref_T_f_w.  Returns one dict per stream, as depth_filter_update returns."""
        S = len(streams)
        n = [len(s["ref_index"]) for s in streams]
        off = np.zeros(S + 1, np.int32)
        off[1:] = np.cumsum(n)
        M = int(off[-1])

        def cat(key, dtype):
            parts = [np.asarray(s[key], dtype).reshape(-1) for s in streams]
            return np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0, dtype), dtype)

        seeds = {k: np.ascontiguousarray(np.concatenate([np.asarray(s["seeds"][k], np.float32).reshape(-1) for s in streams])
                                         if S else np.zeros(0, np.float32), np.float32) for k in ("a", "b", "mu", "z_range", "sigma2")}
        ri, fl, ft, bi = cat("ref_index", np.int32), cat("ftr_level", np.int32), cat("ftr_type", np.int32), cat("batch_id", np.int32)
        fpx, ff, fg = cat("ftr_px", np.float64), cat("ftr_f", np.float64), cat("ftr_grad", np.float64)
        status = np.zeros(max(M, 1), np.uint8)
        pxc, z, nz = np.zeros((max(M, 1), 2)), np.zeros(max(M, 1)), np.zeros(max(M, 1), np.int32)
        curs = (C.c_void_p * max(S, 1))(*[s["cur"].h.value for s in streams])
        cT = c64(np.stack([np.asarray(s["cur_T_f_w"], np.float64).reshape(12) for s in streams]) if S else np.zeros((1, 12)))
        cams = (Camera * max(S, 1))(*[cam_struct(s["cam"]) for s in streams])
        bc = _i32([int(s["batch_counter"]) for s in streams] or [0])
        ra = _frame_array(ref_frames)
        refT = c64(np.asarray(ref_T_f_w, np.float64).reshape(-1) if len(ref_frames) else np.zeros(12))
        opt = DepthOptions(max_n_kfs, sigma2_thresh, max_search_level, align_max_iter, max_epi_search_steps)
        self._check(self.lib.svo_b200_depth_filter_update_streams(
            self.h, S, curs, _p(cT), cams, _p(bc), _p(off), ra, _p(refT), len(ref_frames), C.byref(opt), _p(ri), _p(fpx),
            _p(ff), _p(fl), _p(ft), _p(fg), _p(bi), _p(seeds["a"]), _p(seeds["b"]), _p(seeds["mu"]), _p(seeds["z_range"]),
            _p(seeds["sigma2"]), _p(status), _p(pxc), _p(z), _p(nz)))
        res = []
        for s in range(S):
            a, b = off[s], off[s + 1]
            o = {k: seeds[k][a:b] for k in seeds}
            o.update(status=status[a:b], px_cur=pxc[a:b], z=z[a:b], n_zmssd=nz[a:b])
            res.append(o)
        return res

    def find_epipolar_match_direct(self, ref_frames, ref_T_f_w, cur: Frame, cur_T_f_w, cam, ref_index, ftr_px, ftr_f,
                                   ftr_level, ftr_type, ftr_grad, d_est, d_min, d_max, max_search_level=2, align_max_iter=10,
                                   max_epi_search_steps=1000):
        """Matcher::findEpipolarMatchDirect for M candidates (svo_b200_find_epipolar_match_direct)."""
        M = len(ref_index)
        ra = _frame_array(ref_frames)
        refT = c64(np.asarray(ref_T_f_w)).reshape(-1)
        succ, rej = np.zeros(max(M, 1), np.uint8), np.zeros(max(M, 1), np.uint8)
        depth, epi = np.zeros(max(M, 1)), np.zeros(max(M, 1))
        pxc, A = np.zeros((max(M, 1), 2)), np.zeros((max(M, 1), 4))
        sl, nz = np.zeros(max(M, 1), np.int32), np.zeros(max(M, 1), np.int32)
        cs = cam_struct(cam)
        opt = DepthOptions(3, 200.0, max_search_level, align_max_iter, max_epi_search_steps)
        self._check(self.lib.svo_b200_find_epipolar_match_direct(
            self.h, ra, _p(refT), len(ref_frames), cur.h, _p(c64(cur_T_f_w).reshape(12)), C.byref(cs), C.byref(opt), M,
            _p(_i32(ref_index)), _p(c64(ftr_px)), _p(c64(ftr_f)), _p(_i32(ftr_level)), _p(_i32(ftr_type)), _p(c64(ftr_grad)),
            _p(c64(d_est)), _p(c64(d_min)), _p(c64(d_max)), _p(succ), _p(depth), _p(pxc), _p(sl), _p(epi), _p(rej), _p(A),
            _p(nz)))
        return dict(success=succ[:M].astype(bool), depth=depth[:M], px_cur=pxc[:M], search_level=sl[:M], epi_length=epi[:M],
                    reject=rej[:M].astype(bool), A_cur_ref=A[:M].reshape(M, 2, 2), n_zmssd=nz[:M])

    def set_epipolar_options(self, align_1d=False, subpix_refinement=True, edgelet_filtering=True, edgelet_max_angle=0.7):
        """Matcher::Options of the epipolar search (svo_b200_set_epipolar_options) for find_epipolar_match_direct,
        depth_filter_update and depth_filter_update_streams; the arguments' defaults are the reference's."""
        o = EpipolarOptions(int(align_1d), int(subpix_refinement), int(edgelet_filtering), float(edgelet_max_angle))
        self._check(self.lib.svo_b200_set_epipolar_options(self.h, C.byref(o)))

    def epipolar_options(self) -> dict:
        """The current setting (svo_b200_get_epipolar_options), in set_epipolar_options' keywords."""
        o = EpipolarOptions()
        self._check(self.lib.svo_b200_get_epipolar_options(self.h, C.byref(o)))
        return dict(align_1d=bool(o.align_1d), subpix_refinement=bool(o.subpix_refinement),
                    edgelet_filtering=bool(o.epi_search_edgelet_filtering), edgelet_max_angle=o.epi_search_edgelet_max_angle)

    def epipolar_last_h_inv(self, M: int):
        """(h_inv (M,) float64, ran_1d (M,) bool) of the first M candidates of the last find_epipolar_match_direct call
        (svo_b200_epipolar_last_h_inv): ran_1d where align1D ran and set Matcher::h_inv_ to h_inv."""
        h = np.zeros(max(int(M), 1))
        r = np.zeros(max(int(M), 1), np.uint8)
        self._check(self.lib.svo_b200_epipolar_last_h_inv(self.h, M, _p(h), _p(r)))
        return h[:M], r[:M].astype(bool)

    # ------------------------------------------------------------------ KLT tracking of the two-view initialisation
    def klt_pyramid(self, frame: Frame, derivatives: bool, max_level: int = 4) -> KltPyramid:
        """The LK pyramid of `frame`'s level 0 (already on the device), with the Scharr derivatives if `derivatives`."""
        return KltPyramid(self).build(frame, derivatives, max_level)

    def klt_pyramids(self, builds, pyramids=None):
        """S LK pyramids built together (svo_b200_klt_pyramid_build_streams: one launch per stage, not per pyramid).
        `builds`: one dict per pyramid with frame, derivatives and the optional max_level (4); `pyramids`: handles to
        rebuild (one per entry), new ones when None.  Returns the handles."""
        pyrs = [KltPyramid(self) for _ in builds] if pyramids is None else list(pyramids)
        assert len(pyrs) == len(builds)
        arr = (KltBuild * max(len(builds), 1))(*[KltBuild(p.h.value if p.h else None, b["frame"].h.value if b["frame"].h else None,
                                                          int(b.get("max_level", 4)), int(bool(b["derivatives"])))
                                                 for p, b in zip(pyrs, builds)])
        self._check(self.lib.svo_b200_klt_pyramid_build_streams(self.h, len(builds), arr))
        for p, b in zip(pyrs, builds):
            p.width, p.height = b["frame"].width, b["frame"].height
        return pyrs

    def klt_track(self, prev: KltPyramid | None, nxt: KltPyramid | None, prev_pts, next_pts, max_level=4, max_iter=30,
                  eps=0.001, win_size=30, want_exit=True):
        """calcOpticalFlowPyrLK(prev, next, prev_pts, next_pts, ..., OPTFLOW_USE_INITIAL_FLOW) on the device.
        dict(next_pts (N x 2 float32), status (N uint8), and with want_exit: reason (N), level_reason / iters (N x MAX_LEVELS))."""
        ks, o, _keep = _klt_prepare(prev, nxt, prev_pts, next_pts, max_level, max_iter, eps, win_size, want_exit)
        self._check(self.lib.svo_b200_klt_track(self.h, *_fields(ks)))
        return _klt_result(o)

    def klt_track_streams(self, streams):
        """S streams' calcOpticalFlowPyrLK with one device launch (svo_b200_klt_track_streams).  `streams`: one dict per
        stream with the arguments of klt_track by name (prev, nxt, prev_pts, next_pts and the optional max_level, max_iter,
        eps, win_size, want_exit).  Returns one dict per stream, as klt_track returns."""
        prep = [_klt_prepare(**s) for s in streams]
        arr = (KltStream * max(len(prep), 1))(*[p[0] for p in prep])
        self._check(self.lib.svo_b200_klt_track_streams(self.h, len(prep), arr))
        return [_klt_result(o) for _, o, _ in prep]
