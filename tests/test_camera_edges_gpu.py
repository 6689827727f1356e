"""GPU: the camera functions every projecting kernel inlines, on every camera of tests/camera_cases.py.

- A probe (tests/camera_probe.cu, built here into a temporary directory with the library's nvcc flags and linked against
  libsvo_b200.so for svo::cam_to_dev) runs svo_math.cuh's cam_world2cam / cam_cam2world over the catalogue's inputs:
  every output is one of the exactly rounded statement's candidates (tests/camera_hp.py), bit for bit for pinhole
  cameras, NaN where the statement is NaN.
- findMatchDirect, the depth filter, the epipolar matcher, the reprojector and the alignment kernel on the edge scenes,
  against the oracle; the alignment's general-camera instantiation is chosen exactly for the distorted cameras.
- The streams kernels with streams of different edge cameras equal the single calls bit for bit.
- Every entry point that takes a camera refuses one whose size is not its frames', writing nothing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from rpg_svo_b200 import build, capi, synth
from tests import camera_cases as cc
from tests import camera_hp as hp
from tests import depth_update_hp as dhp
from tests.test_depth_edges_gpu import _match_both
from tests.test_sia_driver_edges_gpu import assert_driver_parity
from tests.test_sia_geometry_gpu import GEOMETRIES, _configure
from tests.test_streams_gpu import RP_KEYS, SEED_KEYS, SIZE_OFFSETS, _resized, _same_bits

pytestmark = pytest.mark.gpu

CAMS = list(cc.CAMERAS)
# |A_cur_ref - oracle|: the camera functions are the statement's (the probe test), bit for bit for pinhole cameras and
# within 2 ulp of atan / tan for ATAN.  A also carries the pose product: the kernel composes T_cur_ref from the two frames'
# [R|t] through its quaternion storage, the oracle's se3_mul / se3_inv through its own, and the two differ in the last bits
# for some candidates of every camera; carried through the 5 px differences of getWarpMatrixAffine that leaves at most
# 2.3e-14 for pinhole and 4.5e-14 for ATAN cameras (measured on an H100).  The matched pixel is exact.
A_TOL = 1e-13
MEASURED = {}       # the largest deviations seen, printed at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("camera edges, largest deviations:", MEASURED)


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    lib = build.build()
    out = str(tmp_path_factory.mktemp("camera_probe") / "camera_probe")
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "camera_probe.cu")
    libdir = os.path.dirname(lib)
    subprocess.check_call([build._nvcc()] + build.NVCC_FLAGS + [src, "-o", out, "-L", libdir, "-l:libsvo_b200.so",
                                                              "-Xlinker", f"-rpath={libdir}"])
    return out


def _run_probe(exe, cam, xyz, px):
    d = os.path.dirname(exe)
    xyz, px = np.ascontiguousarray(xyz, np.float64).reshape(-1, 3), np.ascontiguousarray(px, np.float64).reshape(-1, 2)
    with open(os.path.join(d, "in.bin"), "wb") as f:
        f.write(bytes(capi.cam_struct(cam)) + np.array([len(xyz), len(px)], np.int64).tobytes() + xyz.tobytes() + px.tobytes())
    subprocess.check_call([exe, os.path.join(d, "in.bin"), os.path.join(d, "out.bin")])
    out = np.fromfile(os.path.join(d, "out.bin"), np.float64)
    return out[:2 * len(xyz)].reshape(-1, 2), out[2 * len(xyz):].reshape(-1, 3)


def _measure(key, v):
    MEASURED[key] = max(MEASURED.get(key, 0), v)


@pytest.mark.parametrize("name", CAMS)
def test_probe_outputs_are_statement_candidates(probe, name):
    cam = cc.CAMERAS[name]
    c = hp.cam_const(cam)
    w_in, p_in = cc.unit_plane_inputs(cam), cc.pixel_inputs(name)
    uv, f = _run_probe(probe, cam, [x for _, x in w_in], [p for _, p in p_in])
    for fn, inputs, outs, key in ((hp.world2cam_candidates, w_in, uv, "probe_atan_ulp"),
                                  (hp.cam2world_candidates, p_in, f, "probe_tan_ulp")):
        for (label, x), got in zip(inputs, outs):
            cands = fn(c, x)
            ks = [k for k, r in cands if hp.same_tuple(got, r)]
            assert ks, (name, label, tuple(got), cands)
            assert len(cands) == 1 or c.model == hp.ATAN, (name, label)
            _measure(key, abs(ks[0]))  # how far the device's atan / tan was from the correctly rounded value


# ---- findMatchDirect ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CAMS)
def test_find_match_direct_on_camera_edges(ctx, oracle, name):
    c = cc.match_scene(name)
    cam = c["cam"]
    ref, cur = ctx.frame(c["ref_pyr"]), ctx.frame(c["cur_pyr"])
    M = c["M"]
    g = ctx.find_match_direct([ref], [c["T_ref_w"]], cur, c["T_cur_w"], cam, np.zeros(M, np.int32), c["ref_px"], c["ref_f"],
                              c["ref_level"], c["ftr_type"], c["ref_grad"], c["point_pos"], c["px_cur"], 2)
    ref.destroy(); cur.destroy()
    T_cur_ref = oracle.se3_mul(c["T_cur_w"], oracle.se3_inv(c["T_ref_w"]))
    ref_pos = oracle.se3_inv(c["T_ref_w"])[:, 3]
    n_ok = 0
    for i in range(M):
        o = oracle.find_match_direct(c["ref_pyr"], c["cur_pyr"], cam, T_cur_ref, c["ref_px"][i], c["ref_f"][i],
                                     int(c["ref_level"][i]), int(c["ftr_type"][i]), c["ref_grad"][i],
                                     np.linalg.norm(c["point_pos"][i] - ref_pos), 2, 10, c["px_cur"][i])
        assert bool(g["success"][i]) == bool(o["success"]) and g["search_level"][i] == o["search_level"], (name, i)
        A_g, A_o = g["A_cur_ref"][i].ravel(), np.asarray(o["A_cur_ref"]).ravel()
        dA = float(np.max(np.abs(A_g - A_o)))
        _measure("find_match_direct_dA_" + ("atan" if cam.model else "pinhole"), dA)
        assert dA <= A_TOL, (name, i, dA)
        if o["success"]:
            n_ok += 1
            assert _same_bits(g["px_cur"][i], np.asarray(o["px_cur"], np.float64)), (name, i, g["px_cur"][i], o["px_cur"])
    assert n_ok > M // 3, (name, n_ok, M)


# ---- depth filter and epipolar matcher ----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CAMS)
def test_depth_filter_on_camera_edges(ctx, oracle, name):
    c = cc.depth_scene(name)
    cam = c["cam"]
    ref, cur = ctx.frame(c["ref_pyr"]), ctx.frame(c["cur_pyr"])
    args = (c["ref_index"], c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"], c["batch_counter"],
            c["seeds"])
    g = ctx.depth_filter_update([ref], [c["T_ref_w"]], cur, c["T_cur_w"], cam, *args)
    ref.destroy(); cur.destroy()
    o = oracle.depth_filter_update([c["ref_pyr"]], [c["T_ref_w"]], c["cur_pyr"], c["T_cur_w"], cam, *args)
    assert np.array_equal(g["status"], o["status"]) and np.array_equal(g["n_zmssd"], o["n_zmssd"]), name
    upd = o["status"] >= dhp.UPDATED
    assert upd[-c["n_axis"]:].sum() > 0, name  # seeds whose segment crosses the axis are matched
    dhp.assert_seed_updates(g, o, c["seeds"], [c["T_ref_w"]], c["ref_index"], c["T_cur_w"], c["ftr_f"], cam.fx, oracle)


@pytest.mark.parametrize("name", CAMS)
def test_epipolar_match_on_camera_edges(ctx, oracle, name):
    c = cc.depth_scene(name)
    idx = np.arange(c["M"])
    d_est = 1.0 / c["seeds"]["mu"].astype(np.float64)
    d = (d_est, d_est / 1.5, d_est * 1.8)
    g, os_ = _match_both(ctx, oracle, c, c["cur_pyr"], c["T_cur_w"], idx, d)
    assert sum(o["success"] for o in os_[-c["n_axis"]:]) > 0, name


# ---- reprojector --------------------------------------------------------------------------------------------------------
def _reproject_args(c, kfs, cur):
    return dict(view=c["view"], kf_frames=kfs, cur=cur, cur_T_f_w=c["cur_T_f_w"], cam=c["cam"], options=c["options"],
                cell_order=c["cell_order"], pt_type=c["pt_type"], pt_n_failed=c["pt_n_failed"], pt_n_succeeded=c["pt_n_succeeded"])


@pytest.mark.parametrize("name", CAMS)
def test_reproject_map_on_camera_edges(ctx, oracle, name):
    """Every output exact, with points 1e-11 to 1e-6 px to either side of u = 8 and u = width - 8 (both sides reached:
    test_camera_edges_pins.test_map_scene_reaches_both_sides_of_the_reprojection_border)."""
    c = cc.map_scene(name)
    kfs, cur = [ctx.frame(p) for p in c["kf_pyr"]], ctx.frame(c["cur_pyr"])
    g = ctx.reproject_map(**_reproject_args(c, kfs, cur))
    for f in kfs + [cur]:
        f.destroy()
    o = oracle.reproject_map(c)
    assert g["n_matches"] == o["n_matches"] > 5, name
    for k in ("new_point", "new_level", "new_px", "pt_type", "pt_n_failed", "pt_n_succeeded"):
        assert _same_bits(np.asarray(g[k]), np.asarray(o[k], dtype=np.asarray(g[k]).dtype)), (name, k)


# ---- alignment ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sia_scenes():
    return {}


SIA_N_ITER = 3  # per level: no Gauss-Newton decision of these scenes is then within 2e-5 of a tie (sia_driver_cases.margin)
SIA_SEED = {"pinhole_barrel": 906}  # seed 905's barrel run has a near-tie


def _align(ctx, oracle, sia_scenes, name, geometry):
    """The alignment of the camera's scene in one launch geometry: (kernel result, launch report, oracle result, scene)."""
    cam = cc.CAMERAS[name]
    if name not in sia_scenes:
        d = synth.make_frame_pair(SIA_SEED.get(name, 905), width=cc.W, height=cc.H, n_feat=300, n_levels=5, cam=cam)
        o = oracle.sparse_img_align(d["ref_pyr"], d["cur_pyr"], cam, synth.se3_identity(), d["px"], d["f"], d["pos"],
                                    d["has_point"], d["ref_pos"], 4, 0, n_iter=SIA_N_ITER)
        sia_scenes[name] = (d, o)
    d, o = sia_scenes[name]
    _configure(ctx, GEOMETRIES[geometry])
    ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
    try:
        g = ctx.sparse_img_align(ref, cur, cam, synth.se3_identity(), d["px"], d["f"], d["pos"], d["has_point"], d["ref_pos"],
                                 4, 0, n_iter=SIA_N_ITER, want_trace=True)
        L = ctx.sia_last_launch()
    finally:
        ctx.sia_config(-1, 0)
        ctx.sia_upfront(-1)
        ref.destroy(); cur.destroy()
    return g, L, o, d


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
@pytest.mark.parametrize("name", CAMS)
def test_sparse_img_align_on_camera_edges(ctx, oracle, sia_scenes, name, geometry):
    """test_sia_driver_edges_gpu.assert_driver_parity against the oracle (mask, n_tracked, the whole iteration trace with
    chi2 and steps, the pose; it asserts first that no decision is a near-tie).  A distorted camera runs the general-camera
    instantiation; an undistorted one (d0 = 0 with d1..d4 != 0 and |d0| = 1e-7 included) the same instantiation as the plain
    pinhole camera, which is the plain-pinhole one in the automatic geometry (the 8-CTA cluster geometry is built for the
    general camera only)."""
    cam = cc.CAMERAS[name]
    g, L, o, d = _align(ctx, oracle, sia_scenes, name, geometry)
    if cc.general(cam):
        assert L["general_camera"] == 1, (name, geometry)
    else:
        assert L["general_camera"] == _align(ctx, oracle, sia_scenes, "pinhole_plain", geometry)[1]["general_camera"], name
        if geometry == "auto":
            assert L["general_camera"] == 0, name
    assert_driver_parity(g, o, dict(p=d, name=name, eps=1e-6))
    dt, dr = synth.pose_error(g["T"], o["T"])
    _measure("sparse_img_align_pose", max(dt, dr))


# ---- streams ------------------------------------------------------------------------------------------------------------
STREAM_CAMS = ["atan", "atan_s0", "atan_s_neg", "pinhole_d0_zero", "pinhole_d0_next", "pinhole_barrel", "pinhole_aniso"]


def test_depth_streams_of_edge_cameras_equal_single_calls(ctx):
    scenes = [cc.depth_scene(n) for n in STREAM_CAMS]
    frames, kf_tab, kf_T, streams, singles = [], [], [], [], []
    for j, c in enumerate(scenes):
        kf, cur = ctx.frame(c["ref_pyr"]), ctx.frame(c["cur_pyr"])
        frames += [kf, cur]
        kf_tab.append(kf)
        kf_T.append(c["T_ref_w"])
        args = dict(ftr_px=c["ftr_px"], ftr_f=c["ftr_f"], ftr_level=c["ftr_level"], ftr_type=c["ftr_type"],
                    ftr_grad=c["ftr_grad"], batch_id=c["batch_id"], seeds=c["seeds"])
        singles.append(ctx.depth_filter_update([kf], [c["T_ref_w"]], cur, c["T_cur_w"], c["cam"], c["ref_index"],
                                               args["ftr_px"], args["ftr_f"], args["ftr_level"], args["ftr_type"],
                                               args["ftr_grad"], args["batch_id"], 6, args["seeds"]))
        streams.append(dict(cur=cur, cur_T_f_w=c["T_cur_w"], cam=c["cam"], batch_counter=6,
                            ref_index=np.full(c["M"], j, np.int32), **args))
    batched = ctx.depth_filter_update_streams(streams, kf_tab, kf_T)
    for f in frames:
        f.destroy()
    for s, (g, b) in enumerate(zip(singles, batched)):
        for k in SEED_KEYS:
            assert _same_bits(g[k], b[k]), (STREAM_CAMS[s], k)


def test_reproject_streams_of_edge_cameras_equal_single_calls(ctx):
    scenes = [cc.map_scene(n) for n in STREAM_CAMS]
    frames, streams = [], []
    for c in scenes:
        kfs, cur = [ctx.frame(p) for p in c["kf_pyr"]], ctx.frame(c["cur_pyr"])
        frames += kfs + [cur]
        streams.append(_reproject_args(c, kfs, cur))
    singles = [ctx.reproject_map(**s) for s in streams]
    batched = ctx.reproject_map_streams(streams)
    for f in frames:
        f.destroy()
    for s, (g, b) in enumerate(zip(singles, batched)):
        for k in RP_KEYS:
            if isinstance(g[k], np.ndarray):
                assert _same_bits(g[k], b[k]), (STREAM_CAMS[s], k)
            else:
                assert g[k] == b[k], (STREAM_CAMS[s], k)


# ---- a camera whose size is not its frames' -----------------------------------------------------------------------------
def test_match_and_alignment_refuse_a_camera_of_another_size(ctx):
    """find_match_direct, sparse_img_align, sia_batch_stage and sparse_residuals return SVO_B200_EINVAL, launch nothing and
    write nothing (the other camera-taking entry points: tests/test_streams_gpu.py's refusal tests).  The smaller cameras
    come first: a library without the check accepts them and fails here before it is handed a larger one."""
    for dw, dh in SIZE_OFFSETS:
        _refused(ctx, dw, dh)


def _refused(ctx, dw, dh):
    c = cc.match_scene("pinhole_radtan")
    bad = capi.cam_struct(_resized(c["cam"], dw, dh))
    ref, cur = ctx.frame(c["ref_pyr"]), ctx.frame(c["cur_pyr"])
    M = 4
    ri, lv, ty = np.zeros(M, np.int32), np.zeros(M, np.int32), np.zeros(M, np.int32)
    rpx, rf, rg, pp = [np.ascontiguousarray(c[k][:M], np.float64) for k in ("ref_px", "ref_f", "ref_grad", "point_pos")]
    refT, curT = c["T_ref_w"].reshape(12).copy(), c["T_cur_w"].reshape(12).copy()
    px, succ, sl, A, hinv = np.full((M, 2), 7.0), np.full(M, 77, np.uint8), np.full(M, 77, np.int32), np.full((M, 4), 7.0), np.full(M, 7.0)
    ra = (C.c_void_p * 1)(ref.h.value)
    n0 = ctx.launch_count()
    rc = ctx.lib.svo_b200_find_match_direct(ctx.h, ra, capi._p(refT), 1, cur.h, capi._p(curT), C.byref(bad),
                                            C.byref(capi.MatchOptions(2, 10)), M, capi._p(ri), capi._p(rpx), capi._p(rf),
                                            capi._p(lv), capi._p(ty), capi._p(rg), capi._p(pp), capi._p(px), capi._p(succ),
                                            capi._p(sl), capi._p(A), capi._p(hinv))
    assert rc == -1 and ctx.launch_count() == n0
    assert np.all(px == 7.0) and np.all(succ == 77) and np.all(sl == 77) and np.all(A == 7.0) and np.all(hinv == 7.0)
    assert b"camera" in ctx.lib.svo_b200_last_error(ctx.h)
    # alignment: one pair, the same frames
    d = synth.make_frame_pair(906, width=cc.W, height=cc.H, n_feat=40, n_levels=5, cam=c["cam"])
    N = len(d["px"])
    T = synth.se3_identity().reshape(12).copy()
    vis, H, trace = np.full(N, 77, np.uint8), np.full(36, 7.0), (capi.SiaIter * 8)()
    st, ntr = capi.SiaStats(), C.c_int(77)
    st.n_tracked = 77
    pxa, fa, pa, rp = (np.ascontiguousarray(d[k], np.float64) for k in ("px", "f", "pos", "ref_pos"))
    hpa = np.ascontiguousarray(d["has_point"], np.uint8)
    rc = ctx.lib.svo_b200_sparse_img_align(ctx.h, ref.h, cur.h, C.byref(bad), C.byref(capi.SiaOptions(4, 0, 30, 1e-6)),
                                           capi._p(T), capi._p(pxa), capi._p(fa), capi._p(pa), capi._p(hpa), capi._p(rp), N,
                                           capi._p(vis), capi._p(H), C.byref(st), trace, 8, C.byref(ntr))
    assert rc == -1 and ctx.launch_count() == n0
    assert _same_bits(T, synth.se3_identity().reshape(12)) and np.all(vis == 77) and np.all(H == 7.0)
    assert st.n_tracked == 77 and ntr.value == 77
    fo = np.array([0, N], np.int32)
    rc = ctx.lib.svo_b200_sia_batch_stage(ctx.h, 1, ra, (C.c_void_p * 1)(cur.h.value), C.byref(bad),
                                          C.byref(capi.SiaOptions(4, 0, 30, 1e-6)), capi._p(T), capi._p(fo), capi._p(pxa),
                                          capi._p(fa), capi._p(pa), capi._p(hpa), capi._p(rp))
    assert rc == -1 and ctx.lib.svo_b200_sia_batch_run(ctx.h) == -1 and ctx.launch_count() == n0  # nothing staged
    ref_patch, res, inimg = np.full((N, 16), 7.0, np.float32), np.full((N, 16), 7.0, np.float32), np.full(N, 77, np.uint8)
    Jres, chi2, nm = np.full(6, 7.0), C.c_double(7.0), C.c_int64(77)
    rc = ctx.lib.svo_b200_sparse_residuals(ctx.h, ref.h, cur.h, C.byref(bad), 0, capi._p(T), capi._p(pxa), capi._p(fa),
                                           capi._p(pa), capi._p(hpa), capi._p(rp), N, capi._p(vis), capi._p(ref_patch),
                                           capi._p(res), capi._p(inimg), capi._p(H), capi._p(Jres), C.byref(chi2), C.byref(nm))
    assert rc == -1 and ctx.launch_count() == n0
    assert np.all(vis == 77) and np.all(ref_patch == 7.0) and np.all(res == 7.0) and np.all(inimg == 77)
    assert np.all(H == 7.0) and np.all(Jres == 7.0) and chi2.value == 7.0 and nm.value == 77
    ref.destroy(); cur.destroy()
