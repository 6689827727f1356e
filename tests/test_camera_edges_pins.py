"""CPU: the oracle's camera functions bit for bit against the exactly rounded statement of tests/camera_hp.py (with
glibc's atan / tan, which the oracle calls) on every camera and input of tests/camera_cases.py; the catalogue reaches
every branch on both sides of its threshold; and the statement itself against a 40-digit evaluation of the same formulas
away from the branch points."""
import math

import numpy as np
import pytest

from tests import camera_cases as cc
from tests import camera_hp as hp
from tests.ref_golden import ref  # noqa: F401 (fixture)

CAMS = list(cc.CAMERAS)


def _oracle_rows(oracle, name):
    cam = cc.CAMERAS[name]
    w_in = cc.unit_plane_inputs(cam)
    p_in = cc.pixel_inputs(name)
    with np.errstate(all="ignore"):
        uv = oracle.camera_world2cam(cam, np.array([x for _, x in w_in]))
        f = oracle.camera_cam2world(cam, np.array([p for _, p in p_in]))
    return w_in, uv, p_in, f


@pytest.mark.parametrize("name", CAMS)
def test_oracle_camera_equals_statement(oracle, name):
    c = hp.cam_const(cc.CAMERAS[name])
    w_in, uv, p_in, f = _oracle_rows(oracle, name)
    for (label, xyz), got in zip(w_in, uv):
        want = hp.world2cam(c, xyz)
        assert hp.same_tuple(got, want[:2]), (name, label, tuple(got), want)
    for (label, px), got in zip(p_in, f):
        want = hp.cam2world(c, px[0], px[1])
        assert hp.same_tuple(got, want[:3]), (name, label, tuple(got), want)


def test_catalogue_reaches_every_branch_on_both_sides():
    w_br, c_br = {}, {}
    for name, cam in cc.CAMERAS.items():
        c = hp.cam_const(cam)
        for label, xyz in cc.unit_plane_inputs(cam):
            w_br.setdefault(hp.world2cam(c, xyz)[2], set()).add((name, label))
        for label, px in cc.pixel_inputs(name):
            c_br.setdefault(hp.cam2world(c, *px)[3], set()).add((name, label))
    assert set(w_br) == {"plain", "radtan", "atan_small", "atan"}, set(w_br)
    assert set(c_br) == {"pinhole", "radtan", "atan_inner", "atan", "atan_inner_s0", "atan_s0"}, set(c_br)
    # r < 0.001 (world2cam, ATAN): 0.001's lower neighbour is inside, 0.001 itself and its upper neighbour are not
    for name in cc.ATAN_CAMERAS:
        if name == "atan_s0":
            continue
        for side, want in (("below", "atan_small"), ("at", "atan"), ("above", "atan")):
            assert (name, f"r_{side}_0.001") in w_br[want], (name, side)
        assert (name, "r0") in w_br["atan_small"]
    # dist_r > 0.01 (cam2world, ATAN): 0.01 and its lower neighbour take d_factor = 1, the upper neighbour r / dist_r
    for name in cc.ATAN_CAMERAS:
        sfx = "_s0" if name == "atan_s0" else ""
        for side, want in (("below", "atan_inner"), ("at", "atan_inner"), ("above", "atan")):
            assert (name, f"dist_r_{side}_0.01") in c_br[want + sfx], (name, side)
        assert (name, "principal") in c_br["atan_inner" + sfx]
    # |d0| > 1e-7 (pinhole): d0 = 0 with d1..d4 != 0 and |d0| = 1e-7 are undistorted, the next double above is distorted
    for name in ("pinhole_plain", "pinhole_d0_zero", "pinhole_d0_1e-7", "pinhole_d0_-1e-7"):
        assert not hp.cam_const(cc.CAMERAS[name]).distorted and not cc.general(cc.CAMERAS[name]), name
    for name in ("pinhole_d0_next", "pinhole_d0_-next", "pinhole_k3", "pinhole_barrel", "pinhole_tangential"):
        assert hp.cam_const(cc.CAMERAS[name]).distorted and cc.general(cc.CAMERAS[name]), name
    # ATAN with s = 0: world2cam takes the plain branch, cam2world the ATAN one
    assert ("atan_s0", "corner0_z1.0") in w_br["plain"] and ("atan_s0", "corner0") in c_br["atan_s0"]


def test_catalogue_cameras_do_what_they_say():
    """The barrel camera leaves at least 1 px at the corners after OpenCV's 5 undistortion iterations (its exact inverse
    converges), the k3 camera's r^6 term moves the corners by more than a pixel, the tangential camera's tangential
    displacement exceeds its radial one, and the float rounding of the pixel moves the undistortion."""
    corners = np.array([[0.0, 0.0], [cc.W - 1.0, 0.0], [0.0, cc.H - 1.0], [cc.W - 1.0, cc.H - 1.0]])
    barrel = cc.CAMERAS["pinhole_barrel"]
    assert np.max(np.abs(barrel.world2cam(barrel.cam2world(corners)) - corners)) >= 1.0
    assert np.max(np.abs(barrel.world2cam(barrel.cam2world_exact(corners)) - corners)) < 1e-6
    k3, no_k3 = cc.CAMERAS["pinhole_k3"], cc.CAMERAS["pinhole_radtan"]
    f = no_k3.cam2world_exact(corners)
    assert np.min(np.abs(k3.world2cam(f) - no_k3.world2cam(f))) > 1.0
    t = hp.cam_const(cc.CAMERAS["pinhole_tangential"])
    x, y = 0.6, 0.4
    r2 = x * x + y * y
    assert abs(2 * t.d[2] * x * y + t.d[3] * (r2 + 2 * x * x)) > 10 * abs(x * (t.d[0] * r2 + t.d[1] * r2 * r2))
    c = hp.cam_const(no_k3)
    ties = [px for label, px in cc.pixel_inputs("pinhole_radtan") if label.startswith("f32_tie")]
    outs = {hp.cam2world(c, *px)[:3] for px in ties}
    assert len(outs) >= 2  # neighbouring doubles round to different floats


def _tol(exact, scale, n_ulp):
    return n_ulp * math.ulp(max(abs(float(exact)), scale))


@pytest.mark.parametrize("name", CAMS)
def test_statement_vs_40_digits(name):
    """Away from the branch points (r within 1e-15 of 0.001, dist_r of 0.01) and from overflow, and for finite results,
    the statement lies within 8 ulps (of the largest term: |cx| for u, 1 for a bearing) of the unrounded formulas;
    radial-tangential undistortion ends in a float cast, so there within 2 float ulps."""
    cam = cc.CAMERAS[name]
    c = hp.cam_const(cam)
    n_checked = 0
    for label, xyz in cc.unit_plane_inputs(cam):
        got = hp.world2cam(c, xyz)
        if not all(math.isfinite(v) for v in got[:2]) or xyz[2] == 0 or max(abs(xyz[0]), abs(xyz[1])) > 1e100 * abs(xyz[2]):
            continue
        ex = hp.world2cam(c, xyz, hp.mp.atan, hp.Exact)
        x, y = xyz[0] / hp.mpf(xyz[2]), xyz[1] / hp.mpf(xyz[2])
        if c.model == hp.ATAN and c.distorted and abs(hp.mp.sqrt(x * x + y * y) - 0.001) < 1e-15:
            continue
        assert got[2] == ex[2], (label, got, ex)
        for g, e, s in ((got[0], ex[0], abs(c.cx)), (got[1], ex[1], abs(c.cy))):
            assert abs(g - e) <= _tol(e, s, 8), (label, g, float(e))
        n_checked += 1
    for label, px in cc.pixel_inputs(name):
        got = hp.cam2world(c, *px)
        if not all(math.isfinite(v) for v in got[:3]) or max(abs(px[0]), abs(px[1])) > 1e100:  # overflow inside
            continue
        ex = hp.cam2world(c, px[0], px[1], hp.mp.tan, hp.Exact)
        if c.model == hp.ATAN:
            dx, dy = (hp.mpf(px[0]) - c.cx) * c.fx_inv, (hp.mpf(px[1]) - c.cy) * c.fy_inv
            if abs(hp.mp.sqrt(dx * dx + dy * dy) - 0.01) < 1e-15:
                continue
        assert got[3] == ex[3], (label, got, ex)
        for g, e in zip(got[:3], ex[:3]):
            tol = 2 * 2.0 ** -23 * max(abs(float(e)), 1e-3) if got[3] == "radtan" else _tol(e, 1.0, 8)
            assert abs(g - e) <= tol, (label, g, float(e))
        n_checked += 1
    assert n_checked > 40


# The reference's own Matcher::findMatchDirect (oracle/_ref: svo/src/matcher.cpp over the shim's restated vikit cameras,
# built with GCC's contraction) against the oracle on the edge scenes: success, search level and the matched pixel exact;
# A_cur_ref within 1e-12 (the largest difference recorded over the 16 cameras is 6.8e-14: GCC contracts the pose product
# and the warp's differences into FMAs, the oracle does not).
REF_A_TOL = 1e-12


@pytest.mark.parametrize("name", CAMS)
def test_reference_find_match_direct_on_camera_edges(oracle, ref, name):
    c = cc.match_scene(name)
    cam = c["cam"]
    T_cur_ref = oracle.se3_mul(c["T_cur_w"], oracle.se3_inv(c["T_ref_w"]))
    ref_pos = oracle.se3_inv(c["T_ref_w"])[:, 3]
    dA = dpx = 0.0
    n_ok = 0
    for i in range(c["M"]):
        r = ref.matcher(0, c["ref_pyr"][0], c["cur_pyr"][0], c["n_levels"], cam, c["T_ref_w"], c["T_cur_w"], c["ref_px"][i],
                        c["ref_f"][i], int(c["ref_level"][i]), int(c["ftr_type"][i]), c["ref_grad"][i], c["point_pos"][i],
                        px_cur=c["px_cur"][i], n_pyr_levels=3)
        o = oracle.find_match_direct(c["ref_pyr"], c["cur_pyr"], cam, T_cur_ref, c["ref_px"][i], c["ref_f"][i],
                                     int(c["ref_level"][i]), int(c["ftr_type"][i]), c["ref_grad"][i],
                                     np.linalg.norm(c["point_pos"][i] - ref_pos), 2, 10, c["px_cur"][i])
        assert bool(r["success"]) == bool(o["success"]) and r["search_level"] == o["search_level"], (name, i)
        dA = max(dA, float(np.max(np.abs(np.asarray(r["A_cur_ref"]).ravel() - np.asarray(o["A_cur_ref"]).ravel()))))
        if r["success"]:
            n_ok += 1
            dpx = max(dpx, float(np.max(np.abs(np.asarray(r["px_cur"]) - o["px_cur"]))))
    print(f"{name}: reference vs oracle |dA| {dA:.3g}, |dpx| {dpx:.3g}")
    assert dA <= REF_A_TOL and dpx == 0.0, (name, dA, dpx)
    assert n_ok > c["M"] // 3, (name, n_ok)


@pytest.mark.parametrize("name", CAMS)
def test_map_scene_reaches_both_sides_of_the_reprojection_border(name):
    """isInFrame(px.cast<int>(), 8) in the current frame: for each border (u = 8, u = width - 8) the map has points on
    both sides, and every candidate u of the statement (the pose product in double, atan within 2 ulp) is at least 5e-12
    px from the border, so the kernel and the oracle must decide each the same way."""
    c = cc.map_scene(name)
    cam, T = c["cam"], c["cur_T_f_w"]
    k = hp.cam_const(cam)
    sides = {}
    for p, u, off in c["border"]:
        xyz = T[:, :3] @ c["view"]["pt_pos"][p] + T[:, 3]
        us = [r[0] for _, r in hp.world2cam_candidates(k, tuple(float(v) for v in xyz))]
        assert min(abs(x - u) for x in us) >= 5e-12, (name, p, u, off, us)
        inside = {(8 <= int(x) < cc.W - 8) for x in us}
        assert len(inside) == 1, (name, p, us)
        sides.setdefault(u, set()).add(inside.pop())
    assert sides == {8.0: {False, True}, cc.W - 8.0: {False, True}}, (name, sides)
