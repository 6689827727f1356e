"""A catalogue of cameras and inputs that reach every branch of vikit's world2cam / cam2world on both sides of its
threshold, for the tests of the oracle (tests/test_camera_edges_pins.py) and of the device code of every projecting kernel
(tests/test_camera_edges_gpu.py).  The branch each input takes is the one the exactly rounded statement
(tests/camera_hp.py) says it takes; the inputs next to a threshold are found by searching the statement.

Cameras: the two the reference ships; ATAN with s = 0 (world2cam then takes the plain branch, cam2world the ATAN one with
r = dist_r), s = 1e-4 and a negative s; pinhole without distortion, with d0 = 0 but d1..d4 != 0 (vikit ignores them), with
|d0| = 1e-7 (undistorted) and the next double above (distorted), with k3 != 0, with a barrel distortion strong enough
that OpenCV's 5 undistortion iterations leave 8 px at the corners, with the tangential terms dominant; fx != fy by 20 %
and a principal point off centre and off the pixel grid, for both models.  All are 752 x 480."""
from __future__ import annotations

import math
from functools import lru_cache

import numpy as np

from rpg_svo_b200 import synth
from tests import camera_hp as hp

W, H = 752, 480
_RADTAN = synth.reference_param_camera("pinhole_radtan")
_ATAN = synth.reference_param_camera("atan")
_NEXT_1E7 = float(np.nextafter(1e-7, 1.0))


def _pin(d, fx=_RADTAN.fx, fy=_RADTAN.fy, cx=_RADTAN.cx, cy=_RADTAN.cy):
    return synth.Camera(fx, fy, cx, cy, W, H, 0, tuple(float(v) for v in d))


def _atan(s, fx=0.509326, fy=0.796651, cx=0.45905, cy=0.510056):
    return synth.atan_camera(W, H, fx, fy, cx, cy, s)


CAMERAS = {
    "atan": _ATAN,
    "pinhole_radtan": _RADTAN,
    "atan_s0": _atan(0.0),
    "atan_s1e-4": _atan(1e-4),
    "atan_s_neg": _atan(-0.7),
    "atan_aniso": _atan(0.932, fx=0.509326, fy=0.509326 * 1.2 * W / H, cx=0.43171, cy=0.53713),
    "pinhole_plain": _pin((0.0, 0.0, 0.0, 0.0, 0.0)),
    "pinhole_d0_zero": _pin((0.0, 0.066674, 0.000896, 0.000778, 0.01)),
    "pinhole_d0_1e-7": _pin((1e-7, 0.066674, 0.000896, 0.000778, 0.0)),
    "pinhole_d0_-1e-7": _pin((-1e-7, 0.066674, 0.000896, 0.000778, 0.0)),
    "pinhole_d0_next": _pin((_NEXT_1E7, 0.066674, 0.000896, 0.000778, 0.0)),
    "pinhole_d0_-next": _pin((-_NEXT_1E7, 0.066674, 0.000896, 0.000778, 0.0)),
    "pinhole_k3": _pin((-0.283076, 0.066674, 0.000896, 0.000778, 0.045)),
    "pinhole_barrel": _pin((-0.34, 0.12, 0.0, 0.0, 0.0)),
    "pinhole_tangential": _pin((2e-6, 0.0, 0.02, -0.015, 0.0)),
    "pinhole_aniso": _pin((-0.283076, 0.066674, 0.000896, 0.000778, 0.0), fx=414.536145, fy=414.536145 * 1.2,
                          cx=361.3172, cy=228.6841),
}
ATAN_CAMERAS = [k for k, c in CAMERAS.items() if c.model == 1]


def general(cam) -> bool:
    """Not the plain pinhole: the alignment kernel's general-camera instantiation (pinhole with |d0| > 1e-7, or ATAN)."""
    return cam.model == 1 or abs(cam.d[0]) > 1e-7


def _ulps(v: float, k: int) -> float:
    return hp._step(v, k)


# ---- unit-plane points (world2cam) --------------------------------------------------------------------------------------
def _r_of(x: float, y: float) -> float:
    """The statement's r = sqrt(fma(x, x, y * y))."""
    A = hp.IEEE
    return A.sqrt(A.fma(x, x, A.mul(y, y)))


@lru_cache(maxsize=None)
def r_threshold_points():
    """Unit-plane points (x, y) on a diagonal whose statement r is 0.001's lower neighbour, 0.001 and its upper neighbour,
    found by walking x one double at a time (one step moves r by less than an ulp of r, so every value is met)."""
    targets = {_ulps(0.001, -1): "below", 0.001: "at", _ulps(0.001, 1): "above"}
    y = 0.0006
    x0 = 0.0008
    found = {}
    for k in range(-64, 65):
        x = _ulps(x0, k)
        r = _r_of(x, y)
        if r in targets and targets[r] not in found:
            found[targets[r]] = (x, y)
    assert set(found) == {"below", "at", "above"}, found
    return found


def unit_plane_inputs(cam):
    """(label, xyz) inputs of world2cam: r = 0 (both zero signs), r at 0.001 and its neighbouring doubles, on the axis
    too, the bearings of the image corners and centre, ordinary points at several depths, points behind the camera,
    z = 0 and non-finite coordinates."""
    out = [("r0", (0.0, 0.0, 1.0)), ("r0_neg_zero", (-0.0, 0.0, 1.0)), ("r0_far", (0.0, 0.0, 7.5))]
    for side, (x, y) in r_threshold_points().items():
        out.append((f"r_{side}_0.001", (x, y, 1.0)))
        out.append((f"r_{side}_0.001_neg", (-x, -y, 1.0)))
    out += [("axis_0.001", (0.001, 0.0, 1.0)), ("axis_below_0.001", (_ulps(0.001, -1), 0.0, 1.0)),
            ("axis_y_0.001", (0.0, -0.001, 1.0))]
    corners = [(0.0, 0.0), (W - 1.0, 0.0), (0.0, H - 1.0), (W - 1.0, H - 1.0), (W / 2, H / 2), (cam.cx, cam.cy)]
    for j, f in enumerate(cam.cam2world_exact(np.array(corners))):
        for z in (1.0, 3.7):
            out.append((f"corner{j}_z{z}", tuple(float(v) for v in f * (z / f[2]))))
    rng = np.random.default_rng(11)
    for j in range(12):
        x, y = rng.uniform(-0.8, 0.8), rng.uniform(-0.55, 0.55)
        out.append((f"interior{j}", (x * 2.5, y * 2.5, 2.5)))
    out += [("behind", (0.1, -0.2, -1.0)), ("behind_axis", (0.0, 0.0, -2.0)), ("z0", (0.1, 0.2, 0.0)), ("z0_origin", (0.0, 0.0, 0.0)),
            ("z_neg0", (0.1, 0.2, -0.0)), ("nan_x", (math.nan, 0.1, 1.0)), ("nan_z", (0.1, 0.1, math.nan)),
            ("inf_x", (math.inf, 0.1, 1.0)), ("inf_z", (0.1, 0.1, math.inf)), ("far_off", (3.0, -2.0, 1.0)),
            ("huge", (1e200, 1e200, 1e-200))]
    return out


# ---- pixels (cam2world) -------------------------------------------------------------------------------------------------
@lru_cache(maxsize=None)
def dist_r_threshold_pixels(name):
    """Pixels whose statement dist_r is 0.01's lower neighbour, 0.01 and its upper neighbour: one step of u or v moves
    dist_r by ~70 of its ulps, so both are walked together (IEEE double in numpy, no fma in that expression) and the hits
    confirmed on the statement."""
    c = hp.cam_const(CAMERAS[name])
    k = np.arange(-600, 601)
    found = {}
    for t, side in ((_ulps(0.01, -1), "below"), (0.01, "at"), (_ulps(0.01, 1), "above")):
        for ang in np.arange(0.5, 1.3, 0.05):  # another direction where one has no hit
            u0, v0 = c.cx + 0.01 * math.cos(ang) * c.fx, c.cy + 0.01 * math.sin(ang) * c.fy
            us = u0 + k * np.spacing(u0)  # whole ulps of u0 / v0, exactly (both stay in one binade)
            vs = v0 + k * np.spacing(v0)
            dx = (us - c.cx) * c.fx_inv
            dy = (vs - c.cy) * c.fy_inv
            hits = np.argwhere(np.sqrt(dx[:, None] * dx[:, None] + dy[None, :] * dy[None, :]) == t)
            if len(hits):
                break
        i, j = hits[0]
        px = (float(us[i]), float(vs[j]))
        A = hp.IEEE
        dxs, dys = A.mul(A.sub(px[0], c.cx), c.fx_inv), A.mul(A.sub(px[1], c.cy), c.fy_inv)
        assert A.sqrt(A.add(A.mul(dxs, dxs), A.mul(dys, dys))) == t
        found[side] = px
    return found


def pixel_inputs(name):
    """(label, (u, v)) inputs of cam2world: the principal point (dist_r = 0), pixels at dist_r = 0.01 and its
    neighbouring doubles, float-rounding ties and their neighbours (cv::undistortPoints rounds the pixel to float), the
    image corners and centre, integer and sub-pixel interior pixels, far-off and non-finite pixels."""
    cam = CAMERAS[name]
    out = [("principal", (cam.cx, cam.cy)), ("principal_u", (cam.cx, 100.0)), ("principal_v", (100.0, cam.cy))]
    for side, px in dist_r_threshold_pixels(name).items():
        out.append((f"dist_r_{side}_0.01", px))
    tie_u, tie_v = 300.0 + 2.0 ** -16, 200.0 + 2.0 ** -17 * 3  # halfway between two floats (ulp 2^-15 at 300, 2^-16 at 200)
    for k in (-1, 0, 1):
        out.append((f"f32_tie{k:+d}", (_ulps(tie_u, k), _ulps(tie_v, k))))
    out += [("f32_inexact", (377.3, 239.7)), ("f32_inexact_corner", (750.9, 1.1))]
    for j, px in enumerate([(0.0, 0.0), (W - 1.0, 0.0), (0.0, H - 1.0), (W - 1.0, H - 1.0), (W, H), (-0.5, -0.5),
                            (W / 2, H / 2)]):
        out.append((f"corner{j}", px))
    rng = np.random.default_rng(12)
    for j in range(10):
        out.append((f"interior{j}", (float(rng.uniform(5, W - 5)), float(rng.uniform(5, H - 5)))))
    out += [("far_off", (-1000.0, 5000.0)), ("nan_u", (math.nan, 100.0)), ("inf_u", (math.inf, 100.0)),
            ("ninf", (-math.inf, -math.inf)), ("huge", (1e300, -1e300))]
    return out


# ---- kernel scenes ------------------------------------------------------------------------------------------------------
@lru_cache(maxsize=None)
def two_view(name):
    """Keyframe and current frame of a textured plane seen by the camera (5 levels, 0.15 m baseline)."""
    return synth.make_two_view(900, cam=CAMERAS[name], baseline=0.15, n_levels=5)


def match_scene(name):
    """findMatchDirect candidates: 48 ordinary features, plus features whose ref_px + (5 2^L, 0) or + (0, 5 2^L) -- the
    pixels getWarpMatrixAffine unprojects -- lands on each dist_r = 0.01 pixel (ATAN's cam2world switch) or on the
    principal point, for L = 0, 1, 2, and features on the float-rounding ties."""
    tv = two_view(name)
    cam = tv["cam"]
    rng = np.random.default_rng(901)
    px, lv = [], []
    for _ in range(48):
        L = int(rng.integers(0, 3))
        px.append((float(rng.uniform(40, W - 40)), float(rng.uniform(40, H - 40))))
        lv.append(L)
    targets = list(dist_r_threshold_pixels(name).values()) + [(cam.cx, cam.cy)]
    for L in range(3):
        h = 5.0 * (1 << L)
        for u, v in targets:
            px += [(u - h, v), (u, v - h), (u, v)]
            lv += [L, L, L]
    for label, p in pixel_inputs(name):
        if label.startswith("f32_tie"):
            px.append(p)
            lv.append(0)
    px, lv = np.array(px), np.array(lv, np.int32)
    f = cam.cam2world(px)
    pos = synth.intersect(tv["plane"], tv["T_ref_w"], f)
    Tc = tv["T_cur_w"]
    px_cur = cam.world2cam(pos @ Tc[:, :3].T + Tc[:, 3]) + rng.uniform(-1.5, 1.5, (len(px), 2))
    ang = rng.uniform(0, 2 * np.pi, len(px))
    return dict(tv, M=len(px), ref_px=px, ref_f=f, ref_level=lv, ftr_type=(np.arange(len(px)) % 7 == 3).astype(np.int32),
                ref_grad=np.stack([np.cos(ang), np.sin(ang)], axis=1), point_pos=pos, px_cur=px_cur)


def depth_scene(name, n_random=120):
    """Depth-filter seeds of the two-view scene: random integer features, and features whose epipolar segment in the
    current frame crosses the optical axis (the keyframe pixel of a point on the current frame's principal ray at the
    seed's mean depth), at several depths and levels."""
    tv = two_view(name)
    cam = tv["cam"]
    rng = np.random.default_rng(902)
    px = np.floor(synth.jittered_features(rng, cam, n_random, margin=10.0))
    T_r, T_c = tv["T_ref_w"], tv["T_cur_w"]
    Tc_inv = synth.se3_inv(T_c)
    axis = []
    for d in (1.6, 2.0, 2.4):
        for du, dv in ((0.0, 0.0), (0.7, -0.4), (-3.0, 2.0)):
            b = cam.cam2world_exact(np.array([[cam.cx + du, cam.cy + dv]]))[0]
            pw = Tc_inv[:, :3] @ (b * d / b[2]) + Tc_inv[:, 3]
            axis.append(cam.world2cam(T_r[:, :3] @ pw + T_r[:, 3]))
    px = np.concatenate([px, np.array(axis)])
    n = len(px)
    level = np.concatenate([rng.integers(0, 3, n_random), np.arange(len(axis)) % 3]).astype(np.int32)
    f = cam.cam2world(px)
    ang = rng.uniform(0, 2 * np.pi, n)
    mu = np.full(n, np.float32(0.5))
    mu[n_random:] = (1.0 / np.repeat([1.6, 2.0, 2.4], 3)).astype(np.float32)
    zr = np.float32(2.0)
    seeds = dict(a=np.full(n, 10, np.float32), b=np.full(n, 10, np.float32), mu=mu, z_range=np.full(n, zr, np.float32),
                 sigma2=np.full(n, zr * zr / np.float32(36), np.float32))
    return dict(tv, M=n, ftr_px=px, ftr_f=f, ftr_level=level, ftr_type=(np.arange(n) % 9 == 4).astype(np.int32),
                ftr_grad=np.stack([np.cos(ang), np.sin(ang)], axis=1), seeds=seeds, batch_id=np.full(n, 5, np.int32),
                batch_counter=6, ref_index=np.zeros(n, np.int32), n_axis=len(axis))


@lru_cache(maxsize=None)
def map_scene(name):
    """A small map for reprojectMap whose points include ones that reproject next to u = 8 and u = width - 8 (the
    isInFrame(px, 8) border) in the current frame, 1e-11 to 1e-6 px to either side.  Not closer: a point on the border
    itself is a tie the camera model leaves open (ATAN's atan is allowed 2 ulp, which moves u by up to ~3e-13 px, and
    the pose product's last bits move it by ~1e-13 px).  `border`: (point, border u, offset)."""
    c = synth.make_map_case(903, n_kfs=3, n_points=160, n_candidates=20, cam=CAMERAS[name])
    cam, T = c["cam"], c["cur_T_f_w"]
    Tinv = synth.se3_inv(T)
    v = dict(c["view"])
    pos = v["pt_pos"].copy()
    rng = np.random.default_rng(904)
    k, border = 0, []
    for u in (8.0, W - 8.0):
        for off in (-1e-6, -1e-9, -1e-11, 1e-11, 1e-9, 1e-6):
            for vv in (100.0, 300.0):
                b = cam.cam2world_exact(np.array([[u + off, vv]]))[0]
                pc = b * (2.0 / b[2])
                pos[k] = Tinv[:, :3] @ pc + Tinv[:, 3]
                border.append((k, u, off))
                k += 2 + int(rng.integers(0, 3))
    v["pt_pos"] = pos
    c["view"] = v
    c["border"] = border
    return c
