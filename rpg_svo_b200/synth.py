"""Seeded synthetic inputs for the direct-tracking hot path (SURVEY.md section 8d).

A textured plane seen by a pinhole camera: both images of a frame-pair are rendered from the same
float texture through the exact ray/plane geometry, so the ground-truth relative pose is known.
Nothing here is part of the measured path; it only manufactures inputs of the shapes BASELINE.json
names (there is no dataset: the reference's `sin2_tex2_h1_v8_d` cannot be downloaded).

Conventions: SE3 as 3x4 row-major [R|t] float64 arrays; `T_f_w` maps world -> frame like the
reference's `Frame::T_f_w_` (svo/include/svo/frame.h:51).
"""
from __future__ import annotations

from dataclasses import dataclass
from functools import lru_cache

import numpy as np


@dataclass(frozen=True)
class Camera:
    """[EXT] vk::AbstractCamera: model 0 = vk::PinholeCamera (d = k1 k2 p1 p2 k3, radial-tangential; all zero = no
    distortion), model 1 = vk::ATANCamera (d[0] = s; fx.. are the pixel values the vikit constructor derives).
    numpy restatement used to manufacture test data (features, renders)."""

    fx: float
    fy: float
    cx: float
    cy: float
    width: int
    height: int
    model: int = 0
    d: tuple = (0.0, 0.0, 0.0, 0.0, 0.0)

    @property
    def distorted(self) -> bool:
        return abs(self.d[0]) > 1e-7 if self.model == 0 else self.d[0] != 0.0

    def cam2world(self, px: np.ndarray) -> np.ndarray:
        """Pixel -> unit bearing vector (normalised), rows of px are (u, v)."""
        px = np.asarray(px, dtype=np.float64)
        u, v = px[..., 0], px[..., 1]
        if self.model == 0 and not self.distorted:
            x, y = (u - self.cx) / self.fx, (v - self.cy) / self.fy
        elif self.model == 0:  # cv::undistortPoints on a CV_32FC2 point: float in, 5 iterations, float out
            k = self.d
            uf, vf = u.astype(np.float32).astype(np.float64), v.astype(np.float32).astype(np.float64)
            x0, y0 = (uf - self.cx) * (1.0 / self.fx), (vf - self.cy) * (1.0 / self.fy)
            x, y = x0.copy(), y0.copy()
            for _ in range(5):
                r2 = x * x + y * y
                icdist = 1.0 / (1.0 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
                dX = 2.0 * k[2] * x * y + k[3] * (r2 + 2.0 * x * x)
                dY = k[2] * (r2 + 2.0 * y * y) + 2.0 * k[3] * x * y
                x, y = (x0 - dX) * icdist, (y0 - dY) * icdist
            x, y = x.astype(np.float32).astype(np.float64), y.astype(np.float32).astype(np.float64)
        else:
            dx, dy = (u - self.cx) * (1.0 / self.fx), (v - self.cy) * (1.0 / self.fy)
            dist_r = np.sqrt(dx * dx + dy * dy)
            s = self.d[0]
            r = np.tan(dist_r * s) / (2.0 * np.tan(s / 2.0)) if s != 0.0 else dist_r
            fac = np.where(dist_r > 0.01, r / np.where(dist_r > 0, dist_r, 1.0), 1.0)
            x, y = fac * dx, fac * dy
        xyz = np.stack([x, y, np.ones(px.shape[:-1])], axis=-1)
        return xyz / np.linalg.norm(xyz, axis=-1, keepdims=True)

    def cam2world_exact(self, px: np.ndarray) -> np.ndarray:
        """True inverse of world2cam (for rendering): the radial-tangential model's fixed-point iteration run to
        convergence in double (vikit's cam2world stops after OpenCV's 5 iterations and rounds to float)."""
        if not (self.model == 0 and self.distorted):
            return self.cam2world(px)
        px = np.asarray(px, dtype=np.float64)
        k = self.d
        x0, y0 = (px[..., 0] - self.cx) / self.fx, (px[..., 1] - self.cy) / self.fy
        x, y = x0.copy(), y0.copy()
        for _ in range(60):
            r2 = x * x + y * y
            icdist = 1.0 / (1.0 + ((k[4] * r2 + k[1]) * r2 + k[0]) * r2)
            dX = 2.0 * k[2] * x * y + k[3] * (r2 + 2.0 * x * x)
            dY = k[2] * (r2 + 2.0 * y * y) + 2.0 * k[3] * x * y
            x, y = (x0 - dX) * icdist, (y0 - dY) * icdist
        xyz = np.stack([x, y, np.ones(px.shape[:-1])], axis=-1)
        return xyz / np.linalg.norm(xyz, axis=-1, keepdims=True)

    def world2cam(self, xyz: np.ndarray) -> np.ndarray:
        xyz = np.asarray(xyz, dtype=np.float64)
        x, y = xyz[..., 0] / xyz[..., 2], xyz[..., 1] / xyz[..., 2]
        if not self.distorted:
            return np.stack([self.fx * x + self.cx, self.fy * y + self.cy], axis=-1)
        if self.model == 0:
            k = self.d
            r2 = x * x + y * y
            cdist = 1 + k[0] * r2 + k[1] * r2 * r2 + k[4] * r2 ** 3
            xd = x * cdist + k[2] * 2 * x * y + k[3] * (r2 + 2 * x * x)
            yd = y * cdist + k[2] * (r2 + 2 * y * y) + k[3] * 2 * x * y
            return np.stack([xd * self.fx + self.cx, yd * self.fy + self.cy], axis=-1)
        s = self.d[0]
        r = np.sqrt(x * x + y * y)
        fac = np.where(r < 0.001, 1.0, np.arctan(r * 2.0 * np.tan(s / 2.0)) / (s * np.where(r > 0, r, 1.0)))
        return np.stack([self.cx + self.fx * fac * x, self.cy + self.fy * fac * y], axis=-1)


def atan_camera(width: int, height: int, fx: float, fy: float, cx: float, cy: float, s: float) -> Camera:
    """vk::ATANCamera(width, height, fx, fy, cx, cy, s): the constructor's pixel parameters (fx_ = width*fx,
    cx_ = cx*width - 0.5, ...)."""
    return Camera(width * fx, height * fy, cx * width - 0.5, cy * height - 0.5, width, height, 1, (s, 0.0, 0.0, 0.0, 0.0))


def reference_param_camera(kind: str) -> Camera:
    """The two cameras the reference ships parameter files for (svo_ros/param/camera_atan.yaml, camera_pinhole.yaml)."""
    if kind == "atan":
        return atan_camera(752, 480, 0.509326, 0.796651, 0.45905, 0.510056, 0.9320)
    if kind == "pinhole_radtan":
        return Camera(414.536145, 414.284429, 348.804988, 240.076451, 752, 480, 0, (-0.283076, 0.066674, 0.000896, 0.000778, 0.0))
    raise ValueError(kind)


def camera_for(width: int, height: int) -> Camera:
    """Cameras of SURVEY.md 8d: 640x480 f=320; 752x480 as the reference tests; 1080p f=960."""
    if (width, height) == (752, 480):
        return Camera(315.5, 315.5, 376.0, 240.0, 752, 480)  # svo/test/test_sparse_img_align.cpp:50
    f = width / 2.0
    return Camera(f, f, width / 2.0, height / 2.0, width, height)


# ------------------------------------------------------------------------------------------ SE3
def hat(w: np.ndarray) -> np.ndarray:
    return np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]], dtype=np.float64)


def se3_exp(x: np.ndarray) -> np.ndarray:
    """Tangent [upsilon, omega] (translation first, as Sophus) -> 3x4 [R|t] (numpy re-derivation)."""
    x = np.asarray(x, dtype=np.float64)
    ups, om = x[:3], x[3:]
    th = np.linalg.norm(om)
    O = hat(om)
    if th < 1e-12:
        R = np.eye(3) + O
        V = np.eye(3) + 0.5 * O
    else:
        a = np.sin(th) / th
        b = (1 - np.cos(th)) / th ** 2
        c = (th - np.sin(th)) / th ** 3
        R = np.eye(3) + a * O + b * O @ O
        V = np.eye(3) + b * O + c * O @ O
    T = np.zeros((3, 4))
    T[:, :3] = R
    T[:, 3] = V @ ups
    return T


def se3_mul(A: np.ndarray, B: np.ndarray) -> np.ndarray:
    C = np.zeros((3, 4))
    C[:, :3] = A[:, :3] @ B[:, :3]
    C[:, 3] = A[:, :3] @ B[:, 3] + A[:, 3]
    return C


def se3_inv(A: np.ndarray) -> np.ndarray:
    C = np.zeros((3, 4))
    C[:, :3] = A[:, :3].T
    C[:, 3] = -A[:, :3].T @ A[:, 3]
    return C


def se3_identity() -> np.ndarray:
    return np.hstack([np.eye(3), np.zeros((3, 1))])


def pose_error(T_a: np.ndarray, T_b: np.ndarray) -> tuple[float, float]:
    """(|t_a - t_b|, rotation angle of R_a R_b^T) -- the pose metric of SURVEY.md 8d."""
    dt = float(np.linalg.norm(T_a[:, 3] - T_b[:, 3]))
    R = T_a[:, :3] @ T_b[:, :3].T
    c = np.clip((np.trace(R) - 1) / 2, -1.0, 1.0)
    s = np.linalg.norm([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / 2
    return dt, float(np.arctan2(s, c))


# ------------------------------------------------------------------------------------- texture
TEXELS_PER_M = 320.0  # 1 texel = 3.125 mm; at 2 m and f=320 one level-0 pixel = 2 texels
TEX_SIZE = 2560       # 8 m x 8 m of plane


@lru_cache(maxsize=4)
def make_texture(seed: int) -> np.ndarray:
    """Band-limited noise with energy in every octave a 5-6 level pyramid can see."""
    from scipy.ndimage import gaussian_filter

    from scipy.ndimage import zoom

    rng = np.random.default_rng(seed)
    tex = np.zeros((TEX_SIZE, TEX_SIZE), dtype=np.float32)
    for sigma, amp in ((2.0, 1.0), (5.0, 1.0), (12.0, 1.2), (30.0, 1.4), (70.0, 1.6)):
        # large octaves are synthesised at reduced resolution and bilinearly upsampled (cheap, and
        # still band-limited): sigma_lowres stays ~2.5 texels
        k = max(1, int(sigma // 2.5))
        m = TEX_SIZE // k + 2
        n = rng.standard_normal((m, m) if k > 1 else (TEX_SIZE, TEX_SIZE)).astype(np.float32)
        g = gaussian_filter(n, sigma / k, mode="wrap")
        if k > 1:
            g = zoom(g, k, order=1)[:TEX_SIZE, :TEX_SIZE]
        tex += amp * g / g.std()
    tex -= tex.min()
    tex *= 255.0 / tex.max()
    return tex


@dataclass(frozen=True)
class Plane:
    """World plane n.X = d with an in-plane orthonormal basis for texture lookup."""

    n: np.ndarray
    d: float
    e1: np.ndarray
    e2: np.ndarray

    @staticmethod
    def tilted(tilt_x: float = 0.03, tilt_y: float = -0.02) -> "Plane":
        n = np.array([np.sin(tilt_y), -np.sin(tilt_x), 1.0])
        n /= np.linalg.norm(n)
        e1 = np.cross([0.0, 1.0, 0.0], n)
        e1 /= np.linalg.norm(e1)
        e2 = np.cross(n, e1)
        return Plane(n, 0.0, e1, e2)


def intersect(plane: Plane, T_f_w: np.ndarray, bearing: np.ndarray) -> np.ndarray:
    """World points where rays (frame bearings, any scale) hit the plane."""
    R, t = T_f_w[:, :3], T_f_w[:, 3]
    o = -R.T @ t
    d = bearing @ R  # rows: R^T f
    lam = (plane.d - plane.n @ o) / (d @ plane.n)
    return o[None, :] + lam[:, None] * d


def render(cam: Camera, T_f_w: np.ndarray, plane: Plane, tex: np.ndarray) -> np.ndarray:
    """Exact plane render (bilinear texture lookup, rounded to u8)."""
    u, v = np.meshgrid(np.arange(cam.width, dtype=np.float64), np.arange(cam.height, dtype=np.float64))
    if cam.distorted:  # exact inverse projection of every pixel centre through the camera model
        rays = cam.cam2world_exact(np.stack([u.ravel(), v.ravel()], axis=1))
    else:
        rays = np.stack([(u.ravel() - cam.cx) / cam.fx, (v.ravel() - cam.cy) / cam.fy, np.ones(u.size)], axis=1)
    X = intersect(plane, T_f_w, rays)
    s = (X @ plane.e1) * TEXELS_PER_M + TEX_SIZE / 2
    t = (X @ plane.e2) * TEXELS_PER_M + TEX_SIZE / 2
    s = np.clip(s, 0, TEX_SIZE - 1.001)
    t = np.clip(t, 0, TEX_SIZE - 1.001)
    s0 = np.floor(s).astype(np.int64)
    t0 = np.floor(t).astype(np.int64)
    fs = (s - s0).astype(np.float32)
    ft = (t - t0).astype(np.float32)
    a = tex[t0, s0]
    b = tex[t0, s0 + 1]
    c = tex[t0 + 1, s0]
    d = tex[t0 + 1, s0 + 1]
    val = (a * (1 - fs) + b * fs) * (1 - ft) + (c * (1 - fs) + d * fs) * ft
    return np.clip(np.rint(val), 0, 255).astype(np.uint8).reshape(cam.height, cam.width)


PYR_SCALAR, PYR_X86 = 0, 1


def half_sample(img: np.ndarray, rule: int = PYR_X86) -> np.ndarray:
    """[EXT] vk::halfSample (svo/src/frame.cpp:156-165).  PYR_X86 (default) = what the reference's x86 build computes:
    vikit's SSE2 branch -- rounded vertical average, then rounded average of adjacent columns -- when the input width is
    a multiple of 16, else the scalar rule (a+b+c+d)/4 with integer division; PYR_SCALAR = the scalar rule always."""
    h, w = img.shape[0] // 2, img.shape[1] // 2
    i = img[: 2 * h, : 2 * w].astype(np.uint16)
    if rule == PYR_X86 and img.shape[1] % 16 == 0:
        v = (i[0::2, :] + i[1::2, :] + 1) >> 1
        return ((v[:, 0::2] + v[:, 1::2] + 1) >> 1).astype(np.uint8)
    return ((i[0::2, 0::2] + i[0::2, 1::2] + i[1::2, 0::2] + i[1::2, 1::2]) // 4).astype(np.uint8)


def build_pyramid(img: np.ndarray, n_levels: int, rule: int = PYR_X86) -> list[np.ndarray]:
    pyr = [np.ascontiguousarray(img)]
    for _ in range(1, n_levels):
        pyr.append(np.ascontiguousarray(half_sample(pyr[-1], rule)))
    return pyr


# ------------------------------------------------------------------------------------ datasets
def base_pose() -> np.ndarray:
    """Camera 2 m above the plane looking down (as test scenes: t_w=(0.11,0.11,2.0),
    svo/test/test_matcher.cpp:52), slightly rotated."""
    R_w_f = np.diag([1.0, -1.0, -1.0]) @ se3_exp(np.array([0, 0, 0, 0.02, -0.03, 0.05]))[:, :3]
    T_w_f = np.hstack([R_w_f, np.array([[0.11], [0.11], [2.0]])])
    return se3_inv(T_w_f)


def jittered_features(rng: np.random.Generator, cam: Camera, n: int, margin: float) -> np.ndarray:
    """n sub-pixel feature positions on a jittered grid inside `margin` px from the border."""
    w, h = cam.width - 2 * margin, cam.height - 2 * margin
    nx = max(1, int(round(np.sqrt(n * w / h))))
    ny = int(np.ceil(n / nx))
    cw, ch = w / nx, h / ny
    idx = np.arange(nx * ny)
    rng.shuffle(idx)
    idx = np.sort(idx[:n])
    gx, gy = idx % nx, idx // nx
    px = np.stack([margin + (gx + rng.uniform(0.05, 0.95, n)) * cw,
                   margin + (gy + rng.uniform(0.05, 0.95, n)) * ch], axis=1)
    return px


def features_for(rng, cam: Camera, T_f_w: np.ndarray, plane: Plane, n: int, max_level: int,
                 null_fraction: float = 0.02) -> dict:
    px = jittered_features(rng, cam, n, margin=4.0 * (1 << max_level))
    f = cam.cam2world(px)
    pos = intersect(plane, T_f_w, f)
    has_point = np.ones(n, dtype=np.uint8)
    k = int(round(null_fraction * n))
    if k:
        has_point[rng.choice(n, size=k, replace=False)] = 0
    return dict(px=np.ascontiguousarray(px), f=np.ascontiguousarray(f),
                pos=np.ascontiguousarray(pos), has_point=has_point)


def make_frame_pair(seed: int, width: int = 640, height: int = 480, n_feat: int = 300,
                    n_levels: int = 5, trans: float = 0.03, rot_deg: float = 0.5,
                    tex_seed: int = 7, cam: Camera | None = None) -> dict:
    """One (ref, cur) pair of SURVEY.md 8d: GT motion uniform in +-trans m, +-rot_deg degrees."""
    rng = np.random.default_rng(seed)
    cam = camera_for(width, height) if cam is None else cam
    plane = Plane.tilted()
    tex = make_texture(tex_seed)
    T_ref_w = se3_mul(se3_exp(np.concatenate([rng.uniform(-0.2, 0.2, 3), rng.uniform(-0.03, 0.03, 3)])),
                      base_pose())
    xi = np.concatenate([rng.uniform(-trans, trans, 3), np.deg2rad(rng.uniform(-rot_deg, rot_deg, 3))])
    T_cur_ref = se3_exp(xi)
    T_cur_w = se3_mul(T_cur_ref, T_ref_w)
    ref_pyr = build_pyramid(render(cam, T_ref_w, plane, tex), n_levels)
    cur_pyr = build_pyramid(render(cam, T_cur_w, plane, tex), n_levels)
    feats = features_for(rng, cam, T_ref_w, plane, n_feat, n_levels - 1)
    ref_pos = se3_inv(T_ref_w)[:, 3].copy()
    return dict(cam=cam, ref_pyr=ref_pyr, cur_pyr=cur_pyr, T_ref_w=T_ref_w, T_cur_w=T_cur_w,
                T_cur_ref_gt=T_cur_ref, ref_pos=ref_pos, n_levels=n_levels, seed=seed, **feats)


def make_stream(seed: int, n_frames: int, width: int = 640, height: int = 480, n_feat: int = 300,
                n_levels: int = 5, trans: float = 0.02, rot_deg: float = 0.35, tex_seed: int = 7) -> dict:
    """One synthetic camera stream: n_frames poses on a bounded random walk; frame k is the
    reference of pair k and the current frame of pair k-1 (as in FrameHandlerMono::processFrame,
    svo/src/frame_handler_mono.cpp:129-139, where last_frame_ is the reference)."""
    rng = np.random.default_rng(seed)
    cam = camera_for(width, height)
    plane = Plane.tilted()
    tex = make_texture(tex_seed)
    T = base_pose()
    frames, poses, feats = [], [], []
    drift = np.zeros(6)
    for k in range(n_frames):
        poses.append(T)
        frames.append(build_pyramid(render(cam, T, plane, tex), n_levels))
        feats.append(features_for(rng, cam, T, plane, n_feat, n_levels - 1))
        xi = np.concatenate([rng.uniform(-trans, trans, 3), np.deg2rad(rng.uniform(-rot_deg, rot_deg, 3))])
        xi -= 0.2 * drift  # pull back towards the start so the walk stays over the texture
        drift += xi
        T = se3_mul(se3_exp(xi), T)
    return dict(cam=cam, frames=frames, poses=poses, feats=feats, n_levels=n_levels, seed=seed)


# --------------------------------------------------------------------------- bulk stream (bench)
def render_torch(cam: Camera, poses: list, plane: Plane, tex: np.ndarray, device: str = "cpu"):
    """Same plane render as `render`, batched over poses with torch (data manufacture only, not
    part of any measured path).  Returns a uint8 tensor [len(poses), H, W] on `device`."""
    import torch

    dev = torch.device(device)
    t_tex = torch.from_numpy(tex).to(dev)
    u, v = torch.meshgrid(torch.arange(cam.width, dtype=torch.float64, device=dev),
                          torch.arange(cam.height, dtype=torch.float64, device=dev), indexing="xy")
    rays = torch.stack([(u.reshape(-1) - cam.cx) / cam.fx, (v.reshape(-1) - cam.cy) / cam.fy,
                        torch.ones(u.numel(), dtype=torch.float64, device=dev)], dim=1)
    n = torch.tensor(plane.n, device=dev)
    e1 = torch.tensor(plane.e1, device=dev)
    e2 = torch.tensor(plane.e2, device=dev)
    out = torch.empty((len(poses), cam.height, cam.width), dtype=torch.uint8, device=dev)
    for k, T in enumerate(poses):
        R = torch.tensor(T[:, :3], device=dev)
        t = torch.tensor(T[:, 3], device=dev)
        o = -(R.T @ t)
        d = rays @ R
        lam = (plane.d - n @ o) / (d @ n)
        X = o[None, :] + lam[:, None] * d
        s = ((X @ e1) * TEXELS_PER_M + TEX_SIZE / 2).clamp(0, TEX_SIZE - 1.001)
        tt = ((X @ e2) * TEXELS_PER_M + TEX_SIZE / 2).clamp(0, TEX_SIZE - 1.001)
        s0, t0 = s.floor().long(), tt.floor().long()
        fs, ft = (s - s0).float(), (tt - t0).float()
        a, b = t_tex[t0, s0], t_tex[t0, s0 + 1]
        c, dd = t_tex[t0 + 1, s0], t_tex[t0 + 1, s0 + 1]
        val = (a * (1 - fs) + b * fs) * (1 - ft) + (c * (1 - fs) + dd * fs) * ft
        out[k] = val.round().clamp(0, 255).to(torch.uint8).reshape(cam.height, cam.width)
    return out


def stream_poses(seed: int, n_frames: int, trans: float = 0.02, rot_deg: float = 0.35) -> list:
    """Bounded random walk of camera poses T_f_w (the trajectory of `make_stream`)."""
    rng = np.random.default_rng(seed)
    T = base_pose()
    poses, drift = [], np.zeros(6)
    for _ in range(n_frames):
        poses.append(T)
        xi = np.concatenate([rng.uniform(-trans, trans, 3), np.deg2rad(rng.uniform(-rot_deg, rot_deg, 3))])
        xi -= 0.2 * drift
        drift += xi
        T = se3_mul(se3_exp(xi), T)
    return poses


def make_stream_fast(seed: int, n_frames: int, width: int = 640, height: int = 480, n_feat: int = 300,
                     n_levels: int = 5, device: str = "cpu", tex_seed: int = 7) -> dict:
    """A camera stream for the benchmark: level-0 images as one uint8 torch tensor (rendered with
    torch on `device`, returned on the CPU), per-frame features as numpy arrays."""
    cam = camera_for(width, height)
    plane = Plane.tilted()
    tex = make_texture(tex_seed)
    poses = stream_poses(seed, n_frames)
    imgs = render_torch(cam, poses, plane, tex, device).cpu()
    rng = np.random.default_rng(seed + 77)
    feats = [features_for(rng, cam, T, plane, n_feat, n_levels - 1) for T in poses]
    return dict(cam=cam, level0=imgs, poses=poses, feats=feats, n_levels=n_levels, seed=seed)


# ------------------------------------------------------------ cases for align / matcher / pose-opt / depth filter
def patch_with_border(img: np.ndarray, px: np.ndarray) -> np.ndarray:
    """10x10 bilinear patch around sub-pixel px, truncated to u8 -- the procedure of
    svo/test/test_feature_alignment.cpp:29-52 (generateRefPatchNoWarpInterpolate)."""
    u_r, v_r = int(np.floor(px[0])), int(np.floor(px[1]))
    su, sv = np.float32(px[0] - u_r), np.float32(px[1] - v_r)
    wTL = np.float32((1.0 - su) * (1.0 - sv)); wTR = np.float32(su * (1.0 - sv))
    wBL = np.float32((1.0 - su) * sv); wBR = np.float32(su * sv)
    blk = img[v_r - 5: v_r + 6, u_r - 5: u_r + 6].astype(np.float32)
    val = wTL * blk[:-1, :-1] + wTR * blk[:-1, 1:] + wBL * blk[1:, :-1] + wBR * blk[1:, 1:]
    return val.astype(np.uint8)  # truncation, as the C assignment to uint8_t


def make_align_case(seed: int, m: int, width: int = 640, height: int = 480, n_levels: int = 3) -> dict:
    """m independent align2D/align1D problems on the levels of one rendered frame."""
    rng = np.random.default_rng(seed)
    cam = camera_for(width, height)
    pyr = build_pyramid(render(cam, base_pose(), Plane.tilted(), make_texture(7)), n_levels)
    level = rng.integers(0, n_levels, m).astype(np.int32)
    px_true = np.zeros((m, 2)); px_start = np.zeros((m, 2))
    pwb = np.zeros((m, 100), np.uint8); patch = np.zeros((m, 64), np.uint8)
    direction = np.zeros((m, 2), np.float32)
    for i in range(m):
        im = pyr[level[i]]
        h, w = im.shape
        margin = 12 if i % 10 else 5  # every 10th problem starts close to the border
        px_true[i] = [rng.uniform(margin, w - margin), rng.uniform(margin, h - margin)]
        p = patch_with_border(im, px_true[i])
        pwb[i] = p.ravel()
        patch[i] = p[1:9, 1:9].ravel()
        off = rng.uniform(-1.5, 1.5, 2)
        px_start[i] = px_true[i] - off
        d = off / (np.linalg.norm(off) + 1e-12)
        direction[i] = d.astype(np.float32)
    return dict(cam=cam, pyr=pyr, level=level, px_true=px_true, px_start=px_start, pwb=pwb, patch=patch,
                dir=direction)


def make_two_view(seed: int, width: int = 752, height: int = 480, n_levels: int = 5, baseline: float = 0.3,
                  rot_deg: float = 2.0, cam: Camera | None = None) -> dict:
    """Reference keyframe + current frame with a real baseline (geometry of svo/test/test_matcher.cpp:52-57)."""
    rng = np.random.default_rng(seed)
    cam = camera_for(width, height) if cam is None else cam
    plane, tex = Plane.tilted(), make_texture(7)
    T_ref_w = base_pose()
    d = rng.normal(size=3); d[2] *= 0.2; d *= baseline / np.linalg.norm(d)
    xi = np.concatenate([d, np.deg2rad(rng.uniform(-rot_deg, rot_deg, 3))])
    T_cur_w = se3_mul(se3_exp(xi), T_ref_w)
    ref_pyr = build_pyramid(render(cam, T_ref_w, plane, tex), n_levels)
    cur_pyr = build_pyramid(render(cam, T_cur_w, plane, tex), n_levels)
    return dict(cam=cam, plane=plane, T_ref_w=T_ref_w, T_cur_w=T_cur_w, ref_pyr=ref_pyr, cur_pyr=cur_pyr,
                n_levels=n_levels, rng=rng)


def make_match_case(seed: int, m: int, **kw) -> dict:
    """m Matcher::findMatchDirect candidates: reference features with 3D points and a current-frame
    guess within ~1.5 px of the true reprojection."""
    tv = make_two_view(seed, baseline=kw.pop("baseline", 0.12), **kw)
    rng, cam = tv["rng"], tv["cam"]
    level = rng.integers(0, 3, m).astype(np.int32)
    px = np.stack([rng.uniform(40, cam.width - 40, m), rng.uniform(40, cam.height - 40, m)], axis=1)
    px = np.round(px / (1 << level)[:, None]) * (1 << level)[:, None]  # detected at integer level pixels
    f = cam.cam2world(px)
    pos = intersect(tv["plane"], tv["T_ref_w"], f)
    Tc = tv["T_cur_w"]
    pc = pos @ Tc[:, :3].T + Tc[:, 3]
    px_cur_true = cam.world2cam(pc)
    px_cur = px_cur_true + rng.uniform(-1.5, 1.5, (m, 2))
    ftr_type = (rng.uniform(size=m) < 0.15).astype(np.int32)
    ang = rng.uniform(0, 2 * np.pi, m)
    grad = np.stack([np.cos(ang), np.sin(ang)], axis=1)
    tv.update(M=m, ref_px=px, ref_f=f, ref_level=level, ftr_type=ftr_type, ref_grad=grad, point_pos=pos,
              px_cur=px_cur, px_cur_true=px_cur_true)
    return tv


def make_depth_case(seed: int, n_seeds: int = 2000, **kw) -> dict:
    """BASELINE config C2: seeds `Seed(ftr, 2.0, 0.5)` (svo/test/test_depth_filter.cpp:128) on a jittered
    grid of integer pixels of a 752x480 keyframe, one current frame with a baseline."""
    tv = make_two_view(seed, **kw)
    rng, cam = tv["rng"], tv["cam"]
    px = np.floor(jittered_features(rng, cam, n_seeds, margin=6.0))
    level = rng.integers(0, 3, n_seeds).astype(np.int32)
    px = np.floor(px / (1 << level)[:, None]) * (1 << level)[:, None]
    f = cam.cam2world(px)
    ftr_type = (rng.uniform(size=n_seeds) < 0.1).astype(np.int32)
    ang = rng.uniform(0, 2 * np.pi, n_seeds)
    grad = np.stack([np.cos(ang), np.sin(ang)], axis=1)
    depth_mean, depth_min = np.float32(2.0), np.float32(0.5)
    z_range = np.float32(1.0) / depth_min  # depth_filter.cpp:37-46
    seeds = dict(a=np.full(n_seeds, 10, np.float32), b=np.full(n_seeds, 10, np.float32),
                 mu=np.full(n_seeds, np.float32(1.0) / depth_mean, np.float32),
                 z_range=np.full(n_seeds, z_range, np.float32),
                 sigma2=np.full(n_seeds, z_range * z_range / np.float32(36), np.float32))
    batch_id = np.where(rng.uniform(size=n_seeds) < 0.03, 0, 5).astype(np.int32)  # a few too-old seeds
    depth_gt = np.linalg.norm(intersect(tv["plane"], tv["T_ref_w"], f) - se3_inv(tv["T_ref_w"])[:, 3], axis=1)
    tv.update(M=n_seeds, ftr_px=px, ftr_f=f, ftr_level=level, ftr_type=ftr_type, ftr_grad=grad, seeds=seeds,
              batch_id=batch_id, batch_counter=6, ref_index=np.zeros(n_seeds, np.int32), depth_gt=depth_gt)
    return tv


def make_multi_keyframe_depth_case(seed: int, n_seeds: int = 300, n_kfs: int = 3, baseline: float = 0.3) -> dict:
    """Seeds of n_kfs keyframes with different poses and images (keyframe k moved by up to 15 cm / 3 degrees from
    keyframe 0), updated by one current frame; ref_index interleaves the keyframes seed by seed (0, 1, 2, 0, 1, ...)."""
    c = make_depth_case(seed, n_seeds, baseline=baseline)
    rng = np.random.default_rng(seed + 1000)
    plane, tex, cam = c["plane"], make_texture(7), c["cam"]
    kf_T, kf_pyr = [c["T_ref_w"]], [c["ref_pyr"]]
    for _ in range(1, n_kfs):
        xi = np.concatenate([rng.uniform(-0.15, 0.15, 3), np.deg2rad(rng.uniform(-3, 3, 3))])
        T = se3_mul(se3_exp(xi), c["T_ref_w"])
        kf_T.append(T)
        kf_pyr.append(build_pyramid(render(cam, T, plane, tex), c["n_levels"]))
    ref_index = (np.arange(n_seeds) % n_kfs).astype(np.int32)
    depth_gt = np.array([np.linalg.norm(intersect(plane, kf_T[r], c["ftr_f"][i:i + 1])[0] - se3_inv(kf_T[r])[:, 3])
                         for i, r in enumerate(ref_index)])
    c.update(kf_T=kf_T, kf_pyr=kf_pyr, ref_index=ref_index, depth_gt=depth_gt)
    return c


def make_seed_status_case(seed: int, n_seeds: int = 400) -> dict:
    """One launch's worth of seeds that end in every status DepthFilter::updateSeeds can give them: too old (batch_id),
    behind the camera (negative mu), outside the current frame (a depth of a few cm, so the current frame's 0.3 m
    baseline throws the projection off the image or behind it), no match, updated and converged (a fifth of the seeds start
    at the true depth with a small variance) -- plus seeds whose sigma2 is negative, NaN or infinite."""
    c = make_depth_case(seed, n_seeds, baseline=0.3)
    rng = np.random.default_rng(seed + 2000)
    s = c["seeds"]
    s["sigma2"][::5] *= np.float32(1e-3)
    s["mu"][::5] = (1.0 / c["depth_gt"][::5]).astype(np.float32)
    idx = rng.permutation(n_seeds)
    s["mu"][idx[:20]] = np.float32(-0.5)                                    # behind
    s["mu"][idx[20:45]] = rng.uniform(20, 60, 25).astype(np.float32)        # 2-5 cm in front of the keyframe
    bad = idx[45:75]
    s["sigma2"][bad] = np.array([-0.1, np.nan, np.inf] * 10, np.float32)
    c["batch_id"][idx[75:85]] = 0                                           # too old
    c["bad_sigma2"] = np.zeros(n_seeds, bool)
    c["bad_sigma2"][bad] = True
    return c


def make_pose_opt_case(seed: int, n: int = 1000, width: int = 1920, height: int = 1080, px_noise: float = 1.0,
                       outlier_frac: float = 0.03) -> dict:
    """BASELINE config C3 (pose optimizer part): n observations with N(0, px_noise) pixel noise
    (svo/test/test_pose_optimizer.cpp:92), a few gross outliers, perturbed initial pose."""
    rng = np.random.default_rng(seed)
    cam = camera_for(width, height)
    plane = Plane.tilted()
    T_true = base_pose()
    px = np.stack([rng.uniform(20, width - 20, n), rng.uniform(20, height - 20, n)], axis=1)
    pos = intersect(plane, T_true, cam.cam2world(px))
    noisy = px + rng.normal(0, px_noise, (n, 2))
    k = int(outlier_frac * n)
    if k:
        noisy[rng.choice(n, k, replace=False)] += rng.uniform(-25, 25, (k, 2))
    f = cam.cam2world(noisy)
    level = rng.integers(0, 3, n).astype(np.int32)
    has_point = (rng.uniform(size=n) > 0.02).astype(np.uint8)
    T_init = se3_mul(se3_exp(np.concatenate([rng.uniform(-0.05, 0.05, 3), rng.uniform(-0.01, 0.01, 3)])), T_true)
    return dict(cam=cam, f=f, pos=pos, level=level, has_point=has_point, T_init=T_init, T_true=T_true)


def make_pose_window_case(seed: int, n: int, window_px: float, depth: float = 40.0, width: int = 752, height: int = 480,
                          px_noise: float = 0.3) -> dict:
    """Ill-conditioned pose problems: n observations inside a window_px x window_px pixel window at the image centre, their
    points on a fronto-parallel plane `depth` m away.  The smaller the window (and the larger the depth), the closer the
    translations parallel to the image and the rotations about the two image axes come to explaining the same motion: the
    normal matrix's smallest unpivoted LDL^T pivot falls with the window."""
    rng = np.random.default_rng(seed)
    cam = camera_for(width, height)
    T_true = base_pose()
    px = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.5, 0.5, n)], axis=1) * window_px + [cam.cx, cam.cy]
    bearing = cam.cam2world(px)
    Tinv = se3_inv(T_true)
    pos = (bearing * (depth / bearing[:, 2:3])) @ Tinv[:, :3].T + Tinv[:, 3]
    f = cam.cam2world(px + rng.normal(0, px_noise, (n, 2)))
    level = rng.integers(0, 3, n).astype(np.int32)
    T_init = se3_mul(se3_exp(np.concatenate([rng.uniform(-0.01, 0.01, 3), rng.uniform(-0.002, 0.002, 3)])), T_true)
    return dict(cam=cam, f=f, pos=pos, level=level, has_point=np.ones(n, np.uint8), T_init=T_init, T_true=T_true)


def make_pose_line_case(seed: int, n: int, width: int = 752, height: int = 480, px_noise: float = 0.3) -> dict:
    """A singular pose problem: every point on one 3D line through the scene, so the rotation about that line (with the
    translation that keeps the line in place) does not change any reprojection error."""
    rng = np.random.default_rng(seed)
    cam = camera_for(width, height)
    T_true = base_pose()
    Tinv = se3_inv(T_true)
    a, b = np.array([-1.5, -0.4, 3.0]), np.array([1.2, 0.5, 5.0])  # camera-frame end points, in view
    s = np.sort(rng.uniform(0, 1, n))
    pos = (a + s[:, None] * (b - a)) @ Tinv[:, :3].T + Tinv[:, 3]
    px = cam.world2cam(a + s[:, None] * (b - a))
    f = cam.cam2world(px + rng.normal(0, px_noise, (n, 2)))
    level = rng.integers(0, 3, n).astype(np.int32)
    T_init = se3_mul(se3_exp(np.concatenate([rng.uniform(-0.02, 0.02, 3), rng.uniform(-0.004, 0.004, 3)])), T_true)
    return dict(cam=cam, f=f, pos=pos, level=level, has_point=np.ones(n, np.uint8), T_init=T_init, T_true=T_true)


def make_map_case(seed: int, n_kfs: int = 8, n_points: int = 700, width: int = 752, height: int = 480, n_levels: int = 5,
                  n_candidates: int = 80, spread: float = 0.5, bad_frac: float = 0.2, cam: Camera | None = None,
                  obs_prob: float = 0.45, same_pose: tuple = ()) -> dict:
    """A small map for Reprojector::reprojectMap (svo/src/reprojector.cpp:64-217): n_kfs keyframes on a trajectory above
    the textured plane, world points on the plane observed by 1..n_kfs keyframes (one Feature per observation, detected
    on the integer grid of its level), point types / reprojection counters near the reference's thresholds, converged-
    seed candidates whose single observation is not in its keyframe's fts_ list, five key points per keyframe, a current
    frame close to the last keyframes, and a shuffled cell order.  Everything is flat arrays (the `map view`).
    obs_prob: the probability that a keyframe observes a map point.  same_pose: (src, dst) keyframe pairs; keyframe dst
    gets the pose (and image) of keyframe src, so Point::getCloseViewObs sees exactly equal angles."""
    rng = np.random.default_rng(seed)
    cam = camera_for(width, height) if cam is None else cam
    plane, tex = Plane.tilted(), make_texture(7)
    kf_T = []
    for k in range(n_kfs):
        xi = np.concatenate([rng.uniform(-spread, spread, 2), rng.uniform(-0.15, 0.15, 1), np.deg2rad(rng.uniform(-3, 3, 3))])
        kf_T.append(se3_mul(se3_exp(xi), base_pose()))
    for src, dst in same_pose:
        kf_T[dst] = kf_T[src].copy()
    xi = np.concatenate([rng.uniform(-0.1, 0.1, 3), np.deg2rad(rng.uniform(-2, 2, 3))])
    cur_T = se3_mul(se3_exp(xi), kf_T[-1])
    kf_pyr = [build_pyramid(render(cam, T, plane, tex), n_levels) for T in kf_T]
    cur_pyr = build_pyramid(render(cam, cur_T, plane, tex), n_levels)

    # world points: rays of a virtual wide view around the trajectory
    ext = spread + 2.2
    P = n_points + n_candidates
    a, b = rng.uniform(-ext, ext, P), rng.uniform(-ext, ext, P)
    c0 = se3_inv(base_pose())[:, 3]
    pos = c0[None, :] * [1, 1, 0] + a[:, None] * plane.e1 + b[:, None] * plane.e2
    pos -= np.outer(pos @ plane.n - plane.d, plane.n)                       # on the plane
    pos += rng.normal(0, 0.004, pos.shape)                                 # map noise

    ftr_kf, ftr_px, ftr_f, ftr_level, ftr_type, ftr_grad, ftr_point = [], [], [], [], [], [], []
    kf_fts = [[] for _ in range(n_kfs)]
    pt_obs = [[] for _ in range(P)]

    def add_ftr(k, p, in_fts):
        T = kf_T[k]
        pc = T[:, :3] @ pos[p] + T[:, 3]
        if pc[2] <= 0.1:
            return False
        px = cam.world2cam(pc)
        L = int(rng.integers(0, 3))
        px = np.round(px / (1 << L)) * (1 << L)
        if not (12 <= px[0] < width - 12 and 12 <= px[1] < height - 12):
            return False
        i = len(ftr_kf)
        ftr_kf.append(k); ftr_px.append(px); ftr_f.append(cam.cam2world(px)); ftr_level.append(L)
        ftr_type.append(int(rng.uniform() < 0.12))
        ang = rng.uniform(0, 2 * np.pi)
        ftr_grad.append([np.cos(ang), np.sin(ang)]); ftr_point.append(p)
        if in_fts:
            kf_fts[k].append(i)
        pt_obs[p].insert(0, i)                                             # Point::addFrameRef pushes to the front
        return True

    for p in range(n_points):
        for k in range(n_kfs):
            if rng.uniform() < obs_prob:
                add_ftr(k, p, True)
    cand = []
    for p in range(n_points, P):
        for k in rng.permutation(n_kfs):
            if add_ftr(int(k), p, False):                                  # the seed's feature: not in fts_
                cand.append(p)
                break
    # a few features without a point (Feature::point == NULL)
    for k in range(n_kfs):
        for _ in range(5):
            i = len(ftr_kf)
            px = np.round(rng.uniform([20, 20], [width - 20, height - 20]))
            ftr_kf.append(k); ftr_px.append(px); ftr_f.append(cam.cam2world(px)); ftr_level.append(0); ftr_type.append(0)
            ftr_grad.append([1.0, 0.0]); ftr_point.append(-1)
            kf_fts[k].insert(int(rng.integers(0, len(kf_fts[k]) + 1)), i)

    # map errors: a fraction of the points sits 0.08..0.25 m away from where its features saw it -> failed matches
    bad = rng.uniform(size=P) < bad_frac
    ang = rng.uniform(0, 2 * np.pi, P)
    shift = rng.uniform(0.08, 0.25, P)[:, None] * (np.cos(ang)[:, None] * plane.e1 + np.sin(ang)[:, None] * plane.e2)
    pos = pos + shift * bad[:, None]

    pt_type = rng.choice([2, 3], P, p=[0.6, 0.4]).astype(np.int32)          # UNKNOWN / GOOD
    pt_type[rng.choice(n_points, 12, replace=False)] = 0                   # some already TYPE_DELETED
    pt_type[n_points:] = 1                                                 # TYPE_CANDIDATE
    n_failed = rng.integers(0, 17, P).astype(np.int32)
    n_failed[n_points:] = rng.integers(0, 32, n_candidates)
    n_succ = rng.integers(0, 12, P).astype(np.int32)

    keypt_pos = np.zeros((n_kfs, 5, 3)); keypt_valid = np.zeros((n_kfs, 5), np.uint8)
    keypt_ftr = np.full((n_kfs, 5), -1, np.int32)
    for k in range(n_kfs):
        idx = [i for i in kf_fts[k] if ftr_point[i] >= 0]
        if not idx:
            continue
        pxs = np.array([ftr_px[i] for i in idx]) - [width / 2, height / 2]
        picks = [int(np.argmin(np.max(np.abs(pxs), axis=1)))]
        for sx, sy in ((1, 1), (1, -1), (-1, -1), (-1, 1)):
            picks.append(int(np.argmax(np.where((pxs[:, 0] * sx >= 0) & (pxs[:, 1] * sy >= 0), np.abs(pxs[:, 0] * pxs[:, 1]), -1))))
        for j, q in enumerate(picks):
            keypt_pos[k, j] = pos[ftr_point[idx[q]]]
            keypt_valid[k, j] = 1
            keypt_ftr[k, j] = idx[q]
    if n_kfs > 2:
        keypt_valid[0, :] = 0                                              # one keyframe without key points: never close
        keypt_ftr[0, :] = -1

    off = np.zeros(n_kfs + 1, np.int32)
    off[1:] = np.cumsum([len(x) for x in kf_fts])
    ooff = np.zeros(P + 1, np.int32)
    ooff[1:] = np.cumsum([len(x) for x in pt_obs])
    grid = 30
    n_cells = int(np.ceil(width / grid)) * int(np.ceil(height / grid))
    view = dict(n_kfs=n_kfs, kf_T_f_w=np.stack(kf_T), kf_keypt_pos=keypt_pos, kf_keypt_valid=keypt_valid, kf_fts_offset=off,
                kf_fts=np.array([i for x in kf_fts for i in x], np.int32), n_ftrs=len(ftr_kf),
                ftr_kf=np.array(ftr_kf, np.int32), ftr_px=np.array(ftr_px, np.float64), ftr_f=np.array(ftr_f),
                ftr_level=np.array(ftr_level, np.int32), ftr_type=np.array(ftr_type, np.int32),
                ftr_grad=np.array(ftr_grad), ftr_point=np.array(ftr_point, np.int32), n_points=P, pt_pos=pos,
                pt_obs_offset=ooff, pt_obs=np.array([i for x in pt_obs for i in x], np.int32),
                n_candidates=len(cand), cand_point=np.array(cand, np.int32))
    return dict(cam=cam, view=view, kf_pyr=kf_pyr, cur_pyr=cur_pyr, cur_T_f_w=cur_T, n_levels=n_levels, keypt_ftr=keypt_ftr,
                pt_type=pt_type, pt_n_failed=n_failed, pt_n_succeeded=n_succ, cell_order=rng.permutation(n_cells).astype(np.int32),
                options=dict(grid_size=grid, max_fts=120, max_n_kfs=10, find_match_direct=1, max_search_level=2, align_max_iter=10))
