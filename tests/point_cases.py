"""Points for the tests of point_optimize_kernel (tests/test_point_edges_gpu.py) and of its oracle
(tests/test_point_edge_pins.py): random tracks, the degenerate geometries and the non-finite inputs.

A point is (start position, observing poses T_f_w as [N, 12] row-major [R | t], unit bearings [N, 3])."""
from __future__ import annotations

import numpy as np

from rpg_svo_b200 import synth


def pose_at(centre, rot=(0.0, 0.0, 0.0)) -> np.ndarray:
    """T_f_w (12 values) of a camera at `centre` (world) rotated by the so(3) vector `rot`."""
    R = synth.se3_exp(np.concatenate([[0.0, 0.0, 0.0], rot]))[:, :3]
    return np.hstack([R, (-R @ np.asarray(centre, float))[:, None]]).reshape(12)


def bearings(Ts, X, rng=None, noise=0.0) -> np.ndarray:
    """Unit bearings of the world point X in each pose, with optional Gaussian noise before normalising."""
    fs = []
    for T in Ts:
        T = np.asarray(T).reshape(3, 4)
        f = T[:, :3] @ X + T[:, 3]
        f = f / np.linalg.norm(f)
        if noise:
            f = f + rng.normal(0, noise, 3)
        fs.append(f / np.linalg.norm(f))
    return np.array(fs)


def track(rng, n_obs, noise=1e-3, start_sigma=0.05, spread=0.5, depth=(3.0, 6.0)):
    """A point 3-6 m in front of the world origin seen by n_obs cameras within `spread` m of the origin (small rotations),
    bearings with `noise` (radians), start `start_sigma` m from the truth."""
    X = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(*depth)])
    Ts = np.array([pose_at(rng.uniform(-spread, spread, 3), rng.uniform(-0.05, 0.05, 3)) for _ in range(n_obs)]).reshape(-1, 12)
    fs = bearings(Ts, X, rng, noise) if n_obs else np.zeros((0, 3))
    return X + rng.normal(0, start_sigma, 3), Ts, fs, X


def two_view(baseline, depth=4.0, noise=0.0, seed=0):
    """Two unrotated cameras `baseline` m apart (along x) looking at a point `depth` m away: cond(A) ~ (depth / baseline)^2."""
    rng = np.random.default_rng(seed)
    X = np.array([0.3, -0.2, depth])
    Ts = np.array([pose_at([-baseline / 2, 0.0, 0.0]), pose_at([baseline / 2, 0.0, 0.0])])
    return X + np.array([0.01, -0.02, 0.05]), Ts, bearings(Ts, X, rng, noise), X


def degenerate_cases():
    """(name, n_iter, start, Ts, fs) of the degenerate geometries."""
    rng = np.random.default_rng(11)
    out = []
    # every frame at one centre: A's null space is the ray (rank 2).  Unrotated frames and a point on their optical axis
    # give A = diag(k/z^2, k/z^2, 0) exactly -- the third pivot is exactly 0 (one iteration: the step leaves the axis);
    # rotated frames give a rounding-noise pivot.
    Ts = np.array([pose_at([0.0, 0.0, 0.0])] * 3)
    out.append(("one_centre_axis", 1, np.array([0.0, 0.0, 4.0]), Ts, bearings(Ts, np.array([0.02, -0.01, 4.5]))))
    Ts = np.array([pose_at([0.1, 0.2, -0.1], rng.uniform(-0.3, 0.3, 3)) for _ in range(4)])
    out.append(("one_centre_rotated", 5, np.array([0.5, 0.1, 4.0]), Ts, bearings(Ts, np.array([0.45, 0.12, 4.3]), rng, 1e-3)))
    for b in (2.6e-1, 8e-3, 2.6e-4, 8e-6):
        s, Ts, fs, _ = two_view(b, noise=1e-4, seed=int(b * 1e7))
        out.append((f"baseline_{b:g}", 5, s, Ts, fs))
    s, Ts, fs, _ = track(rng, 3)
    out.append(("duplicated", 5, s, np.concatenate([Ts, Ts[:2], Ts[:1]]), np.concatenate([fs, fs[:2], fs[:1]])))
    _, Ts, fs, X = track(rng, 4)
    T = np.asarray(Ts[0]).reshape(3, 4)
    s = X - 2.0 * (T[:, :3].T @ (T[:, :3] @ X + T[:, 3]))                 # mirrored through camera 0: behind it
    out.append(("behind_camera", 5, s, Ts, fs))
    return out


def nonfinite_cases():
    """(name, n_iter, start, Ts, fs) with a start at z = 0 in an observing frame, a bearing with f_z = 0, or NaN / inf in
    the start, a bearing or a pose."""
    rng = np.random.default_rng(12)
    out = []
    s, Ts, fs, _ = track(rng, 3)
    Ts[0] = pose_at([0.0, 0.0, 0.0])
    out.append(("start_z0", 5, np.array([0.4, -0.3, 0.0]), Ts, fs))  # frame 0 is the world frame: p_z = 0 exactly
    for name, v in (("nan", np.nan), ("inf", np.inf)):
        s, Ts, fs, _ = track(rng, 3)
        s[1] = v
        out.append((f"start_{name}", 5, s, Ts, fs))
        s, Ts, fs, _ = track(rng, 3)
        fs[1, 0] = v
        out.append((f"bearing_{name}", 5, s, Ts, fs))
        s, Ts, fs, _ = track(rng, 3)
        Ts[2, 5] = v                                                    # R_11 of the third pose
        out.append((f"pose_R_{name}", 5, s, Ts, fs))
        s, Ts, fs, _ = track(rng, 3)
        Ts[2, 11] = v                                                   # t_z of the third pose
        out.append((f"pose_t_{name}", 5, s, Ts, fs))
    s, Ts, fs, _ = track(rng, 3)
    fs[0, 2] = 0.0
    out.append(("bearing_fz0", 5, s, Ts, fs))
    return out


def edge_cases():
    return degenerate_cases() + nonfinite_cases()


def ref_outputs(ref):
    """The compiled reference's result for every edge case, in the order the pins recorded them."""
    return [ref.point_optimize(n_iter, s, Ts, fs) for _, n_iter, s, Ts, fs in edge_cases()]


def batch(points):
    """point_optimize_batch arguments (start [P,3], obs_offset, obs_frame, obs_f, frame poses [F,3,4]) of points given
    as (start, Ts, fs): each observation gets its own frame."""
    starts = np.array([p[0] for p in points], float).reshape(-1, 3)
    counts = [len(p[2]) for p in points]
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    Ts = np.concatenate([np.asarray(p[1]).reshape(-1, 12) for p in points] + [np.zeros((0, 12))])
    fs = np.concatenate([np.asarray(p[2]).reshape(-1, 3) for p in points] + [np.zeros((0, 3))])
    if len(Ts) == 0:
        Ts = np.zeros((1, 12))
    return starts, off, np.arange(int(off[-1]), dtype=np.int32), fs, Ts.reshape(-1, 3, 4)
