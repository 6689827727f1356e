"""Pose-optimizer cases shared by the GPU edge tests (test_pose_edges_gpu.py) and the CPU pins of the same corners
against the compiled reference (test_edge_pins.py)."""
import numpy as np

from rpg_svo_b200 import synth

PIVOT_THRESH = 1e-13  # fact6_compute_upper: a pivot <= 1e-13 * max diagonal sends the solve to the pivoted LDL^T


def args(c, n_iter=10):
    return (2.0, n_iter, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], c["has_point"])


def first_normal_matrix(c):
    """The Gauss-Newton normal matrix A of iteration 0 (T_init, MAD scale, Tukey weights), in numpy: what decides whether
    the kernel's first solve takes the unpivoted fast path."""
    return first_normal_system(c)[0]


def first_normal_system(c):
    """(A, b) of iteration 0, as pose_optimizer.cpp:75-97 forms them: the first step dT solves A dT = b."""
    T, hp = c["T_init"], c["has_point"].astype(bool)
    f, pos, lv = c["f"][hp], c["pos"][hp], c["level"][hp]
    p = pos @ T[:, :3].T + T[:, 3]
    sic = 1.0 / (1 << lv)
    e = (f[:, :2] / f[:, 2:3] - p[:, :2] / p[:, 2:3]) * sic[:, None]
    en = np.sqrt((e ** 2).sum(1))
    err = en.astype(np.float32)
    scale = float(np.float32(1.48) * np.partition(err, len(err) // 2)[len(err) // 2])
    x = (en / scale).astype(np.float32)
    b2 = np.float32(4.6851) * np.float32(4.6851)
    tmp = np.float32(1) - x * x / b2  # float arithmetic, as vk::TukeyWeightFunction
    w = np.where(x * x <= b2, tmp * tmp, np.float32(0)).astype(np.float64)
    zi, X, Y = 1 / p[:, 2], p[:, 0], p[:, 1]
    J0 = np.stack([-zi, 0 * zi, X * zi * zi, Y * X * zi * zi, -(1 + X * X * zi * zi), Y * zi], 1) * sic[:, None]
    J1 = np.stack([0 * zi, -zi, Y * zi * zi, 1 + Y * Y * zi * zi, -(Y * X * zi * zi), -X * zi], 1) * sic[:, None]
    b = -((J0.T * w) @ e[:, 0] + (J1.T * w) @ e[:, 1])
    return (J0.T * w) @ J0 + (J1.T * w) @ J1, b


def se3_log(T):
    """Inverse of the SE(3) exponential the optimizer applies (xi = [v, omega], rotation angle < pi)."""
    R, t = T[:, :3], T[:, 3]
    th = np.arccos(np.clip((np.trace(R) - 1) / 2, -1.0, 1.0))
    vee = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / 2
    w = vee * (th / np.sin(th) if th > 1e-8 else 1.0)
    W = synth.hat(w)
    if th > 1e-8:
        V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * W + (th - np.sin(th)) / th ** 3 * W @ W
    else:
        V = np.eye(3) + W / 2
    return np.concatenate([np.linalg.solve(V, t), w])


def first_step(c, T):
    """The step dT of a one-iteration run that ended at T = exp(dT) * T_init."""
    return se3_log(synth.se3_mul(T, synth.se3_inv(c["T_init"])))


def min_pivot_ratio(A):
    """Smallest pivot of the unpivoted LDL^T of A over A's largest |diagonal| (the quantity fact6_compute_upper tests)."""
    d, L = np.zeros(6), np.eye(6)
    for j in range(6):
        d[j] = A[j, j] - sum(L[j, k] ** 2 * d[k] for k in range(j))
        for i in range(j + 1, 6):
            L[i, j] = (A[i, j] - sum(L[i, k] * L[j, k] * d[k] for k in range(j))) / d[j]
    return d.min() / np.abs(np.diag(A)).max()


def degenerate_cases():
    """(name, case) of the degenerate frames; tests/test_edge_pins.py pins the oracle against the reference on the same."""
    out = []
    for n in (1, 2):
        c = synth.make_pose_opt_case(200 + n, n=8, width=752, height=480, px_noise=0.5, outlier_frac=0.0)
        c["has_point"][:] = 0
        c["has_point"][:n] = 1
        out.append((f"{n}obs", c))
    out.append(("line", synth.make_pose_line_case(3, 50)))
    for w in (20.0, 4.0, 1.0):
        out.append((f"window{w}", synth.make_pose_window_case(5, 60, w, px_noise=0.003)))
    return out


def pivot_sweep_cases():
    """degenerate_cases() and two windows small enough (0.3, 0.2 px) that A's smallest pivot falls below the 1e-13 test
    while staying clearly positive.  At cond(A) ~ 1e17 the step is rounding noise in every implementation: these are for
    the choice of path and for one iteration, not for the pose after ten."""
    return degenerate_cases() + [(f"window{w}", synth.make_pose_window_case(5, 60, w, px_noise=0.003)) for w in (0.3, 0.2)]



def backward_error(A, b, x):
    """|A x - b| / (|A| |x| + |b|): small for any backward-stable solve of A x = b however ill-conditioned A is, O(1) for a
    wrong one (a wrong permutation, a dropped pivot)."""
    return np.linalg.norm(A @ x - b) / (np.linalg.norm(A, 2) * np.linalg.norm(x) + np.linalg.norm(b))


def zero_error_case(n, n_off=3, seed=0):
    """A frame whose reprojection errors are exactly 0 for all but n_off observations: T_init = identity and every point is
    its bearing times a power of two, so project2d(T * pos) = project2d(f) to the last bit.  The median error, and with it
    the MAD scale, is exactly 0; every Tukey weight divides an error by 0."""
    rng = np.random.default_rng(seed)
    cam = synth.camera_for(752, 480)
    px = np.stack([rng.uniform(20, 732, n), rng.uniform(20, 460, n)], axis=1)
    f = cam.cam2world(px)
    pos = f * (2.0 ** rng.integers(1, 5, n))[:, None]
    f[:n_off] = cam.cam2world(px[:n_off] + rng.uniform(3, 6, (n_off, 2)))  # a few observations with a real error
    return dict(cam=cam, f=f, pos=pos, level=rng.integers(0, 3, n).astype(np.int32), has_point=np.ones(n, np.uint8),
                T_init=synth.se3_identity(), T_true=synth.se3_identity())
