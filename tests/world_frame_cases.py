"""World-frame cases: camera rotations R_f_w that reach every branch of the rotation-matrix-to-quaternion conversion, the
re-expression of the synth cases in another world frame, and a high-precision statement of the conversion's round trip.

Every kernel that takes a world pose converts the caller's row-major [R|t] into a quaternion (pose_from_rt12 ->
qfrommatrix, svo_math.cuh; se3_from_rt12 -> qfrommatrix in the oracle).  Shoemake's conversion has four branches: the trace
branch (R00 + R11 + R22 > 0) and one branch for each largest diagonal entry (x, y, z; a tie goes to the first of the tied
entries, in that order).  The synth scenes look down at a plane from a camera near diag(1, -1, -1): every pose they make
takes the x branch.  A camera that has turned around (yawed by more than 120 degrees about its own y axis from the first
keyframe, which is SVO's world frame) takes the y branch; one rolled over takes the z branch.

CATALOGUE lists target rotations R_f_w, exact matrices where possible, each with the branch it takes and the edge it
reaches; CATALOGUE_F32 repeats every entry with R rounded to float32 (non-orthonormal by ~1e-8, as a host that stores its
poses in float passes them).  `frame_for` builds the change of world frame G that puts a case's current camera on one of
them; `reframe` applies it to a case.  `hp_roundtrip` is pose_to_rt12(pose_from_rt12(T)) in mpmath at 40 digits;
`ieee_roundtrip` is the same sequence of double operations as the kernels and the oracle, one branch forced, so that a
result can be traced to the branch that made it bit for bit.
"""
from __future__ import annotations

import math

import numpy as np
from mpmath import mp, mpf

from rpg_svo_b200 import synth

BRANCHES = ("trace", "x", "y", "z")
U = 2.0 ** -53
# |R_roundtrip - R_exact| per entry, in units of u = 2^-53.  The conversion picks the branch whose pivot is the largest
# quaternion component (>= 1/2), so every quotient is well conditioned: ~4 roundings reach each quaternion component, ~6
# more each entry of toRotationMatrix.  The catalogue's largest is 3.1 u; 8 u leaves room, and a wrong index or sign moves an
# entry by ~0.1 or more.
ROUNDTRIP_ULP = 8
# |R_roundtrip - R_input|: the round trip returns the rotation nearest the input only to first order.  Exactly orthonormal
# double input comes back within rounding; float32-rounded input (off by ~6e-8 per entry) comes back within that distance.
INPUT_TOL_F64 = 32 * U
INPUT_TOL_F32 = 4e-7


def _rot_mp(axis, angle):
    """Rodrigues' rotation in mpmath, rounded to double entry by entry."""
    with mp.workdps(40):
        a = [mpf(x) for x in axis]
        n = mp.sqrt(sum(x * x for x in a))
        a = [x / n for x in a]
        th = mpf(angle) if not isinstance(angle, mpf) else angle
        c, s = mp.cos(th), mp.sin(th)
        K = [[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]]
        R = [[(c if i == j else 0) + (1 - c) * a[i] * a[j] + s * K[i][j] for j in range(3)] for i in range(3)]
        return np.array([[float(R[i][j]) for j in range(3)] for i in range(3)])


def _yaw(c: float) -> np.ndarray:
    """Rotation about y with cos = c (double), sin = sqrt(1 - c^2) rounded: R11 = 1 exactly."""
    s = math.sqrt(1.0 - c * c)
    return np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])


def _catalogue():
    with mp.workdps(40):  # every angle at 40 digits, whatever mp.dps the importing process has set
        return _catalogue_entries(+mp.pi)


def _catalogue_entries(pi):
    deg = lambda d: mpf(d) * pi / 180
    e = []  # (name, R, branch, edge)
    e.append(("near_identity", _rot_mp((0.3, -0.7, 0.5), 0.02), "trace", "trace_branch"))
    e.append(("default_x", synth.base_pose()[:, :3].copy(), "x", "x_branch"))
    e.append(("yaw_180", np.diag([-1.0, 1.0, -1.0]), "y", "w_zero"))
    e.append(("yaw_150", _rot_mp((0, 1, 0), deg(150)), "y", "y_branch"))
    # 120 degrees about y: trace 1 + 2c = 0; c = -1/2 +- 2^-53 makes it +-2^-52, and R00 + R11 + R22 is exact in double
    e.append(("yaw_120_trace_plus_ulp", _yaw(-0.5 + 2.0 ** -53), "trace", "trace_positive_ulp"))
    e.append(("yaw_120_trace_zero", _yaw(-0.5), "y", "trace_zero"))
    e.append(("yaw_120_trace_minus_ulp", _yaw(-0.5 - 2.0 ** -53), "y", "trace_negative_ulp"))
    e.append(("roll_180", np.diag([-1.0, -1.0, 1.0]), "z", "w_zero"))
    e.append(("roll_150_tilted", _rot_mp((0.1, -0.05, 1.0), deg(150)), "z", "z_branch"))
    # 180 degrees about (1,1,0)/sqrt2, (0,1,1)/sqrt2, (1,0,1)/sqrt2: R = 2 n n^T - I, two diagonal entries tie at 0
    e.append(("tie_xy_180", np.array([[0.0, 1, 0], [1, 0, 0], [0, 0, -1]]), "x", "tie_xy"))
    e.append(("tie_yz_180", np.array([[-1.0, 0, 0], [0, 0, 1], [0, 1, 0]]), "y", "tie_yz"))
    e.append(("tie_xz_180", np.array([[0.0, 0, 1], [0, -1, 0], [1, 0, 0]]), "x", "tie_xz"))
    # the same ties broken by 2e-9 each way
    for name, axis, br in (("tie_xy_x_ahead", (1 + 1e-9, 1, 0), "x"), ("tie_xy_y_ahead", (1, 1 + 1e-9, 0), "y"),
                           ("tie_yz_y_ahead", (0, 1 + 1e-9, 1), "y"), ("tie_yz_z_ahead", (0, 1, 1 + 1e-9), "z"),
                           ("tie_xz_x_ahead", (1 + 1e-9, 0, 1), "x"), ("tie_xz_z_ahead", (1, 0, 1 + 1e-9), "z")):
        e.append((name, _rot_mp(axis, pi), br, "near_tie"))
    # 120 degrees about (1,1,1)/sqrt3: a cyclic permutation, trace exactly 0, all three diagonal entries tie
    e.append(("perm_120", np.array([[0.0, 0, 1], [1, 0, 0], [0, 1, 0]]), "x", "tie_xyz"))
    # pi - 1e-9 about a generic axis: w ~ 5e-10
    e.append(("near_pi_z", _rot_mp((0.3, -0.5, 0.8), pi - mpf("1e-9")), "z", "near_pi"))
    e.append(("near_pi_y", _rot_mp((0.36, 0.8, -0.48), pi - mpf("1e-9")), "y", "near_pi"))
    return [dict(name=n, R=np.ascontiguousarray(R, np.float64), branch=b, edge=ed, f32=False) for n, R, b, ed in e]


CATALOGUE = _catalogue()
CATALOGUE_F32 = [dict(c, name=c["name"] + "_f32", R=c["R"].astype(np.float32).astype(np.float64), branch=None, f32=True)
                 for c in CATALOGUE]
ALL = CATALOGUE + CATALOGUE_F32
BY_NAME = {c["name"]: c for c in ALL}
EDGES = ("trace_branch", "x_branch", "y_branch", "z_branch", "w_zero", "trace_positive_ulp", "trace_zero",
         "trace_negative_ulp", "tie_xy", "tie_yz", "tie_xz", "tie_xyz", "near_tie", "near_pi")
# frames the oracle-vs-reference pins use: the y and z branches, a tie, trace 0 and near pi
PIN_FRAMES = ("yaw_150", "roll_150_tilted", "tie_yz_180", "perm_120", "near_pi_z")
FAR_ORIGIN = (120.0, -80.0, 45.0)  # the canonical origin ~151 m from the new one


def rt12(R, t=(0.0, 0.0, 0.0)) -> np.ndarray:
    return np.hstack([np.asarray(R, np.float64), np.asarray(t, np.float64).reshape(3, 1)])


# ------------------------------------------------------------------------------------------------ the conversion
def hp_roundtrip(T) -> dict:
    """pose_to_rt12(pose_from_rt12(T)) at 40 digits from the exact double entries of T: the branch (trace if
    R00 + R11 + R22 > 0, else the largest diagonal entry, the first of tied ones), Shoemake's formulas, normalisation,
    toRotationMatrix.  Returns dict(R = 3x3 of mpf, branch, q = (w, x, y, z) of mpf, trace = mpf)."""
    T = np.asarray(T, np.float64).reshape(3, -1)
    with mp.workdps(40):
        R = [[mpf(float(T[i, j])) for j in range(3)] for i in range(3)]
        tr = R[0][0] + R[1][1] + R[2][2]
        if tr > 0:
            br = "trace"
            s = mp.sqrt(tr + 1)
            w = s / 2
            s = 1 / (2 * s)
            x, y, z = (R[2][1] - R[1][2]) * s, (R[0][2] - R[2][0]) * s, (R[1][0] - R[0][1]) * s
        else:
            i = 0 if (R[0][0] >= R[1][1] and R[0][0] >= R[2][2]) else (1 if R[1][1] >= R[2][2] else 2)
            br = "xyz"[i]
            j, k = (i + 1) % 3, (i + 2) % 3
            s = mp.sqrt(R[i][i] - R[j][j] - R[k][k] + 1)
            qv = [None] * 3
            qv[i] = s / 2
            s = 1 / (2 * s)
            w = (R[k][j] - R[j][k]) * s
            qv[j] = (R[j][i] + R[i][j]) * s
            qv[k] = (R[k][i] + R[i][k]) * s
            x, y, z = qv
        n = mp.sqrt(w * w + x * x + y * y + z * z)
        w, x, y, z = w / n, x / n, y / n, z / n
        Rq = [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
              [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
              [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]
        return dict(R=Rq, branch=br, q=(w, x, y, z), trace=tr)


def ulp_error(R_out, hp) -> float:
    """max |R_out - R_hp| over the nine entries, in units of u = 2^-53 (NaN if R_out has a NaN)."""
    R_out = np.asarray(R_out, np.float64).reshape(3, -1)
    if not np.all(np.isfinite(R_out[:, :3])):
        return float("nan")
    with mp.workdps(40):
        return max(float(abs(mpf(float(R_out[i, j])) - hp["R"][i][j]) / mpf(U)) for i in range(3) for j in range(3))


def ieee_roundtrip(T, branch: str, n_normalize: int = 1) -> np.ndarray:
    """qfrommatrix with `branch` forced, qnormalized (n_normalize times), qmatrix: the double operations of svo_math.cuh /
    oracle_math.h in their order (contraction off, correctly rounded sqrt and division).  Returns the 3x3 rotation.
    pose_from_rt12 / se3_from_rt12 normalise once; the oracle's se3_mul(T, I) normalises the product q * 1 again (SE3's
    operator*), which can move the last bit of a component."""
    T = np.asarray(T, np.float64).reshape(3, -1)
    R = [np.float64(T[i, j]) for i in range(3) for j in range(3)]
    h, one = np.float64(0.5), np.float64(1.0)
    with np.errstate(all="ignore"):
        if branch == "trace":
            t = np.sqrt(R[0] + R[4] + R[8] + one)
            w = h * t
            t = h / t
            x, y, z = (R[7] - R[5]) * t, (R[2] - R[6]) * t, (R[3] - R[1]) * t
        elif branch == "x":
            t = np.sqrt(R[0] - R[4] - R[8] + one)
            x = h * t
            t = h / t
            w, y, z = (R[7] - R[5]) * t, (R[3] + R[1]) * t, (R[6] + R[2]) * t
        elif branch == "y":
            t = np.sqrt(R[4] - R[8] - R[0] + one)
            y = h * t
            t = h / t
            w, z, x = (R[2] - R[6]) * t, (R[7] + R[5]) * t, (R[1] + R[3]) * t
        else:
            t = np.sqrt(R[8] - R[0] - R[4] + one)
            z = h * t
            t = h / t
            w, x, y = (R[3] - R[1]) * t, (R[6] + R[2]) * t, (R[7] + R[5]) * t
        for _ in range(n_normalize):
            n = np.sqrt(w * w + x * x + y * y + z * z)
            w, x, y, z = w / n, x / n, y / n, z / n
        two = np.float64(2.0)
        tx, ty, tz = two * x, two * y, two * z
        twx, twy, twz = tx * w, ty * w, tz * w
        txx, txy, txz = tx * x, ty * x, tz * x
        tyy, tyz, tzz = ty * y, tz * y, tz * z
        return np.array([[one - (tyy + tzz), txy - twz, txz + twy],
                         [txy + twz, one - (txx + tzz), tyz - twx],
                         [txz - twy, tyz + twx, one - (txx + tyy)]])


def branches_matching(T_out, T_in, n_normalize: int = 1) -> list:
    """The branches whose ieee_roundtrip of T_in equals T_out's rotation bit for bit."""
    got = np.ascontiguousarray(np.asarray(T_out, np.float64).reshape(3, -1)[:, :3])
    return [b for b in BRANCHES if np.array_equal(ieee_roundtrip(T_in, b, n_normalize).view(np.int64), got.view(np.int64))]


# ------------------------------------------------------------------------------------------------ change of world frame
CURRENT = {"pose": "T_init", "match": "T_cur_w", "depth": "T_cur_w", "map": "cur_T_f_w"}


def frame_for(T_cur_w, R_target, origin=(0.0, 0.0, 0.0)) -> np.ndarray:
    """G = [R_G | origin] with R_cur R_G^T = R_target: in the world frame G, the camera T_cur_w has the rotation R_target
    (to rounding; `reframe` makes it exact), and the canonical world origin sits at `origin`."""
    R_G = np.asarray(R_target).T @ np.asarray(T_cur_w)[:, :3]
    return rt12(R_G, origin)


def _pts(G, p):
    p = np.asarray(p, np.float64)
    return np.ascontiguousarray(p @ G[:, :3].T + G[:, 3])


def _pose(T, Ginv):
    return synth.se3_mul(np.asarray(T, np.float64), Ginv)


def reframe(case: dict, kind: str, R_target, origin=(0.0, 0.0, 0.0)) -> tuple[dict, np.ndarray]:
    """The synth case `case` (kind: pose / match / depth / map) re-expressed in the world frame G = frame_for(current camera,
    R_target, origin): every T_f_w becomes T_f_w G^-1, every world point G p.  Images, pixels, bearings and seeds stay as
    they are.  The current camera's rotation is then set to R_target exactly (it differs by rounding).  Returns (case, G)."""
    cur_key = CURRENT[kind]
    G = frame_for(case[cur_key], R_target, origin)
    Ginv = synth.se3_inv(G)
    out = dict(case)
    out.pop("plane", None)  # a canonical-frame object
    for k in ("T_init", "T_true", "T_ref_w", "T_cur_w", "cur_T_f_w"):
        if k in out:
            out[k] = _pose(out[k], Ginv)
    if "kf_T" in out:
        out["kf_T"] = [_pose(T, Ginv) for T in out["kf_T"]]
    for k in ("pos", "point_pos", "ref_pos"):
        if k in out:
            out[k] = _pts(G, out[k])
    if "view" in out:
        v = dict(out["view"])
        v["kf_T_f_w"] = np.stack([_pose(T, Ginv) for T in v["kf_T_f_w"]])
        v["kf_keypt_pos"] = _pts(G, v["kf_keypt_pos"].reshape(-1, 3)).reshape(v["kf_keypt_pos"].shape)
        v["pt_pos"] = _pts(G, v["pt_pos"])
        out["view"] = v
    Rt = np.asarray(R_target, np.float64)
    assert np.max(np.abs(out[cur_key][:, :3] - Rt)) < 1e-14
    out[cur_key] = out[cur_key].copy()
    out[cur_key][:, :3] = Rt
    return out, G


def to_canonical(T_f_w, G) -> np.ndarray:
    """A pose of frame G mapped back to the canonical world frame: T_f_w G."""
    return synth.se3_mul(np.asarray(T_f_w, np.float64), G)


# ------------------------------------------------------------------------------------------------ the canonical cases
def pose_case(seed: int = 11):
    return synth.make_pose_opt_case(seed, n=300, width=752, height=480)


def match_case(seed: int = 21):
    return synth.make_match_case(seed, 120)


def depth_case(seed: int = 31):
    c = synth.make_depth_case(seed, n_seeds=300, baseline=0.3)
    c["seeds"]["sigma2"][::5] *= np.float32(1e-3)   # some seeds close to convergence
    c["seeds"]["mu"][::5] = (1.0 / c["depth_gt"][::5]).astype(np.float32)
    return c


def map_case(seed: int = 41):
    return synth.make_map_case(seed, n_kfs=5, n_points=300, n_candidates=30)
