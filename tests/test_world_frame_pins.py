"""CPU: the oracle's rotation-matrix-to-quaternion conversion on every branch and edge of tests/world_frame_cases.py, against
the 40-digit statement of the round trip, and the oracle against the compiled reference (recorded in
tests/golden/ref/test_world_frame_pins.npz) for the pose optimizer, the depth filter and the reprojector on synth cases
re-expressed in world frames whose current camera takes the y branch, the z branch, a tie, trace 0 and near pi."""
import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import world_frame_cases as wf
from tests.ref_golden import ref  # noqa: F401 (fixture)

I12 = wf.rt12(np.eye(3))
T_OFF = (0.3, -1.2, 2.0)
NAMES = [c["name"] for c in wf.ALL]


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _po_roundtrip(oracle, T):
    """The oracle's bare round trip se3_to_rt12(se3_from_rt12(T)): pose_optimize with no iteration and an observation."""
    c = _po_roundtrip.case
    return oracle.pose_optimize(2.0, 0, c["cam"].fx, T, c["f"][:8], c["pos"][:8], c["level"][:8], np.ones(8, np.uint8))["T"]


_po_roundtrip.case = synth.make_pose_opt_case(3, n=8, width=752, height=480)


def test_catalogue_reaches_every_branch_and_edge():
    """Each entry takes the branch it is labelled with in the 40-digit statement; together they take all four branches and
    reach every edge.  The branch is chosen from the exact entries: for every entry the double sum R00 + R11 + R22 has the
    sign of the exact trace, so the exact choice is the one a double implementation faces."""
    seen_b, seen_e = set(), set()
    for c in wf.CATALOGUE:
        hp = wf.hp_roundtrip(wf.rt12(c["R"]))
        assert hp["branch"] == c["branch"], c["name"]
        R = c["R"]
        fl_tr = (R[0, 0] + R[1, 1]) + R[2, 2]
        assert (fl_tr > 0) == (hp["trace"] > 0) and (fl_tr == 0) == (hp["trace"] == 0), c["name"]
        seen_b.add(hp["branch"])
        seen_e.add(c["edge"])
    assert seen_b == set(wf.BRANCHES)
    assert seen_e == set(wf.EDGES)
    by = wf.BY_NAME
    assert float(wf.hp_roundtrip(wf.rt12(by["yaw_120_trace_plus_ulp"]["R"]))["trace"]) == 2.0 ** -52
    assert float(wf.hp_roundtrip(wf.rt12(by["yaw_120_trace_minus_ulp"]["R"]))["trace"]) == -2.0 ** -52
    for n in ("yaw_180", "roll_180", "tie_xy_180", "tie_yz_180", "tie_xz_180"):
        assert wf.hp_roundtrip(wf.rt12(by[n]["R"]))["q"][0] == 0, n                     # w = 0 exactly
    for n in ("near_pi_z", "near_pi_y"):
        assert 4e-10 < abs(float(wf.hp_roundtrip(wf.rt12(by[n]["R"]))["q"][0])) < 6e-10, n
    f32_branches = {wf.hp_roundtrip(wf.rt12(c["R"]))["branch"] for c in wf.CATALOGUE_F32}
    assert f32_branches == set(wf.BRANCHES)
    off = [np.max(np.abs(c["R"] @ c["R"].T - np.eye(3))) for c in wf.CATALOGUE_F32]
    assert max(off) < 1e-6 and sum(x > 1e-9 for x in off) >= 8


@pytest.mark.parametrize("name", NAMES)
def test_oracle_roundtrip_within_bound_of_hp(oracle, name):
    """se3_mul(T, I) and the bare round trip stay within ROUNDTRIP_ULP of the 40-digit round trip, keep the translation
    bit for bit, and come back to the input rotation within INPUT_TOL_F64 (exact rotations) or INPUT_TOL_F32
    (float32-rounded ones, non-orthonormal by ~1e-8)."""
    c = wf.BY_NAME[name]
    T = wf.rt12(c["R"], T_OFF)
    hp = wf.hp_roundtrip(T)
    tol_in = wf.INPUT_TOL_F32 if c["f32"] else wf.INPUT_TOL_F64
    for who, out in (("se3_mul", oracle.se3_mul(T, I12)), ("bare", _po_roundtrip(oracle, T))):
        err = wf.ulp_error(out, hp)
        assert err <= wf.ROUNDTRIP_ULP, (who, err)
        assert np.max(np.abs(out[:, :3] - c["R"])) <= tol_in, who
        assert np.array_equal(_bits(out[:, 3]), _bits(T[:, 3])), who


def test_oracle_takes_the_branch_hp_reports(oracle):
    """The branch the oracle took, traced bit for bit: its output equals ieee_roundtrip of exactly one branch where the
    branches' roundings differ, and that branch is the one hp_roundtrip reports -- for all four branches, both orders of
    each near tie, the exact ties, trace 0 and the float32-rounded entries."""
    unique, taken = 0, set()
    for c in wf.ALL:
        T = wf.rt12(c["R"], T_OFF)
        br = wf.hp_roundtrip(T)["branch"]
        for out, n_norm in ((oracle.se3_mul(T, I12), 2), (_po_roundtrip(oracle, T), 1)):
            m = wf.branches_matching(out, T, n_norm)
            assert br in m, (c["name"], br, m)
            if m == [br]:
                unique += 1
                taken.add(br)
    assert taken == set(wf.BRANCHES)
    assert unique >= 2 * (len(wf.ALL) - 6), unique   # only trace 0 (trace == y) and the permutation (all equal) are ambiguous


@pytest.mark.parametrize("base", ["near_identity", "default_x", "yaw_150", "roll_150_tilted", "tie_xy_180", "perm_120"])
def test_oracle_nan_entry_gives_an_all_nan_rotation(oracle, base):
    """A NaN in any one of the nine rotation entries makes the whole quaternion NaN (normalisation spreads it), whichever
    branch the finite entries would take."""
    for k in range(9):
        R = wf.BY_NAME[base]["R"].copy()
        R.reshape(-1)[k] = np.nan
        T = wf.rt12(R, T_OFF)
        out = oracle.se3_mul(T, I12)
        assert np.all(np.isnan(out)), (k, out)
        assert np.all(np.isnan(_po_roundtrip(oracle, T)[:, :3])), k


# ---- the oracle against the compiled reference in turned-around world frames ------------------------------------------
@pytest.fixture(scope="module")
def canonical():
    return dict(pose=wf.pose_case(), depth=wf.depth_case(), map=wf.map_case())


@pytest.mark.parametrize("frame", wf.PIN_FRAMES)
def test_reframed_oracle_equals_reference(oracle, canonical, frame, ref):
    """pose_optimizer::optimizeGaussNewton, DepthFilter::updateSeeds and Reprojector::reprojectMap of the compiled
    reference against the oracle, on cases whose current camera sits on the catalogue rotation `frame`, the world origin
    150 m away: the contract of the canonical-frame pins (tests/test_oracle_pins.py)."""
    R = wf.BY_NAME[frame]["R"]
    origin = wf.FAR_ORIGIN
    # pose optimizer
    c, _ = wf.reframe(canonical["pose"], "pose", R, origin)
    r = ref.pose_optimize(2.0, 10, c["cam"], c["T_init"], c["f"], c["pos"], c["level"], c["has_point"])
    o = oracle.pose_optimize(2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], c["has_point"])
    assert np.array_equal(r["has_point"], o["has_point"]) and r["num_obs"] == o["num_obs"]
    assert np.allclose(r["T"], o["T"], rtol=0, atol=1e-10)
    for k in ("estimated_scale", "error_init", "error_final"):
        assert np.isclose(r[k], o[k], rtol=1e-9), k
    # depth filter
    c, _ = wf.reframe(canonical["depth"], "depth", R, origin)
    r = ref.depth_filter_update([c["ref_pyr"][0]], [c["T_ref_w"]], c["cur_pyr"][0], c["T_cur_w"], c["n_levels"], c["cam"],
                                c["ref_index"], c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"],
                                c["batch_id"], c["batch_counter"], c["seeds"])
    o = oracle.depth_filter_update([c["ref_pyr"]], [c["T_ref_w"]], c["cur_pyr"], c["T_cur_w"], c["cam"], c["ref_index"],
                                   c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"],
                                   c["batch_counter"], c["seeds"])
    st = o["status"]
    expect = np.where(st == 6, 1, np.where((st == 1) | (st == 7), 2, 0))
    assert np.array_equal(r["status"], expect)
    assert (st == 6).sum() > 5 and (st == 5).sum() > 50
    keep = expect == 0
    for k in ("a", "b", "mu", "z_range", "sigma2"):
        assert np.array_equal(r[k][keep].view(np.uint32), o[k][keep].view(np.uint32)), k
    conv = expect == 1
    assert np.array_equal(r["sigma2"][conv].view(np.uint32), o["sigma2"][conv].view(np.uint32))
    Tinv = synth.se3_inv(c["T_ref_w"])
    xyz = (c["ftr_f"][conv] / o["mu"][conv][:, None].astype(np.float64)) @ Tinv[:, :3].T + Tinv[:, 3]
    assert np.allclose(r["xyz_world"][conv], xyz, rtol=0, atol=1e-9)
    # reprojector
    c, _ = wf.reframe(canonical["map"], "map", R, origin)
    o, r = oracle.reproject_map(c), ref.reproject_map(c)
    for k in ("n_matches", "n_trials", "n_new", "n_overlap"):
        assert o[k] == r[k], k
    for k in ("overlap_kf", "overlap_count", "new_point", "new_level", "new_type", "pt_type", "pt_n_failed", "pt_n_succeeded"):
        assert np.array_equal(o[k], r[k]), k
    assert np.max(np.abs(o["new_px"] - r["new_px"]), initial=0.0) == 0.0
    assert np.allclose(o["new_grad"], r["new_grad"], rtol=0, atol=1e-9)
    assert np.array_equal(np.minimum(o["pt_action"], 2), np.minimum(r["pt_action"], 2))
    assert o["n_matches"] > 30
