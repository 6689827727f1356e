"""GPU parity: pose_optimizer and DepthFilter kernels vs the CPU oracle."""
import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import depth_update_hp as dhp
from tests import point_hp

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,size", [(1000, (1920, 1080)), (120, (752, 480)), (7, (640, 480))])
def test_pose_optimize_matches_oracle(ctx, oracle, n, size):
    c = synth.make_pose_opt_case(5 + n, n, *size)
    g = ctx.pose_optimize(2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], c["has_point"])
    o = oracle.pose_optimize(2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], c["has_point"])
    assert np.array_equal(g["has_point"], o["has_point"])  # culling mask bit-exact
    assert g["num_obs"] == o["num_obs"] and g["n_iter_done"] == o["n_iter_done"]
    dt, dr = synth.pose_error(g["T"], o["T"])
    assert dt < 1e-8 and dr < 1e-8, (dt, dr)
    for k in ("estimated_scale", "error_init", "error_final"):
        assert abs(g[k] - o[k]) <= 1e-9 * max(1.0, abs(o[k])), k
    assert np.allclose(g["cov"], o["cov"], rtol=1e-6, atol=1e-12)
    if n >= 100:
        assert synth.pose_error(g["T"], c["T_true"])[0] < 5e-3  # the optimiser recovers the pose


def test_pose_optimize_batch_equals_single_calls(ctx, oracle):
    """svo_b200_pose_optimize_batch: frames of different sizes (one without observations) in one launch give exactly
    what single calls give, and match the oracle."""
    cases = [synth.make_pose_opt_case(40 + k, n, *size) for k, (n, size) in
             enumerate([(1000, (1920, 1080)), (120, (752, 480)), (9, (640, 480)), (300, (640, 480))])]
    cases[2]["has_point"][:] = 0
    off = np.concatenate([[0], np.cumsum([len(c["level"]) for c in cases])]).astype(np.int32)
    cat = lambda k: np.concatenate([c[k] for c in cases])
    res = ctx.pose_optimize_batch(2.0, 10, [c["cam"].fx for c in cases], np.stack([c["T_init"] for c in cases]), off,
                                  cat("f"), cat("pos"), cat("level"), cat("has_point"))
    for c, r in zip(cases, res):
        g = ctx.pose_optimize(2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], c["has_point"])
        assert np.array_equal(r["T"], g["T"]) and np.array_equal(r["has_point"], g["has_point"])
        assert (r["num_obs"], r["n_iter_done"], r["error_final"]) == (g["num_obs"], g["n_iter_done"], g["error_final"])
        o = oracle.pose_optimize(2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], c["has_point"])
        assert np.array_equal(r["has_point"], o["has_point"]) and r["num_obs"] == o["num_obs"]
        dt, dr = synth.pose_error(r["T"], o["T"])
        assert dt < 1e-8 and dr < 1e-8


def test_pose_optimize_ties_and_tiny_sets(ctx, oracle):
    """The median select with repeated values (identical observations) and with 1..3 observations."""
    c = synth.make_pose_opt_case(77, 64, 752, 480)
    for k in ("f", "pos", "level"):
        c[k][32:] = c[k][:32]  # every observation twice: the order statistics see ties everywhere
    for n in (64, 3, 2, 1):
        hp = c["has_point"].copy(); hp[:] = 0; hp[:n] = 1
        g = ctx.pose_optimize(2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], hp)
        o = oracle.pose_optimize(2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], hp)
        assert g["num_obs"] == o["num_obs"] and np.array_equal(g["has_point"], o["has_point"]), n
        for key in ("estimated_scale", "error_init", "error_final"):
            assert abs(g[key] - o[key]) <= 1e-9 * max(1.0, abs(o[key])), (n, key)
        # with 1-2 observations A is singular (rank 2 / 4): its smallest pivots are rounding noise that the pivoted LDL^T
        # divides by, in the kernel as in the oracle, so the step -- and the iteration at which chi2 stops falling -- is
        # decided by each implementation's summation order, and so is whether the Gauss-Jordan inverse meets an exactly
        # zero pivot (NaN covariance) or a 1e-30 one (huge finite entries); pose and covariance are compared at full rank
        if n >= 3:
            assert g["n_iter_done"] == o["n_iter_done"], n
            dt, dr = synth.pose_error(g["T"], o["T"])
            assert dt < 1e-8 and dr < 1e-8, (n, dt, dr)
            assert np.array_equal(np.isfinite(g["cov"]), np.isfinite(o["cov"])), n


def test_pose_optimize_no_observations(ctx):
    c = synth.make_pose_opt_case(3, 16, 640, 480)
    hp = np.zeros(16, np.uint8)
    g = ctx.pose_optimize(2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], hp)
    assert g["num_obs"] == 0 and np.allclose(g["T"], c["T_init"])


@pytest.mark.parametrize("n_seeds,baseline", [(2000, 0.3), (300, 0.05), (300, 0.6)])
def test_depth_filter_update_matches_oracle(ctx, oracle, n_seeds, baseline):
    c = synth.make_depth_case(31 + n_seeds, n_seeds, baseline=baseline)
    ref, cur = ctx.frame(c["ref_pyr"]), ctx.frame(c["cur_pyr"])
    g = ctx.depth_filter_update([ref], [c["T_ref_w"]], cur, c["T_cur_w"], c["cam"], c["ref_index"], c["ftr_px"],
                                c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"],
                                c["batch_counter"], c["seeds"])
    o = oracle.depth_filter_update([c["ref_pyr"]], [c["T_ref_w"]], c["cur_pyr"], c["T_cur_w"], c["cam"],
                                   c["ref_index"], c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"],
                                   c["ftr_grad"], c["batch_id"], c["batch_counter"], c["seeds"])
    assert np.array_equal(g["status"], o["status"])      # per-seed outcome bit-exact
    assert np.array_equal(g["n_zmssd"], o["n_zmssd"])    # same pixels scored along the epipolar line
    upd = o["status"] >= 5
    assert upd.sum() > 0.3 * n_seeds
    assert np.max(np.abs(g["px_cur"][upd] - o["px_cur"][upd])) <= 1e-4
    assert np.allclose(g["z"][upd], o["z"][upd], rtol=1e-6)
    dhp.assert_seed_updates(g, o, c["seeds"], [c["T_ref_w"]], c["ref_index"], c["T_cur_w"], c["ftr_f"], c["cam"].fx, oracle)
    # the measurements are real: triangulated depth close to the plane depth
    assert np.median(np.abs(g["z"][upd] - c["depth_gt"][upd])) < 0.05
    ref.destroy(); cur.destroy()


def test_point_optimize_batch_matches_oracle(ctx, oracle):
    """Point::optimize ("next" row f3): 200 points seen from 2..6 keyframes with noisy bearings."""
    rng = np.random.default_rng(17)
    cam = synth.camera_for(752, 480)
    n_frames, P = 6, 200
    poses = [synth.se3_mul(synth.se3_exp(np.concatenate([rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.05, 0.05, 3)])),
                           synth.base_pose()) for _ in range(n_frames)]
    plane = synth.Plane.tilted()
    px = np.stack([rng.uniform(150, 600, P), rng.uniform(100, 380, P)], axis=1)
    truth = synth.intersect(plane, poses[0], cam.cam2world(px))
    pos0 = truth + rng.normal(0, 0.02, (P, 3))
    offs, frs, fs = [0], [], []
    for p in range(P):
        k = int(rng.integers(2, n_frames + 1))
        for fr in rng.choice(n_frames, k, replace=False):
            T = poses[fr]
            pc = T[:, :3] @ truth[p] + T[:, 3]
            pxo = cam.world2cam(pc) + rng.normal(0, 0.3, 2)
            frs.append(fr); fs.append(cam.cam2world(pxo))
        offs.append(len(frs))
    frs, fs = np.array(frs, np.int32), np.array(fs)
    g = ctx.point_optimize_batch(5, pos0, offs, frs, fs, poses)
    for p in range(P):
        Ts = [poses[i].reshape(12) for i in frs[offs[p]:offs[p + 1]]]
        o = oracle.point_optimize(5, pos0[p], Ts, fs[offs[p]:offs[p + 1]])
        # against the exact iteration (tests/point_hp.py): each within the bound of a run it may take -- the exact one
        # where every decision is decisive; two-view points are ill-conditioned along the ray (cond up to ~1e6), and the
        # bound scales with cond(A)
        runs = point_hp.branches(5, pos0[p], Ts, fs[offs[p]:offs[p + 1]])
        for who, x in (("kernel", g[p]), ("oracle", o)):
            run, ratio = point_hp.match_any(x, runs)
            assert run is not None and point_hp.defined(run), (p, who, ratio)
            assert run is runs[0] or not point_hp.decisive(runs[0]), (p, who)
    assert np.median(np.linalg.norm(g - truth, axis=1)) < np.median(np.linalg.norm(pos0 - truth, axis=1))
