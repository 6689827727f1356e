"""GPU: every pose-taking kernel with the camera turned around -- the world frames of tests/world_frame_cases.py, whose
current camera takes each branch and edge of the rotation-matrix-to-quaternion conversion (pose_from_rt12 -> qfrommatrix).

(a) the device's bare round trip pose_to_rt12(pose_from_rt12(T)) -- pose_optimize with no iteration, sparse_img_align
    with no iteration in every launch geometry -- against the 40-digit round trip and bit for bit against the oracle's;
(b) every converting kernel in every catalogue frame against the oracle, at the README's contract;
(c) invariance, without the oracle: each kernel's outputs in a frame G, mapped back, against the same case in the
    canonical frame; a discrete flip only where the oracle flips the same item between the two frames;
(d) batches whose streams each sit in a different frame, bit for bit against their single calls."""
import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import depth_update_hp as dhp
from tests import world_frame_cases as wf

pytestmark = pytest.mark.gpu

I12 = wf.rt12(np.eye(3))
T_OFF = (0.3, -1.2, 2.0)
FRAMES = [(c["name"], (0.0, 0.0, 0.0)) for c in wf.ALL] + [(n, wf.FAR_ORIGIN) for n in wf.PIN_FRAMES]
FRAME_IDS = [n + ("@far" if o != (0.0, 0.0, 0.0) else "") for n, o in FRAMES]
# (ctas_per_pair, features_per_thread, upfront mode): the configurations tests/test_sia_geometry_gpu.py forces
GEOMETRIES = {"auto": (-1, 0, -1), "cta-1fpt": (1, 1, -1), "cta-2fpt": (1, 2, -1), "cluster-2": (2, 0, -1),
              "cluster-4": (4, 0, -1), "cluster-4-per-level": (4, 0, 0), "cluster-8": (8, 0, -1)}
# Invariance tolerances (canonical frame): what rounding the inputs at ~1e-16 relative (~2e-14 m at the far origin) can
# move.  The oracle's own spread over the exactly rotated frames: pose < 1e-12, pixels < 1e-9, seeds bit for bit.  The
# kernels' on an H100: pose 1.3e-13, pixels and seeds bit for bit, and for the unconverted control (point_optimize_batch,
# two-view points with cond(A) up to ~1e6) 4.1e-8 m.  The float32-rounded frames are not compared: rounding R moves the
# camera by ~1e-8 rad, a different problem (the oracle's seeds then move by up to 5e-4 relative), so they take part in (b)
# only.
INV_POSE, INV_PX, INV_SEED_REL, INV_POINT = 1e-10, 1e-6, 1e-6, 4e-7


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _po_case():
    return synth.make_pose_opt_case(3, n=8, width=752, height=480)


def _po_roundtrip(run, c, T):
    return run(2.0, 0, c["cam"].fx, T, c["f"], c["pos"], c["level"], np.ones(8, np.uint8))["T"]


# ---- (a) the bare round trip --------------------------------------------------------------------------------------------
def test_pose_optimize_roundtrip_matches_hp_and_oracle_bits(ctx, oracle):
    """pose_optimize with n_iter = 0 and observations writes pose_to_rt12(pose_from_rt12(T)) back: within ROUNDTRIP_ULP
    of hp_roundtrip, made by the branch hp reports, translation untouched, and bit-identical to the oracle's round trip
    (same IEEE sequence: contraction off, correctly rounded sqrt and division) for every catalogue entry."""
    c = _po_case()
    unique = 0
    for e in wf.ALL:
        T = wf.rt12(e["R"], T_OFF)
        g = _po_roundtrip(ctx.pose_optimize, c, T)
        o = _po_roundtrip(oracle.pose_optimize, c, T)
        hp = wf.hp_roundtrip(T)
        assert wf.ulp_error(g, hp) <= wf.ROUNDTRIP_ULP, (e["name"], wf.ulp_error(g, hp))
        assert np.array_equal(_bits(g), _bits(o)), (e["name"], g - o)
        assert np.array_equal(_bits(g[:, 3]), _bits(T[:, 3])), e["name"]
        m = wf.branches_matching(g, T)
        assert hp["branch"] in m, (e["name"], hp["branch"], m)
        unique += m == [hp["branch"]]
    assert unique >= len(wf.ALL) - 3


def test_pose_optimize_roundtrip_nan_entry_gives_all_nan(ctx, oracle):
    """A NaN in any one of the nine rotation entries: an all-NaN rotation on the device, as in the oracle."""
    c = _po_case()
    for base in ("near_identity", "default_x", "yaw_150", "roll_150_tilted", "tie_xy_180", "perm_120"):
        for k in range(9):
            R = wf.BY_NAME[base]["R"].copy()
            R.reshape(-1)[k] = np.nan
            T = wf.rt12(R, T_OFF)
            g = _po_roundtrip(ctx.pose_optimize, c, T)
            o = _po_roundtrip(oracle.pose_optimize, c, T)
            assert np.all(np.isnan(g[:, :3])) and np.all(np.isnan(o[:, :3])), (base, k)
            assert np.array_equal(_bits(g[:, 3]), _bits(T[:, 3])), (base, k)


@pytest.fixture(scope="module")
def sia_pair(ctx, pair300):
    n = 90  # within every forced geometry's capacity (two CTAs x 96 features is the smallest)
    d = {k: pair300[k][:n] for k in ("px", "f", "pos", "has_point")}
    fr = (ctx.frame(pair300["ref_pyr"]), ctx.frame(pair300["cur_pyr"]))
    yield dict(d, cam=pair300["cam"], ref_pos=pair300["ref_pos"], frames=fr)
    for f in fr:
        f.destroy()


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_sparse_img_align_start_pose_roundtrip(ctx, oracle, sia_pair, geometry):
    """sparse_img_align with n_iter = 0 writes T_out from the converted start pose: the same bits as the oracle's bare
    round trip, in every launch geometry (the launch that ran is checked: a fallback would hide a geometry)."""
    cfg = GEOMETRIES[geometry]
    c = _po_case()
    d = sia_pair
    ctx.sia_config(cfg[0], cfg[1])
    ctx.sia_upfront(cfg[2])
    try:
        for e in wf.ALL:
            T = wf.rt12(e["R"], (0.01, -0.02, 0.03))
            g = ctx.sparse_img_align(d["frames"][0], d["frames"][1], d["cam"], T, d["px"], d["f"], d["pos"], d["has_point"],
                                     d["ref_pos"], 4, 0, 0)
            L = ctx.sia_last_launch()
            if cfg[0] > 0:
                assert L["ctas_per_pair"] == cfg[0], (geometry, L)
            if cfg[2] == 0:
                assert not L["upfront"], (geometry, L)
            o = _po_roundtrip(oracle.pose_optimize, c, T)
            assert np.array_equal(_bits(g["T"]), _bits(o)), (geometry, e["name"], g["T"] - o)
            assert wf.ulp_error(g["T"], wf.hp_roundtrip(T)) <= wf.ROUNDTRIP_ULP, (geometry, e["name"])
    finally:
        ctx.sia_config(-1, 0)
        ctx.sia_upfront(-1)


# ---- the kernels in every frame ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scenes(ctx):
    pose, match, depth, mp_ = wf.pose_case(), wf.match_case(), wf.depth_case(), wf.map_case()
    s = dict(pose=pose, match=match, depth=depth, map=mp_)
    s["match_frames"] = (ctx.frame(match["ref_pyr"]), ctx.frame(match["cur_pyr"]))
    s["depth_frames"] = (ctx.frame(depth["ref_pyr"]), ctx.frame(depth["cur_pyr"]))
    s["map_frames"] = ([ctx.frame(p) for p in mp_["kf_pyr"]], ctx.frame(mp_["cur_pyr"]))
    yield s
    for f in list(s["match_frames"]) + list(s["depth_frames"]) + s["map_frames"][0] + [s["map_frames"][1]]:
        f.destroy()


def _frames_for(kind, scenes):
    """(frame id, G, case) for every frame, plus the canonical case as ("canonical", identity, case)."""
    out = [("canonical", wf.rt12(np.eye(3)), scenes[kind])]
    for (name, origin), fid in zip(FRAMES, FRAME_IDS):
        c, G = wf.reframe(scenes[kind], kind, wf.BY_NAME[name]["R"], origin)
        out.append((fid, G, c))
    return out


def _pose_runs(ctx, oracle, c):
    a = (2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], c["has_point"])
    return ctx.pose_optimize(*a), oracle.pose_optimize(*a)


def _match_runs(ctx, oracle, c, frames):
    M = c["M"]
    g = ctx.find_match_direct([frames[0]], [c["T_ref_w"]], frames[1], c["T_cur_w"], c["cam"], np.zeros(M, np.int32), c["ref_px"],
                              c["ref_f"], c["ref_level"], c["ftr_type"], c["ref_grad"], c["point_pos"], c["px_cur"], 2, 10)
    # the oracle composes T_cur_ref from the two world poses through its own conversion, as the kernel does
    T_cur_ref = oracle.se3_mul(c["T_cur_w"], oracle.se3_inv(c["T_ref_w"]))
    ref_pos = oracle.se3_inv(c["T_ref_w"])[:, 3]
    o = dict(success=[], search_level=[], px_cur=[])
    for i in range(M):
        depth = float(np.linalg.norm(ref_pos - c["point_pos"][i]))
        r = oracle.find_match_direct(c["ref_pyr"], c["cur_pyr"], c["cam"], T_cur_ref, c["ref_px"][i], c["ref_f"][i],
                                     int(c["ref_level"][i]), int(c["ftr_type"][i]), c["ref_grad"][i], depth, 2, 10, c["px_cur"][i])
        for k in o:
            o[k].append(r[k])
    return g, {k: np.array(v) for k, v in o.items()}


def _depth_runs(ctx, oracle, c, frames):
    a = (c["ref_index"], c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"], c["batch_counter"],
         c["seeds"])
    g = ctx.depth_filter_update([frames[0]], [c["T_ref_w"]], frames[1], c["T_cur_w"], c["cam"], *a)
    o = oracle.depth_filter_update([c["ref_pyr"]], [c["T_ref_w"]], c["cur_pyr"], c["T_cur_w"], c["cam"], *a)
    return g, o


EPI_N = 100


def _epi_runs(ctx, oracle, c, frames):
    s = c["seeds"]
    mu, sig = s["mu"][:EPI_N].astype(np.float64), np.sqrt(s["sigma2"][:EPI_N].astype(np.float64))
    d_est, d_min, d_max = 1.0 / mu, 1.0 / (mu + sig), 1.0 / np.maximum(mu - sig, 1e-7)
    sel = lambda k: np.asarray(c[k])[:EPI_N]
    g = ctx.find_epipolar_match_direct([frames[0]], [c["T_ref_w"]], frames[1], c["T_cur_w"], c["cam"], np.zeros(EPI_N, np.int32),
                                       sel("ftr_px"), sel("ftr_f"), sel("ftr_level"), sel("ftr_type"), sel("ftr_grad"), d_est, d_min,
                                       d_max, 2)
    T_cur_ref = oracle.se3_mul(c["T_cur_w"], oracle.se3_inv(c["T_ref_w"]))
    o = dict(success=[], reject=[], n_zmssd=[], px_cur=[], depth=[])
    for i in range(EPI_N):
        r = oracle.find_epipolar_match_direct(c["ref_pyr"], c["cur_pyr"], c["cam"], T_cur_ref, c["ftr_px"][i], c["ftr_f"][i],
                                              int(c["ftr_level"][i]), int(c["ftr_type"][i]), c["ftr_grad"][i], d_est[i], d_min[i],
                                              d_max[i], 2)
        for k in o:
            o[k].append(r[k])
    return g, {k: np.array(v) for k, v in o.items()}


def _map_runs(ctx, oracle, c, frames):
    g = ctx.reproject_map(c["view"], frames[0], frames[1], c["cur_T_f_w"], c["cam"], c["options"], c["cell_order"], c["pt_type"],
                          c["pt_n_failed"], c["pt_n_succeeded"])
    return g, oracle.reproject_map(c)


RP_EXACT = ("overlap_kf", "overlap_count", "new_point", "new_level", "new_type", "pt_type", "pt_n_failed", "pt_n_succeeded")
RP_COUNTS = ("n_matches", "n_trials", "n_new", "n_overlap")


def _same_reprojection(a, b) -> bool:
    return all(a[k] == b[k] for k in RP_COUNTS) and all(np.array_equal(a[k], b[k]) for k in RP_EXACT)


def _flips(a, b):
    return np.flatnonzero(np.asarray(a) != np.asarray(b))


def _exact(fid) -> bool:
    """A frame whose rotation is an exact (double) catalogue entry: the invariance checks (c) apply."""
    return not fid.endswith("_f32")


def test_pose_optimize_in_every_frame(ctx, oracle, scenes):
    """(b) mask exact, pose within 1e-8 of the oracle in the canonical frame; (c) the same answer as the canonical run."""
    runs = [(fid, G, *_pose_runs(ctx, oracle, c)) for fid, G, c in _frames_for("pose", scenes)]
    _, _, g0, o0 = runs[0]
    worst, edges = 0.0, 0
    for fid, G, g, o in runs:
        assert np.array_equal(g["has_point"], o["has_point"]) and g["num_obs"] == o["num_obs"], fid
        dt, dr = synth.pose_error(wf.to_canonical(g["T"], G), wf.to_canonical(o["T"], G))
        assert dt < 1e-8 and dr < 1e-8, (fid, dt, dr)
        if not _exact(fid):
            continue
        flips = _flips(g["has_point"], g0["has_point"])
        assert set(flips) <= set(_flips(o["has_point"], o0["has_point"])), fid
        edges += len(flips)
        dt, dr = synth.pose_error(wf.to_canonical(g["T"], G), g0["T"])
        worst = max(worst, dt, dr)
        assert dt < INV_POSE and dr < INV_POSE, (fid, dt, dr)
    print(f"pose_optimize: {len(runs) - 1} frames, worst invariance {worst:.1e}, knife-edge mask flips {edges}")


def test_point_optimize_batch_in_every_frame_control(ctx):
    """(c) the control: point_optimize_batch uses the keyframe matrices as given, without a conversion, so it sees the
    same change of frame as the converting kernels and shows what a change of frame alone moves."""
    rng = np.random.default_rng(17)
    cam = synth.camera_for(752, 480)
    poses = [synth.se3_mul(synth.se3_exp(np.concatenate([rng.uniform(-0.3, 0.3, 3), rng.uniform(-0.05, 0.05, 3)])),
                           synth.base_pose()) for _ in range(5)]
    P = 100
    px = np.stack([rng.uniform(150, 600, P), rng.uniform(100, 380, P)], axis=1)
    truth = synth.intersect(synth.Plane.tilted(), poses[0], cam.cam2world(px))
    pos0 = truth + rng.normal(0, 0.02, (P, 3))
    offs, frs, fs = [0], [], []
    for p in range(P):
        for fr in rng.choice(5, int(rng.integers(2, 6)), replace=False):
            pc = poses[fr][:, :3] @ truth[p] + poses[fr][:, 3]
            frs.append(fr)
            fs.append(cam.cam2world(cam.world2cam(pc) + rng.normal(0, 0.3, 2)))
        offs.append(len(frs))
    frs, fs = np.array(frs, np.int32), np.array(fs)
    g0 = ctx.point_optimize_batch(5, pos0, offs, frs, fs, poses)
    worst = 0.0
    for (name, origin), fid in zip(FRAMES, FRAME_IDS):
        if not _exact(fid):
            continue
        G = wf.frame_for(poses[0], wf.BY_NAME[name]["R"], origin)
        Ginv = synth.se3_inv(G)
        g = ctx.point_optimize_batch(5, pos0 @ G[:, :3].T + G[:, 3], offs, frs, fs, [synth.se3_mul(T, Ginv) for T in poses])
        back = g @ Ginv[:, :3].T + Ginv[:, 3]
        d = float(np.max(np.abs(back - g0)))
        worst = max(worst, d)
        assert d < INV_POINT, (fid, d)
    print(f"point_optimize_batch: worst invariance {worst:.1e} m")


def test_find_match_direct_in_every_frame(ctx, oracle, scenes):
    """(b) success and search level exact, pixels within 1e-4 of the oracle; (c) against the canonical run."""
    runs = [(fid, *_match_runs(ctx, oracle, c, scenes["match_frames"])) for fid, _, c in _frames_for("match", scenes)]
    _, g0, o0 = runs[0]
    worst, edges = 0.0, 0
    for fid, g, o in runs:
        assert np.array_equal(g["success"], o["success"]) and np.array_equal(g["search_level"], o["search_level"]), fid
        ok = g["success"]
        assert np.max(np.abs(g["px_cur"][ok] - o["px_cur"][ok]), initial=0.0) <= 1e-4, fid
        if not _exact(fid):
            continue
        flips = _flips(g["success"], g0["success"])
        assert set(flips) <= set(_flips(o["success"], o0["success"])), fid
        edges += len(flips)
        both = g["success"] & g0["success"]
        d = float(np.max(np.abs(g["px_cur"][both] - g0["px_cur"][both]), initial=0.0))
        worst = max(worst, d)
        assert d <= INV_PX, (fid, d)
    assert g0["success"].sum() > scenes["match"]["M"] // 2
    print(f"find_match_direct: worst invariance {worst:.1e} px, knife-edge flips {edges}")


def test_depth_filter_in_every_frame(ctx, oracle, scenes):
    """(b) status and ZMSSD counts exact, every updated seed bit for bit one of the exactly rounded statement's candidates
    (tests/depth_update_hp.py); (c) against the canonical run."""
    runs = [(fid, c, *_depth_runs(ctx, oracle, c, scenes["depth_frames"])) for fid, _, c in _frames_for("depth", scenes)]
    _, _, g0, o0 = runs[0]
    worst, edges = 0.0, 0
    for fid, c, g, o in runs:
        assert np.array_equal(g["status"], o["status"]) and np.array_equal(g["n_zmssd"], o["n_zmssd"]), fid
        dhp.assert_seed_updates(g, o, c["seeds"], [c["T_ref_w"]], c["ref_index"], c["T_cur_w"], c["ftr_f"], c["cam"].fx,
                                oracle, oracle_statement=False)
        if not _exact(fid):
            continue
        flips = _flips(g["status"], g0["status"])
        assert set(flips) <= set(_flips(o["status"], o0["status"])), fid
        edges += len(flips)
        same = np.setdiff1d(np.arange(len(g["status"])), flips)
        for k in ("a", "b", "mu", "sigma2"):
            x, y = g[k][same].astype(np.float64), g0[k][same].astype(np.float64)
            d = float(np.max(np.abs(x - y) / np.maximum(np.abs(y), 1e-7), initial=0.0))
            worst = max(worst, d)
            assert d <= INV_SEED_REL, (fid, k, d)
    assert (o0["status"] >= 5).sum() > 50
    print(f"depth_filter_update: worst invariance {worst:.1e} rel, knife-edge status flips {edges}")


def test_epipolar_matcher_in_every_frame(ctx, oracle, scenes):
    """(b) success, reject and ZMSSD counts exact, pixels within 1e-4 and depths within 2e-5 relative of the oracle;
    (c) against the canonical run."""
    runs = [(fid, *_epi_runs(ctx, oracle, c, scenes["depth_frames"])) for fid, _, c in _frames_for("depth", scenes)]
    _, g0, o0 = runs[0]
    worst, edges = 0.0, 0
    for fid, g, o in runs:
        for k in ("success", "reject", "n_zmssd"):
            assert np.array_equal(g[k], o[k]), (fid, k)
        ok = g["success"]
        assert np.max(np.abs(g["px_cur"][ok] - o["px_cur"][ok]), initial=0.0) <= 1e-4, fid
        assert np.allclose(g["depth"][ok], o["depth"][ok], rtol=2e-5), fid
        if not _exact(fid):
            continue
        flips = np.union1d(_flips(g["success"], g0["success"]), _flips(g["n_zmssd"], g0["n_zmssd"]))
        oflips = np.union1d(_flips(o["success"], o0["success"]), _flips(o["n_zmssd"], o0["n_zmssd"]))
        assert set(flips) <= set(oflips), fid
        edges += len(flips)
        both = g["success"] & g0["success"]
        d = float(np.max(np.abs(g["px_cur"][both] - g0["px_cur"][both]), initial=0.0))
        worst = max(worst, d)
        assert d <= INV_PX, (fid, d)
    assert g0["success"].sum() > EPI_N // 4
    print(f"find_epipolar_match_direct: worst invariance {worst:.1e} px, knife-edge flips {edges}")


def test_reproject_map_in_every_frame(ctx, oracle, scenes):
    """(b) added features and point counters / types exact, pixels within 1e-4 of the oracle; (c) the same features and
    point state as the canonical run unless the oracle's own outcome changes between the two frames."""
    runs = [(fid, *_map_runs(ctx, oracle, c, scenes["map_frames"])) for fid, _, c in _frames_for("map", scenes)]
    _, g0, o0 = runs[0]
    worst, edges = 0.0, 0
    for fid, g, o in runs:
        assert _same_reprojection(g, o), fid
        assert np.max(np.abs(g["new_px"] - o["new_px"]), initial=0.0) <= 1e-4, fid
        if not _exact(fid):
            continue
        if not _same_reprojection(o, o0):  # the cell policy cascades: any knife edge changes the whole outcome
            edges += 1
            continue
        assert _same_reprojection(g, g0), fid
        d = float(np.max(np.abs(g["new_px"] - g0["new_px"]), initial=0.0))
        worst = max(worst, d)
        assert d <= INV_PX, (fid, d)
    assert g0["n_matches"] > 30
    print(f"reproject_map: worst invariance {worst:.1e} px, frames at a knife edge {edges}")


# ---- (d) mixed-frame batches ------------------------------------------------------------------------------------------
MIXED = ("default_x", "yaw_150", "roll_180", "tie_yz_180", "perm_120", "near_pi_y", "yaw_120_trace_plus_ulp_f32")


def test_pose_optimize_batch_mixed_frames_equals_single_calls(ctx, scenes):
    cases = [wf.reframe(scenes["pose"], "pose", wf.BY_NAME[n]["R"], wf.FAR_ORIGIN if k % 2 else (0, 0, 0))[0]
             for k, n in enumerate(MIXED)]
    off = np.concatenate([[0], np.cumsum([len(c["level"]) for c in cases])]).astype(np.int32)
    cat = lambda k: np.concatenate([c[k] for c in cases])
    res = ctx.pose_optimize_batch(2.0, 10, [c["cam"].fx for c in cases], np.stack([c["T_init"] for c in cases]), off,
                                  cat("f"), cat("pos"), cat("level"), cat("has_point"))
    for n, c, r in zip(MIXED, cases, res):
        g = ctx.pose_optimize(2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], c["has_point"])
        assert np.array_equal(_bits(r["T"]), _bits(g["T"])) and np.array_equal(r["has_point"], g["has_point"]), n
        for k in ("num_obs", "n_iter_done", "error_init", "error_final", "estimated_scale"):
            assert r[k] == g[k], (n, k)
        assert np.array_equal(_bits(r["cov"]), _bits(g["cov"])), n


def test_depth_filter_streams_mixed_frames_equals_single_calls(ctx, scenes):
    ref, cur = scenes["depth_frames"]
    cases = [wf.reframe(scenes["depth"], "depth", wf.BY_NAME[n]["R"], wf.FAR_ORIGIN if k % 2 else (0, 0, 0))[0]
             for k, n in enumerate(MIXED)]
    keys = ("ftr_px", "ftr_f", "ftr_level", "ftr_type", "ftr_grad", "batch_id", "seeds")
    streams = [dict({k: c[k] for k in keys}, cur=cur, cur_T_f_w=c["T_cur_w"], cam=c["cam"], batch_counter=c["batch_counter"],
                    ref_index=np.full(c["M"], s, np.int32)) for s, c in enumerate(cases)]
    batched = ctx.depth_filter_update_streams(streams, [ref] * len(cases), np.stack([c["T_ref_w"] for c in cases]))
    for n, c, b in zip(MIXED, cases, batched):
        g = ctx.depth_filter_update([ref], [c["T_ref_w"]], cur, c["T_cur_w"], c["cam"], c["ref_index"], c["ftr_px"], c["ftr_f"],
                                    c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"], c["batch_counter"], c["seeds"])
        for k in ("a", "b", "mu", "z_range", "sigma2", "status", "px_cur", "z", "n_zmssd"):
            assert np.ascontiguousarray(b[k]).tobytes() == np.ascontiguousarray(g[k]).tobytes(), (n, k)


def test_reproject_map_streams_mixed_frames_equals_single_calls(ctx, scenes):
    kfs, cur = scenes["map_frames"]
    cases = [wf.reframe(scenes["map"], "map", wf.BY_NAME[n]["R"], wf.FAR_ORIGIN if k % 2 else (0, 0, 0))[0]
             for k, n in enumerate(MIXED)]
    args = lambda c: dict(view=c["view"], kf_frames=kfs, cur=cur, cur_T_f_w=c["cur_T_f_w"], cam=c["cam"], options=c["options"],
                          cell_order=c["cell_order"], pt_type=c["pt_type"], pt_n_failed=c["pt_n_failed"],
                          pt_n_succeeded=c["pt_n_succeeded"])
    batched = ctx.reproject_map_streams([args(c) for c in cases])
    for n, c, b in zip(MIXED, cases, batched):
        g = ctx.reproject_map(**args(c))
        for k in RP_EXACT + ("pt_action", "new_px", "new_grad"):
            assert np.ascontiguousarray(b[k]).tobytes() == np.ascontiguousarray(g[k]).tobytes(), (n, k)
        for k in RP_COUNTS + ("n_projected", "n_speculative"):
            assert b[k] == g[k], (n, k)
