"""GPU parity: svo_b200_sparse_img_align / svo_b200_sparse_residuals vs the CPU oracle.

Tolerances are the ones BASELINE.json's north_star states: 1e-4 on the final SE3 and on per-patch
residuals, bit-exact visibility masks.
"""
import functools

import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import sia_cases as sc

pytestmark = pytest.mark.gpu

POSE_TOL = 1e-4
RES_TOL = 1e-4

# Launch geometries of the alignment kernel (svo_b200_sia_config): every parity test of this file runs on each.
#   auto        the library's choice (a 4-CTA cluster per pair for these small batches)
#   cta-1fpt    one CTA per pair, one feature per thread (320 / 384 / 512 threads)
#   cta-2fpt    one CTA per pair, two features per thread (160 threads for <= 320 features: the full-batch kernel)
#   cluster-4/8 the pair's features split over a thread-block cluster, partial sums exchanged through DSMEM
# third entry: svo_b200_sia_upfront mode (-1 = all levels prepared before the first iteration where the geometry allows it,
# 0 = every level prepared when it is reached)
GEOMETRIES = {"auto": (-1, 0, -1), "cta-1fpt": (1, 1, -1), "cta-2fpt": (1, 2, -1), "cluster-4": (4, 0, -1),
              "cluster-4-per-level": (4, 0, 0), "cluster-8": (8, 0, -1)}


@pytest.fixture(params=list(GEOMETRIES), autouse=True)
def geometry(request, ctx):
    g = GEOMETRIES[request.param]
    ctx.sia_config(g[0], g[1])
    ctx.sia_upfront(g[2])
    yield request.param
    ctx.sia_config(-1, 0)
    ctx.sia_upfront(-1)


def _run_both(ctx, oracle, d, max_level, min_level, n_iter=30, T0=None, trace=True):
    T0 = synth.se3_identity() if T0 is None else T0
    ref = ctx.frame(d["ref_pyr"])
    cur = ctx.frame(d["cur_pyr"])
    g = ctx.sparse_img_align(ref, cur, d["cam"], T0, d["px"], d["f"], d["pos"], d["has_point"],
                             d["ref_pos"], max_level, min_level, n_iter, want_trace=trace)
    o = oracle.sparse_img_align(d["ref_pyr"], d["cur_pyr"], d["cam"], T0, d["px"], d["f"], d["pos"],
                                d["has_point"], d["ref_pos"], max_level, min_level, n_iter)
    ref.destroy()
    cur.destroy()
    return g, o


@pytest.mark.parametrize("levels", [(4, 0), (4, 2), (2, 0), (0, 0)])
def test_final_pose_and_mask_c1(ctx, oracle, pair300, levels):
    g, o = _run_both(ctx, oracle, pair300, *levels)
    dt, dr = synth.pose_error(g["T"], o["T"])
    assert dt <= POSE_TOL and dr <= POSE_TOL, (dt, dr)
    assert np.array_equal(g["visible"], o["visible"])  # bit-exact mask
    assert g["n_tracked"] == o["n_tracked"]
    # both must actually have tracked the motion
    assert synth.pose_error(g["T"], pair300["T_cur_ref_gt"])[0] < 1e-3


def test_iteration_trace_matches(ctx, oracle, pair300):
    g, o = _run_both(ctx, oracle, pair300, 4, 0)
    assert len(g["trace"]) == len(o["trace"])
    for a, b in zip(g["trace"], o["trace"]):
        assert (a["level"], a["iter"], a["accepted"], a["n_meas"]) == (b["level"], b["iter"], b["accepted"], b["n_meas"])
        assert abs(a["chi2"] - b["chi2"]) <= 1e-4 * max(1.0, abs(b["chi2"]))
        assert np.allclose(a["x"], b["x"], rtol=1e-4, atol=1e-7)
        assert np.allclose(a["T"], b["T"], atol=1e-6)


@functools.lru_cache(maxsize=None)
def _residual_case(case):
    """(frame pair, pose) of a residual-pass case: the border case (features 3-5 px from every border, patches leaving the
    image at the motion) and the ATAN camera (general-camera projection) at their true motion."""
    if case == "border":
        d = sc.border_pair(5, 640, 480, 300)
        return d, d["T_gt"]
    cam = synth.reference_param_camera("atan")
    d = synth.make_frame_pair(1000, width=cam.width, height=cam.height, n_feat=300, n_levels=5, cam=cam)
    return d, d["T_cur_ref_gt"]


RESIDUAL_CASES = [("pair300", lv) for lv in range(5)] + [("border", 2), ("atan", 1)]


@pytest.mark.parametrize("case,level", RESIDUAL_CASES,
                         ids=[str(lv) if case == "pair300" else f"{case}-{lv}" for case, lv in RESIDUAL_CASES])
def test_residual_pass_matches(ctx, oracle, pair300, case, level):
    if case == "pair300":
        d, T = pair300, synth.se3_exp(np.array([0.004, -0.003, 0.002, 0.001, -0.002, 0.0015]))
    else:
        d, T = _residual_case(case)
    ref = ctx.frame(d["ref_pyr"])
    cur = ctx.frame(d["cur_pyr"])
    g = ctx.sparse_residuals(ref, cur, d["cam"], level, T, d["px"], d["f"], d["pos"], d["has_point"], d["ref_pos"])
    ref.destroy()
    cur.destroy()
    o = oracle.sparse_residuals(d["ref_pyr"][level], d["cur_pyr"][level], level, d["cam"], T, d["px"],
                                d["f"], d["pos"], d["has_point"], d["ref_pos"])
    assert np.array_equal(g["visible"], o["visible"])
    assert np.array_equal(g["in_image"], o["in_image"])
    # The patch rows of features that are not visible hold whatever the kernel's shared memory held: they depend on the
    # launch geometry's shared-memory layout (the reference leaves those rows of its cv::Mat cache uninitialised too).  So
    # the patch cache is compared on the visible rows.
    v = o["visible"].astype(bool)
    assert np.array_equal(g["ref_patch"][v], o["ref_patch"][v])  # f32 stage: bit-exact by construction
    m = o["in_image"].astype(bool)
    assert np.max(np.abs(g["residuals"][m] - o["residuals"][m])) <= RES_TOL
    assert np.all(np.isnan(g["residuals"][~m]))
    assert g["n_meas"] == o["n_meas"]
    assert abs(g["chi2"] - o["chi2"]) <= 1e-5 * abs(o["chi2"])
    assert np.allclose(g["H"], o["H"], rtol=1e-9, atol=1e-6)
    assert np.allclose(g["Jres"], o["Jres"], rtol=1e-5, atol=1e-3)


def test_no_features_returns_zero(ctx, pair300):
    d = pair300
    ref = ctx.frame(d["ref_pyr"])
    cur = ctx.frame(d["cur_pyr"])
    e = np.zeros((0, 3))
    g = ctx.sparse_img_align(ref, cur, d["cam"], synth.se3_identity(), np.zeros((0, 2)), e, e,
                             np.zeros(0, np.uint8), d["ref_pos"], 4, 0)
    assert g["n_tracked"] == 0 and np.allclose(g["T"], synth.se3_identity())


def _border_case(seed, n_feat, width=640, height=480, trans=0.08, rot_deg=1.5, margin=4.0):
    """Features right up to the image border + a large motion: patches leave the current image during the
    iterations (the 'slow path' that re-forms H from the contributing patches) and some never become visible."""
    rng = np.random.default_rng(seed)
    cam = synth.camera_for(width, height)
    plane, tex = synth.Plane.tilted(), synth.make_texture(7)
    T_ref_w = synth.base_pose()
    xi = np.concatenate([rng.uniform(-trans, trans, 3), np.deg2rad(rng.uniform(-rot_deg, rot_deg, 3))])
    T_cur_w = synth.se3_mul(synth.se3_exp(xi), T_ref_w)
    ref_pyr = synth.build_pyramid(synth.render(cam, T_ref_w, plane, tex), 5)
    cur_pyr = synth.build_pyramid(synth.render(cam, T_cur_w, plane, tex), 5)
    px = synth.jittered_features(rng, cam, n_feat, margin=margin)
    f = cam.cam2world(px)
    pos = synth.intersect(plane, T_ref_w, f)
    hp = (rng.uniform(size=n_feat) > 0.05).astype(np.uint8)
    return dict(cam=cam, ref_pyr=ref_pyr, cur_pyr=cur_pyr, px=px, f=f, pos=pos, has_point=hp,
                ref_pos=synth.se3_inv(T_ref_w)[:, 3].copy(), T_gt=synth.se3_exp(xi))


@pytest.mark.parametrize("case", ["300", "37", "edges-300"])
def test_patches_leaving_the_image_slow_path(ctx, oracle, case):
    # edges-300: a quarter of the features 3-5 px from one of the four borders, four in the bottom-right corner
    d = _residual_case("border")[0] if case == "edges-300" else _border_case(5, int(case))
    g, o = _run_both(ctx, oracle, d, 4, 0)
    # the case really exercises the per-iteration in-image test: some pass saw fewer patches than are visible
    vis_per_level = {l: 0 for l in range(5)}
    assert any(t["n_meas"] < 16 * int(o["visible"].sum()) for t in o["trace"])
    assert len(g["trace"]) == len(o["trace"])
    for a, b in zip(g["trace"], o["trace"]):
        assert (a["level"], a["iter"], a["accepted"], a["n_meas"]) == (b["level"], b["iter"], b["accepted"], b["n_meas"])
        # the kernel sums dx*r, dy*r over the 16 pixels of a patch in f32 (then f64 across patches); near
        # convergence Jres is a small difference of large terms, so x agrees to ~1e-6 absolute, not relative
        assert np.allclose(a["x"], b["x"], rtol=1e-4, atol=2e-6)
    dt, dr = synth.pose_error(g["T"], o["T"])
    assert dt <= POSE_TOL and dr <= POSE_TOL
    assert np.array_equal(g["visible"], o["visible"]) and g["n_tracked"] == o["n_tracked"]
    assert np.allclose(g["H"], o["H"], rtol=1e-8, atol=1e-6)


@pytest.mark.parametrize("n_feat,size", [(17, (752, 480)), (33, (640, 480)), (600, (752, 480)), (1000, (1920, 1080))])
def test_feature_counts_and_geometries(ctx, oracle, n_feat, size):
    """N not a multiple of 16 / 32, the two-features-per-thread kernels (N > 512), other image sizes."""
    d = synth.make_frame_pair(77 + n_feat, width=size[0], height=size[1], n_feat=n_feat, n_levels=5)
    g, o = _run_both(ctx, oracle, d, 4, 1, trace=False)
    dt, dr = synth.pose_error(g["T"], o["T"])
    assert dt <= POSE_TOL and dr <= POSE_TOL, (dt, dr)
    assert np.array_equal(g["visible"], o["visible"]) and g["n_tracked"] == o["n_tracked"]


def test_rank_deficient_single_feature_does_not_crash(ctx, oracle):
    """One feature gives a rank-2 normal matrix: the reference's result is then whatever Eigen's LDLT makes of
    rounding noise, so only the pose-independent outputs are compared (mask, patch count) and the call must return."""
    d = synth.make_frame_pair(78, n_feat=1, n_levels=5)
    d["has_point"][:] = 1
    g, o = _run_both(ctx, oracle, d, 4, 1, trace=False)
    assert np.array_equal(g["visible"], o["visible"])
    assert g["T"].shape == (3, 4)


def test_batch_of_pairs_matches_individual_runs(ctx, oracle):
    ds = [synth.make_frame_pair(2000 + k, n_feat=n, n_levels=5) for k, n in enumerate([300, 120, 299, 5])]
    refs = [ctx.frame(d["ref_pyr"]) for d in ds]
    curs = [ctx.frame(d["cur_pyr"]) for d in ds]
    off = np.concatenate([[0], np.cumsum([len(d["px"]) for d in ds])]).astype(np.int32)
    ctx.sia_batch_stage(refs, curs, ds[0]["cam"], np.tile(synth.se3_identity(), (4, 1, 1)), off,
                        np.concatenate([d["px"] for d in ds]), np.concatenate([d["f"] for d in ds]),
                        np.concatenate([d["pos"] for d in ds]), np.concatenate([d["has_point"] for d in ds]),
                        np.stack([d["ref_pos"] for d in ds]), 4, 0)
    ctx.sia_batch_run()
    r = ctx.sia_batch_fetch(want_H=True)
    for k, d in enumerate(ds):
        o = oracle.sparse_img_align(d["ref_pyr"], d["cur_pyr"], d["cam"], synth.se3_identity(), d["px"], d["f"], d["pos"],
                                    d["has_point"], d["ref_pos"], 4, 0, want_trace=False)
        dt, dr = synth.pose_error(r["T"][k], o["T"])
        assert dt <= POSE_TOL and dr <= POSE_TOL
        assert np.array_equal(r["visible"][off[k]:off[k + 1]], o["visible"])
        assert r["stats"]["n_tracked"][k] == o["n_tracked"]
    for f in refs + curs:
        f.destroy()


def test_argument_errors_are_reported_not_crashes(ctx, pair300):
    from rpg_svo_b200 import capi

    d = pair300
    ref, cur = ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"])
    with pytest.raises(capi.SvoB200Error):  # level outside the pyramid
        ctx.sparse_img_align(ref, cur, d["cam"], synth.se3_identity(), d["px"], d["f"], d["pos"], d["has_point"],
                             d["ref_pos"], 7, 0)
    n = 2100  # more features than the kernels support
    with pytest.raises(capi.SvoB200Error):
        ctx.sparse_img_align(ref, cur, d["cam"], synth.se3_identity(), np.zeros((n, 2)), np.zeros((n, 3)), np.zeros((n, 3)),
                             np.zeros(n, np.uint8), d["ref_pos"], 4, 0)
    ref.destroy(); cur.destroy()
