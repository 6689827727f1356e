"""Inputs and comparisons shared by the alignment-kernel tests (test_sia_geometry_gpu.py, test_sia_gpu.py,
test_oracle_pins.py): feature sets sized to the capacity edges of every launch
geometry, and frame pairs at pyramid sizes whose levels take every staging path of the kernel."""
import numpy as np

from rpg_svo_b200 import synth

POSE_TOL = 1e-4
RES_TOL = 1e-4
# Below about a dozen features the normal matrix is (nearly) rank deficient: the reference's result is then whatever
# Eigen's LDLT makes of rounding noise, so only the pose-independent outputs are compared.
RANK_OK = 12

# Pyramid sizes and what their levels exercise (level widths in parentheses):
#   644x484   (644, 322, 161, 80, 40): no windows at levels 0-1 (W % 8 != 0), an odd width at level 2, staged whole
#   648x488   (648, 324, 162, ...):    W % 16 == 8 at level 0, the window copied as two 8-byte cp.async per row
#   160x120   (160, 80, 40, 20, 10):   level 0 staged whole by TMA where the staging region holds 19 KB
#   1280x720  (1280, 640, 320, ...):   16-byte window copies at levels 0-2
ODD_SIZES = [(644, 484), (648, 488), (160, 120), (1280, 720)]

# Features whose has_point is cleared: the first and last slot of every CTA slice of every geometry (96 per cluster CTA,
# 320 / 384 / 512 per CTA), slots 159 / 160 (the two features of thread 0 / 159 in the 160-thread geometry) and 303 (the
# last slot of its 304-slot arrays).
EDGE_SLOTS = sorted({s for k in range(9) for s in (96 * k, 96 * k - 1) if s >= 0} |
                    {159, 160, 303, 304, 319, 320, 383, 384, 511, 512, 1023})


def base_pair():
    """640x480, 1100 features in a fixed shuffled order: feature sets of any size up to 1100 are its first N."""
    d = synth.make_frame_pair(4242, n_feat=1100, n_levels=5)
    perm = np.random.default_rng(4242).permutation(1100)
    for k in ("px", "f", "pos", "has_point"):
        d[k] = np.ascontiguousarray(d[k][perm])
    d["has_point"][:] = 1
    return d


def subset(d, n, clear_edges=True):
    """The first n features of `d`, has_point cleared at EDGE_SLOTS (unless the set is too small to solve)."""
    s = dict(d)
    for k in ("px", "f", "pos", "has_point"):
        s[k] = np.ascontiguousarray(d[k][:n]).copy()
    if clear_edges and n >= RANK_OK:
        s["has_point"][[e for e in EDGE_SLOTS if e < n]] = 0
    return s


def border_pair(seed, width, height, n_feat, trans=0.08, rot_deg=1.5, cam=None, n_levels=5):
    """Like test_sia_gpu._border_case at any size: jittered features plus a quarter of them 3-5 px from one of the four
    borders (and four in the bottom-right corner), and a motion large enough that patches leave the current image."""
    rng = np.random.default_rng(seed)
    cam = synth.camera_for(width, height) if cam is None else cam
    plane, tex = synth.Plane.tilted(), synth.make_texture(7)
    T_ref_w = synth.base_pose()
    xi = np.concatenate([rng.uniform(-trans, trans, 3), np.deg2rad(rng.uniform(-rot_deg, rot_deg, 3))])
    T_cur_w = synth.se3_mul(synth.se3_exp(xi), T_ref_w)
    ref_pyr = synth.build_pyramid(synth.render(cam, T_ref_w, plane, tex), n_levels)
    cur_pyr = synth.build_pyramid(synth.render(cam, T_cur_w, plane, tex), n_levels)
    px = synth.jittered_features(rng, cam, n_feat, margin=4.0)
    W, H = cam.width, cam.height
    nb = n_feat // 4
    side = rng.integers(0, 4, nb)
    along = rng.uniform(0.0, 1.0, nb)
    dist = rng.uniform(3.0, 5.0, nb)
    # x = dist from the left edge / W - dist from the right one: at level 0 the features 3-4 px from the right or bottom edge
    # sit on the last column / row whose 7x7 footprint fits (floor(x) + 3 == W - 1)
    bx = np.where(side == 0, dist, np.where(side == 1, W - dist, along * (W - 1)))
    by = np.where(side == 2, dist, np.where(side == 3, H - dist, along * (H - 1)))
    px[:nb] = np.stack([bx, by], axis=1)
    px[nb:nb + 4] = np.stack([W - rng.uniform(3.0, 5.0, 4), H - rng.uniform(3.0, 5.0, 4)], axis=1)  # bottom right
    f = cam.cam2world(px)
    pos = synth.intersect(plane, T_ref_w, f)
    hp = (rng.uniform(size=n_feat) > 0.05).astype(np.uint8)
    return dict(cam=cam, ref_pyr=ref_pyr, cur_pyr=cur_pyr, px=np.ascontiguousarray(px), f=np.ascontiguousarray(f),
                pos=np.ascontiguousarray(pos), has_point=hp, ref_pos=synth.se3_inv(T_ref_w)[:, 3].copy(),
                T_gt=synth.se3_exp(xi), T_ref_w=T_ref_w, n_levels=n_levels)


ODD_SEEDS = {(644, 484): 4,(648, 488): 1, (160, 120): 760, (1280, 720): 1880}


def odd_pair(size, n_feat=180):
    """The border case at one of ODD_SIZES (180 features: every geometry, the 2-CTA cluster included, can run it).  The
    seeds are chosen so that no Gauss-Newton decision of the case is a near-tie (decision_margin)."""
    return border_pair(ODD_SEEDS[size], size[0], size[1], n_feat)


def decision_margin(o):
    """How far the oracle's run `o` is from flipping a Gauss-Newton decision: the smallest relative chi2 change between an
    iteration and the last accepted one (accept / roll back), and the smallest |log(|x|_inf / eps)| of an accepted step
    (converged or not).  The reference sums chi2 serially in f32, the kernel per patch and then per warp; the two differ by
    ~1e-6 relative, so a case whose iteration trace is compared exactly needs a margin well above that."""
    m, prev = np.inf, None
    for t in o["trace"]:
        if t["iter"] > 0 and prev is not None:
            m = min(m, abs(t["chi2"] - prev) / prev)
        if t["accepted"]:
            prev = t["chi2"]
            m = min(m, abs(np.log(np.abs(t["x"]).max() / 1e-6)))
    return m


def oracle_run(oracle, d, max_level=4, min_level=0, T0=None, n_iter=30):
    T0 = synth.se3_identity() if T0 is None else T0
    return oracle.sparse_img_align(d["ref_pyr"], d["cur_pyr"], d["cam"], T0, d["px"], d["f"], d["pos"], d["has_point"],
                                   d["ref_pos"], max_level, min_level, n_iter)


def gpu_run(ctx, d, max_level=4, min_level=0, T0=None, n_iter=30, frames=None):
    T0 = synth.se3_identity() if T0 is None else T0
    ref, cur = frames if frames is not None else (ctx.frame(d["ref_pyr"]), ctx.frame(d["cur_pyr"]))
    g = ctx.sparse_img_align(ref, cur, d["cam"], T0, d["px"], d["f"], d["pos"], d["has_point"], d["ref_pos"], max_level,
                             min_level, n_iter, want_trace=True)
    if frames is None:
        ref.destroy(); cur.destroy()
    return g


def assert_parity(g, o, n_feat=None):
    """GPU result `g` vs oracle result `o`, with the tolerances of test_sia_gpu.py: mask and n_tracked bit-exact, the trace's
    (level, iter, accepted, n_meas) identical, chi2 within 1e-4 relative, final pose within 1e-4.  Rank-deficient
    problems (n_feat < RANK_OK): the mask and the first pass's n_meas only."""
    assert np.array_equal(g["visible"], o["visible"]), "visibility mask"
    if n_feat is not None and n_feat < RANK_OK:
        if o["trace"] and "trace" in g:  # (batch results carry no trace)
            assert g["trace"][0]["n_meas"] == o["trace"][0]["n_meas"]
        return
    assert g["n_tracked"] == o["n_tracked"], (g["n_tracked"], o["n_tracked"])
    if "trace" in g:
        assert len(g["trace"]) == len(o["trace"]), (len(g["trace"]), len(o["trace"]))
        for a, b in zip(g["trace"], o["trace"]):
            assert (a["level"], a["iter"], a["accepted"], a["n_meas"]) == (b["level"], b["iter"], b["accepted"], b["n_meas"])
            assert abs(a["chi2"] - b["chi2"]) <= 1e-4 * max(1.0, abs(b["chi2"])), (a["chi2"], b["chi2"])
    dt, dr = synth.pose_error(g["T"], o["T"])
    assert dt <= POSE_TOL and dr <= POSE_TOL, (dt, dr)


def assert_residual_parity(g, o):
    """svo_b200_sparse_residuals vs the oracle's residual pass: patch cache bit-exact, residuals within 1e-4, NaN where
    the patch was not evaluated."""
    assert np.array_equal(g["visible"], o["visible"]) and np.array_equal(g["in_image"], o["in_image"])
    v, m = o["visible"].astype(bool), o["in_image"].astype(bool)
    assert np.array_equal(g["ref_patch"][v], o["ref_patch"][v])
    if m.any():
        assert np.max(np.abs(g["residuals"][m] - o["residuals"][m])) <= RES_TOL
    assert np.all(np.isnan(g["residuals"][~m]))
    assert g["n_meas"] == o["n_meas"]
