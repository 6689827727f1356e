"""Cases of the robust alignment cost (svo_b200_sia_robust: MAD scale with unit, Tukey or Huber weights), shared by
test_sia_robust_pins.py (oracle vs the compiled reference) and test_sia_robust_gpu.py (kernel vs oracle).

Each case is a frame pair plus the run's parameters.  What they exercise:
  tukey / huber / unit          the three weight functions on one 200-feature pair, levels 4..0
  atan_tukey / radtan_huber     the distorted camera models
  occluded_tukey / _unit        a block of foreign texture pasted over about a quarter of the features in the current image
  iters_0 / iters_1             n_iter 0 (every level ends at iteration 0 and recomputes the scale; run() returns what the
                                pre-passes counted) and 1 (the coarsest level's scale carries through every finer level)
  zero_median_tukey / _huber    more than half the patches on a constant region: the MAD scale is exactly 0, every Tukey
                                weight is 0 (x = 0, the level ends at iteration 0 and the next recomputes the scale), Huber
                                weights of zero residuals are NaN (stop_ latches)
  feat_0 / feat_1 / feat_5      tiny feature sets, and no_points (no feature has a 3D point)
Observed on the oracle: on occluded_tukey Tukey ends about 1.8e-3 m from the ground-truth pose where plain Gauss-Newton
(occluded_unit, and the unweighted run) ends 1.3 m away; iters_0 returns 925 patches, the sum of the five pre-passes'
counts, where the unweighted run returns 0."""
import numpy as np

from oracle import binding_robust
from rpg_svo_b200 import synth

WEIGHTS = {"unit": 0, "tukey": 2, "huber": 3}  # SVO_B200_WEIGHT_*
RANK_OK = 12  # below this many features H is (nearly) rank deficient: only pose-independent outputs are compared


def _subset(p, n):
    """Features 1 .. n of `p` (feature 0 has no 3D point)."""
    q = dict(p)
    for k in ("px", "f", "pos", "has_point"):
        q[k] = np.ascontiguousarray(p[k][1:1 + n]).copy()
    return q


def occlude(p, frac=0.25, seed=99):
    """A block of another texture pasted into level 0 of the current image over the `frac` of the features with the
    smallest x + y (their footprints, as the ground-truth pose moves them), pyramid rebuilt."""
    cur = p["cur_pyr"][0].copy()
    H, W = cur.shape
    key = p["px"][:, 0] + p["px"][:, 1]
    n = int(round(frac * len(key)))
    edge = np.sort(key)[n]
    yy, xx = np.mgrid[0:H, 0:W]
    tex = synth.make_texture(seed)
    block = tex[:H, :W] if tex.shape[0] >= H and tex.shape[1] >= W else np.resize(tex, (H, W))
    mask = (xx + yy) < edge + 6
    cur[mask] = block[mask]
    q = dict(p)
    q["cur_pyr"] = synth.build_pyramid(cur, p["n_levels"])
    return q


def constant_region(p, frac=0.7, value=128):
    """Columns [0, frac W) of both level-0 images set to one grey value, pyramids rebuilt."""
    q = dict(p)
    for k in ("ref_pyr", "cur_pyr"):
        img = p[k][0].copy()
        img[:, : int(frac * img.shape[1])] = value
        q[k] = synth.build_pyramid(img, p["n_levels"])
    return q


def cases():
    base = synth.make_frame_pair(11, n_feat=200)
    base["has_point"][::17] = 0
    c = []

    def add(name, p, weight, n_iter=30, max_level=4, min_level=0):
        c.append(dict(name=name, p=p, weight=WEIGHTS[weight], n_iter=n_iter, max_level=max_level, min_level=min_level))

    for w in ("tukey", "huber", "unit"):
        add(w, base, w)
    add("atan_tukey", synth.make_frame_pair(61, n_feat=200, cam=synth.reference_param_camera("atan")), "tukey")
    add("radtan_huber", synth.make_frame_pair(61, n_feat=200, cam=synth.reference_param_camera("pinhole_radtan")), "huber")
    occ = occlude(synth.make_frame_pair(23, n_feat=240, trans=0.04, rot_deg=0.8))
    add("occluded_tukey", occ, "tukey")
    add("occluded_unit", occ, "unit")
    add("iters_0", base, "tukey", n_iter=0)
    add("iters_1", base, "tukey", n_iter=1)
    const = constant_region(synth.make_frame_pair(31, n_feat=200))
    add("zero_median_tukey", const, "tukey")
    add("zero_median_huber", const, "huber")
    for n in (0, 1, 5):
        add(f"feat_{n}", _subset(base, n), "tukey")
    nop = dict(base)
    nop["has_point"] = np.zeros_like(base["has_point"])
    add("no_points", nop, "tukey")
    return c


# No patch is ever in the image: the reference would take the median of no errors (undefined behaviour in vk::getMedian),
# so it is not called; the oracle and the kernel keep scale_ (0 here) -- not pinned.
NO_REF = {"no_points"}
# n_iter 0 or no features: the loop never writes H_, whose content the reference leaves undefined
NO_H = {"iters_0", "feat_0"}


def case(name):
    return next(k for k in cases() if k["name"] == name)


def oracle_run(k, T0=None):
    """The robust-cost oracle (oracle/binding_robust.py) on case k."""
    p = k["p"]
    T0 = synth.se3_identity() if T0 is None else T0
    return binding_robust.sparse_img_align_robust(p["ref_pyr"], p["cur_pyr"], p["cam"], T0, p["px"], p["f"], p["pos"], p["has_point"],
                                          p["ref_pos"], k["max_level"], k["min_level"], k["weight"], k["n_iter"])


def ref_run(ref, k):
    """The compiled reference on case k through the `ref` fixture (tests/ref_golden.py): its recorded outputs, or -- when
    recording -- oracle/_ref/libsvo_ref_robust.so through oracle/binding_robust.py."""
    p = k["p"]
    if ref.record_dir:
        ref.oracle = binding_robust
    return ref.call("sparse_img_align_robust", p["ref_pyr"][0], p["cur_pyr"][0], p["n_levels"], p["cam"], p["T_ref_w"], p["T_ref_w"],
                    p["px"], p["f"], p["pos"], p["has_point"], k["max_level"], k["min_level"], k["weight"], k["n_iter"])


def same_bits(a, b):
    """Equal as f32 bit patterns, any NaN equal to any NaN."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)].view(np.uint32), b[~np.isnan(b)].view(np.uint32))
