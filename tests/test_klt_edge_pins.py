"""CPU: the KLT oracle (oracle/svo_oracle_klt.cpp) against OpenCV's own buildOpticalFlowPyramid and calcOpticalFlowPyrLK
(recorded in tests/golden/ref/test_klt_edge_pins.npz) on the edge cases of tests/klt_edge_cases.py: non-finite points,
images below the window, level capacity, option clamps."""
import numpy as np
import pytest

from oracle import binding_klt
from tests import klt_cases as kc
from tests import klt_edge_cases as ke
from tests.ref_golden import ref, sha256_u8  # noqa: F401 (ref: fixture)
from tests.test_klt_pins import numpy_pyr_down

# level count of each pinned pyramid (OpenCV's, recorded)
N_LEVELS = {(1, 1, 4): 1, (2, 3, 4): 1, (17, 29, 4): 1, (30, 30, 4): 1, (31, 31, 4): 1, (61, 62, 4): 2, (62, 62, 4): 2,
            (63, 63, 4): 2, (645, 485, 4): 5, (3968, 3968, 7): 8, (3968, 3968, 10): 8, (7936, 7936, 7): 8}


@pytest.mark.parametrize("spec", ke.EDGE_PYRAMIDS, ids=[f"{w}x{h}_max{m}" for w, h, m in ke.EDGE_PYRAMIDS])
def test_edge_pyramid_equals_opencv(spec, ref):
    """Level count, every level and its Scharr derivatives bit for bit: the oracle's and the numpy rule's levels against
    OpenCV's, on images below the window, with a 31- or 32-pixel coarsest level, and at the 8-level capacity."""
    w, h, max_level = spec
    img = ke.pyramid_image(w, h)
    r = ke.ref_pyramid(ref, img, max_level)
    o = binding_klt.pyramid(img, max_level)
    assert len(o["images"]) == r["n_levels"] == N_LEVELS[spec] == len(binding_klt.level_sizes(w, h, max_level))
    lv = img
    for l in range(r["n_levels"]):
        if l > 0:
            lv = numpy_pyr_down(lv)
        assert np.array_equal(sha256_u8(lv), r["images"][l]), l
        assert np.array_equal(sha256_u8(o["images"][l]), r["images"][l]), l
        assert np.array_equal(sha256_u8(o["derivs"][l]), r["derivs"][l]), l
    if spec[:2] == (3968, 3968):
        assert o["images"][-1].shape == (31, 31)


def test_level_cut_past_capacity_is_refused():
    """OpenCV builds 9 levels at 7936 x 7936 from max_level 8 on; the oracle refuses those cuts (as the device does) and
    keeps 8 levels where the cut stops at 8 by itself."""
    assert len(binding_klt.level_sizes(7936, 7936, 7)) == 8
    for m in (8, 9, 100):
        with pytest.raises(ValueError):
            binding_klt.level_sizes(7936, 7936, m)
    assert len(binding_klt.level_sizes(3968, 3968, 100)) == 8 and len(binding_klt.level_sizes(7680, 7680, 100)) == 8
    with pytest.raises(ValueError):  # the smallest side whose ninth level (31) is wider than the window
        binding_klt.level_sizes(7681, 7681, 8)
    img = np.zeros((1, 1), np.uint8)
    with pytest.raises(ValueError):  # the tracker checks the size before it reads the images
        binding_klt.track(np.broadcast_to(img, (7936, 7936)), np.broadcast_to(img, (7936, 7936)), np.zeros((1, 2)), np.zeros((1, 2)), 8)


@pytest.mark.parametrize("name", ke.NAMES)
def test_oracle_equals_opencv(name, ref):
    """Statuses identical; tracked points within TOL_PX; where OpenCV returns a non-finite coordinate the oracle returns
    the same; no decision of the oracle within MARGINS of flipping."""
    k = ke.case(name)
    o = kc.oracle_run(k)
    r = kc.ref_run(ref, k)
    assert np.array_equal(o["status"], r["status"])
    m = r["status"] == 1
    d = float(np.abs(o["next_pts"][m] - r["next_pts"][m]).max()) if m.any() else 0.0
    print(f"{name}: {int(m.sum())}/{len(m)} tracked, max |oracle - OpenCV| = {d:.3g} px")
    assert d <= kc.TOL_PX
    assert ke.same_nonfinite(o["next_pts"], r["next_pts"])
    assert kc.margins_ok(k, o).all(), np.where(~kc.margins_ok(k, o))[0]


def test_cases_reach_their_branches():
    """Each case reaches the branch it was built for (see tests/klt_edge_cases.py)."""
    R = {n: kc.oracle_run(ke.case(n)) for n in ke.NAMES}
    k = ke.case("nonfinite")
    nf, sp, od = R["nonfinite"], k["special"], k["ordinary"]
    assert np.all(nf["status"][sp] == 0) and np.all(nf["level_reason"][sp, :4] == binding_klt.OUT_OF_BOUNDS)
    assert np.all(nf["iters"][sp] == 0) and np.all(nf["status"][od] == 1)
    assert ke.bits_equal(nf["next_pts"][sp], k["next_pts"][sp])  # the guess, scaled down and back up by powers of 2
    assert np.isnan(nf["next_pts"][sp]).sum() == 2 and np.isinf(nf["next_pts"][sp]).sum() == 4
    alone = binding_klt.track(k["prev"], k["cur"], k["prev_pts"][od], k["next_pts"][od])
    assert ke.bits_equal(alone["next_pts"], nf["next_pts"][od]) and np.array_equal(alone["iters"], nf["iters"][od])
    for w, h in ke.TINY:
        t = R[f"tiny_{w}x{h}"]
        assert t["n_levels"] == {(61, 62): 2, (62, 62): 2, (63, 63): 2, (645, 485): 5}.get((w, h), 1)
        if (w, h) in ((1, 1), (2, 3)):
            assert np.all(t["reason"] == binding_klt.SMALL_EIG) and np.all(t["status"] == 0)
        else:
            assert t["status"].sum() > len(t["status"]) // 2
    assert np.any(R["tiny_30x30"]["reason"] == binding_klt.OUT_OF_BOUNDS)  # walked out of a level smaller than the window
    bk = ke.case("binary")
    assert set(np.unique(bk["prev"]).tolist()) == {0, 255}
    assert np.abs(binding_klt.pyramid(bk["prev"], 0)["derivs"][0]).max() == 4080
    assert R["binary"]["status"].sum() > 150
    for n in ("iter_0", "iter_neg3"):
        assert np.all(R[n]["iters"] == 0) and np.all(R[n]["level_reason"][:, :4] == binding_klt.MAX_ITER)
        assert ke.bits_equal(R[n]["next_pts"], ke.case(n)["next_pts"])
    assert np.all(R["iter_1x"]["iters"][:, :4] == 1)
    it = R["iter_150"]["iters"]
    assert it.max() == 100 and np.sum(it == 100) > 90  # clamped: 150 runs as 100
    for key in ("next_pts", "status", "level_reason", "iters"):
        assert np.array_equal(R["eps_10"][key], R["eps_1e6"][key])
    assert [R[f"level_{m}"]["n_levels"] for m in (0, 1, 2, 3, 7)] == [1, 2, 3, 4, 4]
    for key in ("next_pts", "status", "level_reason", "iters"):
        assert np.array_equal(R["level_7"][key], R["level_3"][key])
        assert np.array_equal(R["mixed_levels"][key], R["level_2"][key])
    assert R["capacity"]["n_levels"] == 8 and np.all(R["capacity"]["level_reason"][:, 7] >= 0) and R["capacity"]["status"].all()
