"""CPU: the KLT oracle (oracle/svo_oracle_klt.cpp) against OpenCV's own buildOpticalFlowPyramid and calcOpticalFlowPyrLK
as the two-view initialisation calls them (recorded in tests/golden/ref/test_klt_pins.npz) on the cases of
tests/klt_cases.py."""
import numpy as np
import pytest

from oracle import binding_klt
from tests import klt_cases as kc
from tests.ref_golden import ref, sha256_u8  # noqa: F401 (ref: fixture)


def numpy_pyr_down(img):
    """pyrDown as one numpy statement: separable [1 4 6 4 1], reflect-101 borders, even rows and columns, (sum + 128) >> 8."""
    h, w = img.shape
    k = np.array([1, 4, 6, 4, 1])
    p = np.pad(img.astype(np.int64), 2, mode="reflect")
    t = sum(k[i] * p[:, i:i + w] for i in range(5))
    t = sum(k[i] * t[i:i + h, :] for i in range(5))
    return ((t[::2, ::2] + 128) >> 8).astype(np.uint8)


@pytest.mark.parametrize("size", kc.PYR_SIZES, ids=[f"{w}x{h}" for w, h in kc.PYR_SIZES])
def test_pyramid_and_derivatives_equal_opencv(size, ref):
    """Level count (buildOpticalFlowPyramid's return value + 1), every level and every level's Scharr derivatives bit for
    bit: the oracle's and the numpy rule's levels against OpenCV's."""
    w, h = size
    img = kc.pyr_image(w, h)
    r = kc.ref_pyramid(ref, img)
    o = binding_klt.pyramid(img, 4)
    assert len(o["images"]) == r["n_levels"] == len(binding_klt.level_sizes(w, h, 4))
    lv = img
    for l in range(r["n_levels"]):
        if l > 0:
            lv = numpy_pyr_down(lv)
        assert np.array_equal(sha256_u8(lv), r["images"][l]), l
        assert np.array_equal(sha256_u8(o["images"][l]), r["images"][l]), l
        assert np.array_equal(sha256_u8(o["derivs"][l]), r["derivs"][l]), l
    assert r["n_levels"] == {(640, 480): 4, (752, 480): 4, (644, 484): 5, (645, 485): 5, (60, 40): 1}[size]


@pytest.mark.parametrize("name", kc.NAMES)
def test_oracle_equals_opencv(name, ref):
    """Statuses identical, tracked points within TOL_PX, and no decision of the oracle within MARGINS of flipping."""
    k = kc.case(name)
    o = kc.oracle_run(k)
    r = kc.ref_run(ref, k)
    assert np.array_equal(o["status"], r["status"])
    m = r["status"] == 1
    d = float(np.abs(o["next_pts"][m] - r["next_pts"][m]).max()) if m.any() else 0.0
    print(f"{name}: {int(m.sum())}/{len(m)} tracked, max |oracle - OpenCV| = {d:.3g} px")
    assert d <= kc.TOL_PX
    assert kc.margins_ok(k, o).all(), np.where(~kc.margins_ok(k, o))[0]


def test_cases_reach_every_branch():
    """Each branch the cases are built for occurs on the oracle (see tests/klt_cases.py)."""
    R = {n: kc.oracle_run(kc.case(n)) for n in kc.NAMES}
    s640 = R["shift_640"]
    assert {binding_klt.CONVERGED, binding_klt.HALF_STEP, binding_klt.OUT_OF_BOUNDS} <= set(s640["reason"].tolist())
    assert s640["n_levels"] == 4 and R["shift_644"]["n_levels"] == 5
    assert np.all(R["iter_1"]["level_reason"][:, :4] == binding_klt.MAX_ITER) and np.all(R["iter_1"]["iters"][:, :4] == 1)
    t = R["iter_30_tight"]
    assert np.all((t["reason"] == binding_klt.HALF_STEP) | (t["reason"] == binding_klt.MAX_ITER) | (t["reason"] == binding_klt.OUT_OF_BOUNDS))
    assert np.sum((R["far_flow"]["reason"] == binding_klt.MAX_ITER) & (R["far_flow"]["iters"][:, 0] == 30)) > 50  # the limit at 30
    f = R["far_flow"]
    assert np.any(f["level_reason"][:, 1:4] == binding_klt.OUT_OF_BOUNDS)
    assert np.any((f["level_reason"][:, 3] == binding_klt.OUT_OF_BOUNDS) & (f["level_reason"][:, 0] >= 0))  # finer levels go on
    fl = R["flat"]
    assert np.all(fl["reason"][:120] == binding_klt.SMALL_EIG) and np.all(fl["status"][:120] == 0)
    b = R["border"]
    assert np.all(b["reason"][[*range(16), *range(20, 36)]] != binding_klt.OUT_OF_BOUNDS)
    assert np.all(b["reason"][[16, 17, 18, 19, 36, 37, 38, 39]] == binding_klt.OUT_OF_BOUNDS)
