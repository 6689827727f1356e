"""GPU: depth_filter_kernel's general instantiation (svo_b200_set_epipolar_options) over the grid of
tests/epipolar_options_cases.py -- the match-only launch and the depth filter against the options oracle and the compiled
reference's recorded outputs, the defaults set explicitly against never set, the multi-stream launch against single
calls, refused settings and the C++ host mirror (host_epipolar_options_demo)."""
import math
import subprocess

import numpy as np
import pytest

from oracle import binding_epipolar
from rpg_svo_b200 import capi
from tests import epipolar_options_cases as ec
from tests.ref_golden import RefCalls
from tests.test_depth_edges_gpu import _check_update
from tests.test_host_cpp_gpu import build_demo

pytestmark = pytest.mark.gpu

CAMS = list(ec.CAMERAS)


@pytest.fixture
def ectx(ctx):
    """The session context with the reference's defaults restored after the test, whatever it set."""
    ctx.set_epipolar_options()
    yield ctx
    ctx.set_epipolar_options()


@pytest.fixture(scope="module")
def epi():
    binding_epipolar.build()
    return binding_epipolar


def _same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)].view(np.uint64),
                                                                        b[~np.isnan(b)].view(np.uint64))


def _match(ctx, name, idx=None):
    """One match-only launch over the candidates idx (default all) of candidates(name), both keyframes in the table."""
    s, c = ec.scene(name), ec.candidates(name)
    idx = np.arange(len(c["kind"])) if idx is None else np.asarray(idx)
    frames = [ctx.frame(p) for p in s["kf_pyr"]]
    cur = ctx.frame(s["cur_pyr"])
    g = ctx.find_epipolar_match_direct(frames, s["kf_T"], cur, s["T_cur_w"], s["cam"], c["ref_index"][idx], c["ftr_px"][idx],
                                       c["ftr_f"][idx], c["ftr_level"][idx], c["ftr_type"][idx], c["ftr_grad"][idx],
                                       c["d_est"][idx], c["d_min"][idx], c["d_max"][idx], max_search_level=ec.N_LEVELS - 1)
    g["h_inv"], g["ran_1d"] = ctx.epipolar_last_h_inv(len(idx))
    for f in frames + [cur]:
        f.destroy()
    return g


def _check_one(g, j, o, what):
    assert bool(g["success"][j]) == o["success"] and bool(g["reject"][j]) == o["reject"], what
    assert g["search_level"][j] == o["search_level"], what
    assert bool(g["ran_1d"][j]) == o["ran_1d"] and _same(g["h_inv"][j], o["h_inv"]), (what, g["h_inv"][j], o["h_inv"])
    assert np.allclose(g["px_cur"][j], o["px_cur"], rtol=0, atol=1e-4, equal_nan=True), (what, g["px_cur"][j], o["px_cur"])
    if o["success"]:
        assert np.isclose(g["depth"][j], o["depth"], rtol=1e-6, atol=0), what


@pytest.mark.parametrize("name", CAMS)
def test_epipolar_options_kernel_vs_oracle_and_reference(ectx, epi, name):
    """Every setting of the grid, one launch each: statuses, rejects, search levels and ZMSSD counts exact, px_cur within
    1e-4 px, depth within 1e-6, h_inv_ and whether align1D ran exact -- against the oracle, and (but for the counts, which
    the reference does not expose) against the reference's outputs recorded for the oracle's pin."""
    c = ec.candidates(name)
    r = RefCalls("test_epipolar_options_pins", f"test_epipolar_options_oracle_equals_reference[{name}]")
    runs = {}
    for j, label, opt in [(j, lab, o) for lab, o in ec.settings() for j in range(len(c["kind"]))
                          if o["edgelet_max_angle"] == 0.7 or c["ftr_type"][j] == 1]:
        runs.setdefault(label, (opt, []))[1].append(j)
    n_ref = 0
    for label, (opt, js) in runs.items():
        ectx.set_epipolar_options(**opt)
        g = _match(ectx, name)
        for j in js:
            o = ec.oracle_match(epi, name, j, opt)
            _check_one(g, j, o, (name, label, j))
            assert g["n_zmssd"][j] == o["n_zmssd"], (name, label, j)
            _check_one(g, j, ec.ref_match(r, name, j, opt), (name, label, j, "reference"))
            n_ref += 1
    r.finish()
    assert n_ref > 1000


@pytest.mark.parametrize("name", CAMS)
def test_epipolar_options_kernel_edgelet_angle_at_its_cosangle(ectx, epi, name):
    """The kernel's filter at its own cosangle (found by bisection over launches): kept at cosangle, rejected at the next
    double above; its cosangle is the oracle's within 1e-12."""
    for j in ec.threshold_candidates(name):
        def rejected(ang):
            ectx.set_epipolar_options(edgelet_max_angle=ang)
            return bool(_match(ectx, name, [j])["reject"][0])

        lo, hi = np.float64(0.0).view(np.int64), np.float64(1.0).view(np.int64)
        assert not rejected(0.0) and rejected(1.0)
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if rejected(float(np.int64(mid).view(np.float64))):
                hi = mid
            else:
                lo = mid
        cos = float(np.int64(lo).view(np.float64))
        assert not rejected(cos) and rejected(float(np.nextafter(cos, 2.0)))
        oc = ec.cosangle_threshold(epi, name, j, binding_epipolar.DEFAULTS)
        assert abs(cos - oc) <= 1e-12 * oc, (name, j, cos, oc)


def test_epipolar_options_defaults_explicit_equal_never_set(ectx):
    """Setting the defaults explicitly is not setting them: bit-identical outputs of the match-only launch and the filter."""
    name = "pinhole_radtan"
    s, k = ec.scene(name), ec.seeds(name)
    ectx.set_epipolar_options(align_1d=True)  # something else first, then the defaults by value and by NULL

    def both():
        g = _match(ectx, name)
        frames = [ectx.frame(p) for p in s["kf_pyr"]]
        cur = ectx.frame(s["cur_pyr"])
        d = ectx.depth_filter_update(frames, s["kf_T"], cur, s["T_cur_w"], s["cam"], k["ref_index"], k["ftr_px"], k["ftr_f"],
                                     k["ftr_level"], k["ftr_type"], k["ftr_grad"], k["batch_id"], k["batch_counter"], k["seeds"])
        for f in frames + [cur]:
            f.destroy()
        return g, d

    ectx.lib.svo_b200_set_epipolar_options(ectx.h, None)
    g0, d0 = both()
    ectx.set_epipolar_options(align_1d=False, subpix_refinement=True, edgelet_filtering=True, edgelet_max_angle=0.7)
    g1, d1 = both()
    for a, b in ((g0, g1), (d0, d1)):
        for key in a:
            assert np.array_equal(np.asarray(a[key]).view(np.uint8), np.asarray(b[key]).view(np.uint8)), key
    assert not g0["ran_1d"].any() and not g0["h_inv"].any()


def test_epipolar_options_instantiation_by_setting(ectx):
    """The defaults, set or not, launch depth_filter_kernel<false>; any other setting launches depth_filter_kernel<true>."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    def kernels(**opt):
        ectx.set_epipolar_options(**opt)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _match(ectx, "pinhole", [0, 1, 2])
            torch.cuda.synchronize()
        return {e.name for e in prof.events() if "depth_filter_kernel" in e.name}

    assert all("<false>" in k for k in kernels()) and kernels()
    assert all("<true>" in k for k in kernels(edgelet_max_angle=0.5)) and kernels(edgelet_max_angle=0.5)
    assert all("<true>" in k for k in kernels(align_1d=True))


def test_epipolar_options_streams_equal_single_calls(ectx):
    """svo_b200_depth_filter_update_streams under a non-default setting: the three cameras' seeds as three streams of one
    launch (one keyframe table of all six keyframes) are bit for bit three single calls."""
    ectx.set_epipolar_options(align_1d=True, subpix_refinement=False, edgelet_max_angle=0.5)
    kf_frames, kf_T, streams, singles, owned = [], [], [], [], []
    for name in CAMS:
        s, k = ec.scene(name), ec.seeds(name)
        fr = [ectx.frame(p) for p in s["kf_pyr"]]
        cur = ectx.frame(s["cur_pyr"])
        owned += fr + [cur]
        singles.append(ectx.depth_filter_update(fr, s["kf_T"], cur, s["T_cur_w"], s["cam"], k["ref_index"], k["ftr_px"], k["ftr_f"],
                                                k["ftr_level"], k["ftr_type"], k["ftr_grad"], k["batch_id"], k["batch_counter"],
                                                k["seeds"]))
        streams.append(dict(k, cur=cur, cur_T_f_w=s["T_cur_w"], cam=s["cam"], ref_index=k["ref_index"] + len(kf_frames)))
        kf_frames += fr
        kf_T += list(s["kf_T"])
    outs = ectx.depth_filter_update_streams(streams, kf_frames, kf_T)
    for o, g in zip(outs, singles):
        for key in g:
            assert np.array_equal(np.asarray(o[key]).view(np.uint8), np.asarray(g[key]).view(np.uint8)), key
    assert sum(int((g["status"] >= 5).sum()) for g in singles) > 20
    for f in owned:
        f.destroy()


@pytest.mark.parametrize("name", CAMS)
def test_depth_filter_options_kernel_vs_oracle_and_reference(ectx, epi, name):
    """The filter under each setting of the oracle's pin: the kernel against the oracle as the depth filter's edge tests
    check it (statuses and ZMSSD counts exact, seeds bit for bit or one of the exactly rounded statement's candidates,
    px_cur -- what setGridOccpuancy reads -- within 1e-4 px, depth within 1e-6), and the statuses against the reference's
    recorded ones."""
    from tests.test_epipolar_options_pins import DF_SETTINGS, _ref_status

    s, k = ec.scene(name), ec.seeds(name)
    r = RefCalls("test_epipolar_options_pins", f"test_depth_filter_options_oracle_equals_reference[{name}]")
    frames = [ectx.frame(p) for p in s["kf_pyr"]]
    cur = ectx.frame(s["cur_pyr"])
    c = dict(k, T_cur_w=s["T_cur_w"], cam=s["cam"])
    for label, opt in DF_SETTINGS:
        ectx.set_epipolar_options(**opt)
        g = ectx.depth_filter_update(frames, s["kf_T"], cur, s["T_cur_w"], s["cam"], k["ref_index"], k["ftr_px"], k["ftr_f"],
                                     k["ftr_level"], k["ftr_type"], k["ftr_grad"], k["batch_id"], k["batch_counter"], k["seeds"])
        o = ec.oracle_update(epi, name, opt)
        _check_update(g, o, c, s["kf_T"], min_updated=5)
        rr = ec.ref_update(r, name, opt)
        assert np.array_equal(_ref_status(g["status"]), rr["status"]), label
    r.finish()
    for f in frames + [cur]:
        f.destroy()


def test_epipolar_options_refused_settings_change_nothing(ectx):
    """A flag other than 0 or 1 is refused and leaves the setting; a refused match call leaves the last h_inv_ query."""
    ectx.set_epipolar_options(align_1d=True, edgelet_max_angle=math.nan)
    before = ectx.epipolar_options()
    for bad in (dict(align_1d=2), dict(subpix_refinement=-1), dict(edgelet_filtering=7)):
        with pytest.raises(capi.SvoB200Error):
            ectx.set_epipolar_options(**dict(dict(align_1d=True, edgelet_max_angle=math.nan), **bad))
        after = ectx.epipolar_options()
        assert after["align_1d"] and after["subpix_refinement"] and after["edgelet_filtering"]
        assert math.isnan(after["edgelet_max_angle"]) and math.isnan(before["edgelet_max_angle"])
    g = _match(ectx, "pinhole")
    s, c = ec.scene("pinhole"), ec.candidates("pinhole")
    fr, cur = ectx.frame(s["kf_pyr"][0]), ectx.frame(s["cur_pyr"])
    with pytest.raises(capi.SvoB200Error):
        ectx.find_epipolar_match_direct([fr], [s["kf_T"][0]], cur, s["T_cur_w"], s["cam"], np.array([3], np.int32),
                                        c["ftr_px"][:1], c["ftr_f"][:1], c["ftr_level"][:1], c["ftr_type"][:1], c["ftr_grad"][:1],
                                        c["d_est"][:1], c["d_min"][:1], c["d_max"][:1])
    fr.destroy(); cur.destroy()
    h, ran = ectx.epipolar_last_h_inv(len(c["kind"]))
    assert _same(h, g["h_inv"]) and np.array_equal(ran, g["ran_1d"]) and ran.any()
    with pytest.raises(capi.SvoB200Error):
        ectx.epipolar_last_h_inv(len(c["kind"]) + 1)


def test_host_epipolar_options_demo():
    """svo_host.h: a DepthFilter subclass setting matcher_.options_, Matcher::h_inv_, a refused mixed streams call."""
    out = subprocess.run([build_demo("host_epipolar_options_demo")], capture_output=True, text=True, timeout=600)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "epipolar options demo: ok" in out.stdout
