"""GPU: pose_opt_kernel (pose_optimizer::optimizeGaussNewton) against the high-precision statement of tests/pose_hp.py and
the compiled reference's recorded outputs on the case catalogue of tests/pose_hp_cases.py, batched launches of the whole
catalogue, the output bits of the ordinary frames against the parent commit, and the refusals of
svo_b200_pose_optimize_batch.

A frame whose every decision is decisive must take the exact run's decisions: n_iter_done, estimated_scale, has_point
and num_obs exact, error_init and error_final inside their candidate intervals, the pose within the run's bound and the
covariance within (A fx^2)^-1's bound; a frame with a near-tie may end on any run `pose_hp.branches` allows."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from rpg_svo_b200 import synth
from rpg_svo_b200.capi import PoseOptResult, _p, c64
from tests import pose_hp as hp
from tests import pose_hp_cases as pc
from tests.ref_golden import RefCalls
from tests.test_pose_hp_pins import ROLLBACK_COV, reference_outputs, same_as_reference

pytestmark = pytest.mark.gpu

WORST = {"ratio": 0.0, "where": None}
CASES = pc.all_cases()


@pytest.fixture(scope="module")
def statements():
    """The branches of every catalogue case, computed once for the module."""
    return {c["name"]: hp.branches(*c["args"], exact=c["exact"]) for c in CASES}


def _check(g, c, runs):
    if c["name"] in pc.NAN_MEDIAN:
        assert g["estimated_scale"] == runs[0]["est_out"], c["name"]   # NaN above +inf: the statement's median exactly
    if c["name"] in pc.RANK_DEFICIENT:
        hp.assert_rank_deficient(g, runs[0])
        return runs[0]
    run, ratio, why = hp.match_any(g, runs, c["args"][2])
    assert run is not None, (c["name"], why, ratio, g["n_iter_done"], g["estimated_scale"], g["num_obs"])
    if hp.decisive(runs[0]):
        assert run is runs[0], c["name"]
    ok, cratio, checked = hp.cov_check(g, run, c["args"][2])
    assert ok, (c["name"], "cov", cratio)
    if c["name"] in ROLLBACK_COV:  # the covariance after a roll-back: the inverse of the rejected iteration's A, checked
        assert checked and run["trace"][-1]["decision"] == "rollback", c["name"]
    for r, where in ((ratio, c["name"]), (cratio, c["name"] + " cov")):
        if np.isfinite(r) and r > WORST["ratio"]:
            WORST.update(ratio=r, where=where)
    return run


@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_pose_kernel_matches_statement(ctx, statements, name):
    c = next(x for x in CASES if x["name"] == name)
    runs = statements[name]
    g = ctx.pose_optimize(*c["args"])
    run = _check(g, c, runs)
    r0, edge = runs[0], c["edge"]
    if edge.get("cull_exact"):   # the threshold stays, its upper neighbour goes, at every level
        assert hp.decisive(r0)
        assert g["has_point"].tolist() == [1, 1, 0] * 6 and g["num_obs"] == 12
    if edge.get("cull_majority"):
        assert g["num_obs"] == 3 and g["error_final"] > 2.0   # the median of all nine errors, a culled one (10 px)
    if edge.get("subnormal_scale"):
        assert 0 < g["estimated_scale"] / c["args"][2] < 1.2e-38                # a float-subnormal MAD scale
        assert np.isfinite(g["cov"]).all()                                     # zero errors keep their weight 1
    if edge.get("end"):
        assert r0["trace"] == [] if edge["end"] == "empty" else r0["trace"][-1]["decision"] == edge["end"], name
        if "at" in edge:
            assert r0["trace"][-1]["it"] == edge["at"]
    if edge.get("eps_side"):
        for r in runs:  # every MAD-scale candidate's run decides the EPS test the same way, decisively
            m = r["trace"][0]["eps_margin"]
            assert hp.decisive(r) and (m < 0) == (edge["eps_side"] == "below") and 0.02 < abs(m) < 0.04, m
        assert g["n_iter_done"] == (1 if edge["eps_side"] == "below" else 2)
    if edge.get("unconverged_at"):
        assert all(rec["decision"] == "step" for rec in r0["trace"][:5])
    print(f"{name}: decisions {[x.get('decision') for x in run['trace']]}, worst |kernel - exact| / bound so far "
          f"{WORST['ratio']:.3g} ({WORST['where']})")


def test_pose_batch_of_every_case_equals_single_calls(ctx, statements):
    """The whole catalogue in batched launches: svo_b200_pose_optimize_batch takes one reproj_thresh and one n_iter per
    launch, so the cases go in one launch per (reproj_thresh, n_iter) pair, each frame with its own fx, with
    obs_offset[0] > 0 (NaN observations with bad levels before it are never read).  Each frame is bit for bit its single
    call and within its statement's bound."""
    groups = {}
    for c in CASES:
        groups.setdefault(c["args"][:2], []).append(c)
    pre = 5
    for (rt, n_iter), cs in groups.items():
        frames = [c["args"] for c in cs]
        f = np.concatenate([np.full((pre, 3), np.nan)] + [a[4] for a in frames])
        pos = np.concatenate([np.full((pre, 3), np.nan)] + [a[5] for a in frames])
        lv = np.concatenate([np.full(pre, -7, np.int32)] + [a[6] for a in frames])
        hpv = np.concatenate([np.ones(pre, np.uint8)] + [a[7] for a in frames])
        off = (pre + np.concatenate([[0], np.cumsum([len(a[7]) for a in frames])])).astype(np.int32)
        res = ctx.pose_optimize_batch(rt, n_iter, [a[2] for a in frames], np.stack([a[3] for a in frames]), off, f, pos, lv,
                                      hpv)
        for a, r, c in zip(frames, res, cs):
            g = ctx.pose_optimize(*a)
            assert np.array_equal(r["T"].view(np.int64), g["T"].view(np.int64)), c["name"]
            assert np.array_equal(r["has_point"], g["has_point"]), c["name"]
            for k in ("num_obs", "n_iter_done", "estimated_scale", "error_init", "error_final"):
                assert r[k] == g[k] or (np.isnan(r[k]) and np.isnan(g[k])), (c["name"], k)
            assert np.array_equal(r["cov"], g["cov"], equal_nan=True), c["name"]
            _check(r, c, statements[c["name"]])
    assert len(groups) < len(CASES)


def test_pose_kernel_matches_reference(ctx):
    """The kernel against the compiled reference's outputs recorded for tests/test_pose_hp_pins.py (replayed; the inputs
    must hash to the recorded ones)."""
    r = RefCalls("test_pose_hp_pins", "test_pose_oracle_matches_reference")
    refs = reference_outputs(r)
    r.finish()
    for c, rr in zip(CASES, refs):
        same_as_reference(ctx.pose_optimize(*c["args"]), rr, c)


# SHA-256 of every output of pose_optimize / pose_optimize_batch on the synth.make_pose_opt_case frames of
# tests/test_pose_depth_gpu.py as the parent commit computed them on an H100 (this module's _digest run against the parent
# commit's build, before the reciprocal range guard): the guard
# changes no bit of an in-range frame.
PARENT_DIGEST = "c5919aefc988c0a8d0e465208a93050036befa20ae2c83a3688bc8b0ad3de7a4"


def _digest(ctx) -> str:
    h = hashlib.sha256()

    def put(g):
        for k in sorted(g):
            a = np.ascontiguousarray(g[k])
            h.update(k.encode() + a.dtype.str.encode() + str(a.shape).encode() + a.tobytes())

    for n, size in [(1000, (1920, 1080)), (120, (752, 480)), (7, (640, 480))]:
        c = synth.make_pose_opt_case(5 + n, n, *size)
        put(ctx.pose_optimize(2.0, 10, c["cam"].fx, c["T_init"], c["f"], c["pos"], c["level"], c["has_point"]))
    cases = [synth.make_pose_opt_case(40 + k, n, *size) for k, (n, size) in
             enumerate([(1000, (1920, 1080)), (120, (752, 480)), (9, (640, 480)), (300, (640, 480))])]
    cases[2]["has_point"][:] = 0
    off = np.concatenate([[0], np.cumsum([len(c["level"]) for c in cases])]).astype(np.int32)
    cat = lambda k: np.concatenate([c[k] for c in cases])
    for r in ctx.pose_optimize_batch(2.0, 10, [c["cam"].fx for c in cases], np.stack([c["T_init"] for c in cases]), off,
                                     cat("f"), cat("pos"), cat("level"), cat("has_point")):
        put(r)
    return h.hexdigest()


def test_pose_output_bits_unchanged(ctx):
    assert _digest(ctx) == PARENT_DIGEST


def test_pose_batch_refusals_write_nothing(ctx):
    """A refused call -- a negative first offset, a decreasing offset, an observation with a point at level -1 or 31, a
    frame beyond the shared-memory capacity -- returns its error before anything is launched or written: a sentinel-filled
    `out`, T and has_point come back unchanged."""
    lib = ctx.lib
    n = 8
    f = c64(np.tile([0.1, 0.05, 1.0], (n, 1)))
    pos = c64(np.tile([0.0, 0.0, 2.0], (n, 1)))
    big = 4000
    for what, off, lvl, nobs, rc_want in (("negative offset", [-1, n], 0, n, -1), ("decreasing", [0, n, 2], 0, n, -1),
                                          ("level -1", [0, n], -1, n, -1), ("level 31", [0, n], 31, n, -1),
                                          ("capacity", [0, big], 0, big, -4)):
        B = len(off) - 1
        fb = c64(np.tile([0.1, 0.05, 1.0], (nobs, 1)))
        pb = c64(np.tile([0.0, 0.0, 2.0], (nobs, 1)))
        lv = np.zeros(nobs, np.int32)
        lv[3 % nobs] = lvl
        hpv = np.ones(nobs, np.uint8)
        hsnap = hpv.copy()
        T = c64(np.full((B, 12), 7.25))
        Tsnap = T.copy()
        out = (PoseOptResult * B)()
        C.memset(out, 0x5A, C.sizeof(out))
        osnap = bytes(out)
        fx = c64([300.0] * B)
        o = np.array(off, np.int32)
        n0 = ctx.launch_count()
        rc = lib.svo_b200_pose_optimize_batch(ctx.h, B, C.c_double(2.0), 10, _p(fx), _p(T), _p(o), _p(fb), _p(pb), _p(lv),
                                              _p(hpv), out)
        assert rc == rc_want, (what, rc)
        assert ctx.launch_count() == n0, what
        assert bytes(out) == osnap, what
        assert np.array_equal(T.view(np.int64), Tsnap.view(np.int64)) and np.array_equal(hpv, hsnap), what
    # a level outside [0, 30] on an observation without a point is never read: accepted
    lv = np.full(n, 99, np.int32)
    hpv = np.zeros(n, np.uint8)
    hpv[0] = 1
    lv[0] = 0
    g = ctx.pose_optimize(2.0, 10, 300.0, synth.se3_identity(), f, pos, lv, hpv)
    assert g["num_obs"] == 1
    print(f"module: worst |kernel - exact| / bound {WORST['ratio']:.3g} ({WORST['where']})")
