"""CPU: the exactly rounded statement of updateSeed / computeTau (tests/depth_update_hp.py) against the oracle, bit for
bit, with glibc's expf, acos, sin and atan called as the oracle calls them; and the oracle against the compiled
reference's recorded outputs (tests/golden/ref/test_depth_update_pins.npz) on the same edges."""
import math

import numpy as np
import pytest

from rpg_svo_b200 import synth
from tests import depth_update_cases as cases
from tests import depth_update_hp as hp
from tests.ref_golden import ref  # noqa: F401 (fixture)

KEYS = ("a", "b", "mu", "sigma2")


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _evolved_tuples(n=300, seed=5):
    """Ordinary and far-out updates of evolved seeds: a, b over 0.5 .. 1e4, sigma2 over 1e-10 .. 1, tau2 over 1e-12 .. 1."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        x = rng.uniform(0.1, 2)
        mu = x * (1 + rng.normal(0, 10 ** rng.uniform(-4, 0)))
        out.append(tuple(float(np.float32(v)) for v in (x, 10 ** rng.uniform(-12, 0), 10 ** rng.uniform(-0.3, 4),
                                                      10 ** rng.uniform(-0.3, 4), mu, rng.choice([2.0, 0.5, 1e-3, 100.0]),
                                                      10 ** rng.uniform(-10, 0))))
    return out


def _tau_tuples():
    """(t, f, z, px_error_angle) of the small-parallax and evolved cases at their true depths, plus far and near z."""
    out = []
    for c in [cases.small_parallax(77, b, n_seeds=40) for b in cases.SMALL_BASELINES] + [cases.evolved(n_seeds=40)]:
        T = synth.se3_mul(c["T_ref_w"], synth.se3_inv(c["T_cur_w"]))
        pea = hp.px_error_angle(c["cam"].fx)
        for i in range(len(c["depth_gt"])):
            for z in (c["depth_gt"][i], c["depth_gt"][i] * 50, c["depth_gt"][i] * 1e-3):
                out.append((T, c["ftr_f"][i], float(z), pea))
    return out


def test_update_seed_statement_equals_oracle(oracle):
    tuples = cases.edge_tuples() + _evolved_tuples()
    for t in tuples:
        o = oracle.update_seed(*t)
        s = hp.update_seed(*t, hp.c_expf)
        got = tuple(float(o[j]) for j in (0, 1, 2, 4))
        assert all(hp.same(u, v) for u, v in zip(got, s)), (t, got, s)
    assert len(tuples) > 300


def test_compute_tau_statement_equals_oracle(oracle):
    n_neg = 0
    for T, f, z, pea in _tau_tuples():
        o = oracle.compute_tau(T, f, z, pea)
        s = hp.compute_tau(T[:, 3], f, z, pea)
        assert hp.same(o, s), (T, f, z, o, s)
        n_neg += o < -z
    assert n_neg > 0  # gamma_plus < 0 and z_plus < 0 among them
    assert hp.same(hp.px_error_angle(315.5), math.atan(1.0 / 631.0) * 2.0)


def _oracle_run(oracle, c):
    return oracle.depth_filter_update([c["ref_pyr"]], [c["T_ref_w"]], c["cur_pyr"], c["T_cur_w"], c["cam"], c["ref_index"],
                                      c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"], c["ftr_grad"], c["batch_id"],
                                      c["batch_counter"], c["seeds"])


@pytest.mark.parametrize("name", ["small_parallax_0.004", "small_parallax_0.05", "evolved", "degenerate"])
def test_oracle_depth_filter_update_restated_from_its_own_z(oracle, name):
    """The oracle's full DepthFilter::updateSeeds, every updated seed bit for bit: the statement from the oracle's own
    depth, with exp pinned to glibc's expf and tau2 to computeTau restated in IEEE double with glibc's acos / sin / atan
    from the oracle's own T_ref_cur (which must also lie among the floats of the computeTau enclosure)."""
    c = cases.small_parallax(77, float(name.rsplit("_", 1)[1])) if name.startswith("small") else getattr(cases, name)()
    o = _oracle_run(oracle, c)
    rep = hp.check_launch(o, c["seeds"], [c["T_ref_w"]], c["ref_index"], c["T_cur_w"], c["ftr_f"], c["cam"].fx, exp="glibc",
                          oracle=oracle)
    print(name, {k: v for k, v in rep.items() if k != "bad"})
    assert not rep["bad"], rep["bad"][:3]
    assert rep["n"] > 100 and rep["single"] == rep["n"] and rep["k"] == {0: rep["n"]}


def test_oracle_equals_reference(oracle, ref):
    """updateSeed and computeTau on the edge tuples bit for bit; DepthFilter::updateSeeds on the small-parallax and
    evolved cases: the same verdicts, b + 1 of unmatched seeds bit for bit, updated seeds within expf's and the
    reference's contracted arithmetic."""
    diff_seed = []
    for t in cases.edge_tuples() + _evolved_tuples(60):
        r, o = ref.update_seed(*t), oracle.update_seed(*t)
        if not all(hp.same(float(u), float(v)) for u, v in zip(r, o)):
            diff_seed.append((t, r, o))
    # The reference is built with GCC's default -ffp-contract=fast: computeTau's f * z - t and dot products become fused
    # multiply-adds there, so its tau differs from the oracle's (which spells IEEE double, like the kernel) in the last bits.
    diff_tau, worst = 0, 0.0
    for T, f, z, pea in _tau_tuples()[::7]:
        r, o = ref.compute_tau(T, f, z, pea), oracle.compute_tau(T, f, z, pea)
        diff_tau += not hp.same(r, o)
        worst = max(worst, abs(r - o) / abs(o))
    print(f"updateSeed: {len(diff_seed)} tuples differ from the reference; computeTau: {diff_tau} differ, "
          f"by at most {worst:.3g} relative")
    for d in diff_seed[:5]:
        print("  ", d)
    assert not diff_seed and worst < 1e-9
    for c in [cases.small_parallax(77, 0.004), cases.small_parallax(77, 0.05), cases.evolved()]:
        o = _oracle_run(oracle, c)
        rr = ref.depth_filter_update([c["ref_pyr"][0]], [c["T_ref_w"]], c["cur_pyr"][0], c["T_cur_w"], c["n_levels"],
                                     c["cam"], c["ref_index"], c["ftr_px"], c["ftr_f"], c["ftr_level"], c["ftr_type"],
                                     c["ftr_grad"], c["batch_id"], c["batch_counter"], c["seeds"])
        st = o["status"]
        assert np.array_equal(rr["status"], np.where(st == 6, 1, np.where((st == 1) | (st == 7), 2, 0)))
        nm = st == 4
        for k in KEYS:
            assert np.array_equal(_bits(rr[k][nm]), _bits(o[k][nm])), k
        kept = (st == 5) & (rr["status"] == 0)
        same = np.all([_bits(rr[k][kept]) == _bits(o[k][kept]) for k in KEYS], axis=0)
        print(f"updated seeds bit-identical to the reference: {int(same.sum())} of {int(kept.sum())}")
        for k in KEYS:
            assert np.allclose(rr[k][kept], o[k][kept], rtol=2e-5, atol=1e-7), k
