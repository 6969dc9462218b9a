"""CPU tests of the update between two chained corrections (b2_micp_correct): the convergence progress of micp_localization.cpp:988-1007 and
the adaptive gate of CorrespondencesCPU.cpp:21-23, as the product computes them (icp_loop.cuh, compiled for the CPU by tests/chain_ref.py) and
as a C restatement / the oracle state them; and the reference chain (chain_ref.oracle_chain) against single oracle steps fed from outside."""
import numpy as np
import pytest

import chain_ref
from chain_ref import progress_np
from conftest import mesh


def _ulps(a, b):
    a, b = np.float32(a), np.float32(b)
    if a == b:
        return 0
    return abs(int(a.view(np.int32)) - int(b.view(np.int32)))


def _inputs(synth):
    """(Tom, T_onew_oold, n_meas, valid, adaptive): random poses near and far from the origin, plus the edges"""
    rng = np.random.default_rng(7)
    cases = []
    for k in range(400):
        scale = (0.02, 0.1, 0.3, 1.0, 9.5, 50.0)[k % 6]           # |t| ~ 9-10: trans_progress is a float denormal
        Tom = synth.make_transform(tuple(rng.uniform(-scale, scale, 3)), tuple(rng.uniform(-0.4, 0.4, 3)))
        Td = synth.make_transform(tuple(rng.normal(0, 0.05, 3)), tuple(rng.normal(0, 0.02, 3)))
        if k % 5 == 0:
            Tom["R"] = -Tom["R"]                                  # negative w: the same rotation, rot_progress = w^2 unchanged
        valid = int(rng.integers(1, 200000))
        cases.append((Tom, Td, int(rng.integers(1, valid + 1)), valid, True))
    I = synth.make_transform()
    Tfar = synth.make_transform((1e4, -3e3, 2e2), (0.1, 0.0, 2.0))
    cases += [(I, I, 100, 100, True), (I, I, 0, 100, True), (I, I, 100, 100, False), (Tfar, I, 5, 10, True),
              (synth.make_transform((0.01, 0, 0), (0, 0, 3.1)), I, 1, 3, True), (I, synth.make_transform((0.0, 0.0, 0.0), (np.pi, 0, 0)), 7, 7, True)]
    return cases


def test_progress_emul_equals_oracle(po, synth):
    """The product's update (icp_loop.cuh: micp_progress, run on the CPU) equals the oracle's C restatement bit for bit on random and edge inputs
    (n_meas = 0, adaptive off, large |t|, negative w); both are within one float ulp of the numpy restatement."""
    seen = {"zero": 0, "denormal": 0, "big": 0}
    for Tom, Td, n, valid, adaptive in _inputs(synth):
        a = chain_ref.product_progress(Tom, Td, n, valid, adaptive)
        b = chain_ref.oracle_progress(po, Tom, Td, n, valid, adaptive)
        c = progress_np(po, Tom, Td, n, valid, adaptive)
        assert np.float64(a).tobytes() == np.float64(b).tobytes(), (a, b)
        assert np.float32(a) == a                                  # a float widened to double (:1002, :1006)
        assert _ulps(a, c) <= 1 and _ulps(b, c) <= 1, (a, b, c)
        seen["zero"] += a == 0.0
        seen["denormal"] += 0.0 < a < np.finfo(np.float32).tiny
        seen["big"] += a > 0.5
    assert seen["zero"] >= 3 and seen["denormal"] >= 1 and seen["big"] >= 3, seen


def test_adaptive_gate_emul_equals_oracle(po):
    """The loop's gate for a chain step (icp_adaptive_max_dist) is the oracle's / the host's expression bit for bit."""
    rng = np.random.default_rng(3)
    for md, mn, cp in [(1.0, 0.15, 0.0), (1.0, 0.15, 1.0), (0.5, 0.5, 0.3)] + [tuple(x) for x in rng.uniform(0, 3, (200, 3))]:
        cp = float(cp) / 3.0
        assert np.float32(chain_ref.product_gate(md, mn, cp)) == np.float32(po.adaptive_max_dist(md, mn, cp))


def _scene(po, synth):
    V, F = mesh("cube29")
    osc = po.Scene(V, F)
    Tgt = synth.make_transform((0.04, -0.02, 0.01), (0.0, 0.0, 0.02))
    sensors = []
    for k, (m, Tsb) in enumerate(((synth.c1_sensor(), synth.make_transform((0.1, 0, 0.2), (0, 0, 0.05))),
                                  (synth.PinholeModel(32, 24, 26.25, 26.25, 15.5, 11.5, 0.1, 30.0), synth.make_transform((0.05, 0.1, 0.3), (0, 0.1, -0.3))))):
        o, d = po.model_rays(m)
        r = synth.noisy_ranges(osc.simulate(Tgt, Tsb, o, d, m.range_max)["ranges"], m.range_max, seed=k)
        r[np.random.default_rng(9 + k).random(r.shape) < 0.06] += np.float32(0.7)
        dp, dm, _ = po.dataset_from_ranges(o, d, r, m.range_min, m.range_max)
        sensors.append(dict(origs=o, dirs=d, range_max=m.range_max, dataset_points=dp, dataset_mask=dm, Tbo=synth.make_transform((0.01 * k, 0, 0), (0, 0, 0.01)),
                            Tsb=Tsb, max_dist=1.0, adaptive_max_dist_min=0.15, weight=(1.0, 0.35)[k]))
    Tom = synth.compose(Tgt, synth.make_transform((0.08, -0.05, 0.03), (0.0, 0.0, 0.03)))
    return osc, sensors, Tom


@pytest.mark.parametrize("adaptive", [True, False])
def test_oracle_chain_equals_fed_steps(po, synth, adaptive):
    """The reference chain of N steps equals N orc_micp_correct_once_multi calls, each at the previous Tom_new and with the numpy progress of the
    previous step."""
    osc, sensors, Tom = _scene(po, synth)
    valid = int(sum(int((sd["dataset_mask"] > 0).sum()) for sd in sensors))
    T, cp, steps = chain_ref.oracle_chain(po, osc, sensors, Tom, n_corrections=4, iterations=5, convergence_progress=0.0, adaptive_max_dist=adaptive)
    Tc, cpc = Tom, 0.0
    for s in range(4):
        Tn, Td, Cm = osc.micp_correct_once_multi(sensors, Tc, 5, cpc, f64_accum=True)
        assert Tn.tobytes() == steps[s]["Tom_new"].tobytes() and Td.tobytes() == steps[s]["T_onew_oold"].tobytes()
        assert Cm.tobytes() == steps[s]["Cmerged_o"].tobytes()
        cpc = progress_np(po, Tc, Td, int(Cm["n_meas"]), valid, adaptive)
        assert steps[s]["convergence_progress"] == cpc and steps[s]["valid_measurements"] == valid
        Tc = Tn
    assert T.tobytes() == Tc.tobytes() and cp == cpc
    if adaptive:
        assert steps[-1]["convergence_progress"] > 0.1                 # near the map origin the progress grows (SURVEY.md D12)
    else:
        assert (steps["convergence_progress"] == 0.0).all()
