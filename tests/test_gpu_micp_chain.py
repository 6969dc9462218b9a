"""b2_micp_correct: chained correctOnce steps on the device (micp_localization.cpp:847-1007), run on an H100 (pytest -m gpu).

Bars: per step, the chain is bit-identical to host-fed b2_micp_correct_once calls given the previous Tom_new and the chain's reported
progress (same kernels, same inputs); each progress is within one float ulp of the numpy restatement (chain_ref.progress_np); against
the oracle's chain (FP64 sums) the pose is within 1e-5 per step and n_meas is equal."""
import ctypes as C

import numpy as np
import pytest

from conftest import gpu_map, mesh, quat_close
import chain_ref
from chain_ref import progress_np

pytestmark = pytest.mark.gpu
TOL_DT = 1e-5


def _ulp_close(a, b):
    a, b = np.float32(a), np.float32(b)
    return abs(float(a) - float(b)) <= float(np.spacing(max(abs(a), abs(b), np.float32(np.finfo(np.float32).tiny))))


def _near_origin_case(po, synth):
    """Four sensors on a robot near the map origin inside the 20 m cube (the progress only grows there: SURVEY.md D12), scans taken at T_gt with
    1 cm noise and 6 % ghost returns 0.7 m behind the wall (kept by the full gate, cut once the progress narrows it)."""
    V, F = mesh("cube29")
    osc = po.Scene(V, F)
    Tgt = synth.make_transform((0.03, -0.02, 0.01), (0.0, 0.0, 0.02))
    models = [synth.SphericalModel(np.radians(-40.0), np.radians(80.0) / 23, 24, -np.pi, 2 * np.pi / 256, 256, 0.1, 100.0),
              synth.PinholeModel(64, 48, 52.5, 52.5, 31.5, 23.5, 0.1, 30.0),
              synth.SphericalModel(np.radians(-30.0), np.radians(60.0) / 15, 16, -np.pi, 2 * np.pi / 128, 128, 0.1, 100.0),      # closest point
              synth.SphericalModel(np.radians(-20.0), np.radians(40.0) / 11, 12, -np.pi, 2 * np.pi / 96, 96, 0.1, 100.0)]
    Tsbs = [synth.make_transform((0.1, 0.0, 0.2), (0, 0, 0.05)), synth.make_transform((0.05, 0.1, 0.3), (0.0, 0.1, -0.3)),
            synth.make_transform((0.0, -0.1, 0.1), (0, 0, -0.1)), synth.make_transform((-0.05, 0.0, 0.25), (0.02, 0, 0.2))]
    Tbos = [synth.make_transform((0.01, 0.0, 0.0), (0, 0, 0.01)), synth.make_transform((0.0, 0.01, 0.0), (0, 0, 0.012)),
            synth.make_transform((0.01, 0.01, 0.0), (0, 0, 0.008)), synth.make_transform((0.0, 0.0, 0.0), (0, 0, 0.011))]
    sensors = []
    for k, (m, Tsb, Tbo) in enumerate(zip(models, Tsbs, Tbos)):
        o, d = po.model_rays(m)
        r = synth.noisy_ranges(osc.simulate(Tgt, Tsb, o, d, m.range_max)["ranges"], m.range_max, seed=20 + k)
        ghost = np.random.default_rng(30 + k).random(r.shape) < 0.06
        r[ghost & (r < m.range_max)] += np.float32(0.7)
        dp, dm, _ = po.dataset_from_ranges(o, d, r, m.range_min, m.range_max)
        sensors.append(dict(model=m, origs=o, dirs=None if k == 2 else d, range_max=m.range_max, dataset_points=dp, dataset_mask=dm, Tbo=Tbo, Tsb=Tsb,
                            max_dist=1.0, adaptive_max_dist_min=0.15, weight=(1.0, 0.35, 0.6, 2.0)[k], ranges=r))
    Tom = synth.compose(synth.compose(Tgt, synth.make_transform((0.08, -0.05, 0.03), (0.0, 0.0, 0.03))), synth.inverse(Tbos[0]))
    return osc, sensors, Tom


def _handles(sensors, bind=False):
    import torch
    import rmcl_b200
    hs, keep = [], []
    for k, sd in enumerate(sensors):
        if sd["dirs"] is None:
            h = rmcl_b200.CPCB200(gpu_map("cube29"))
        else:
            cls = rmcl_b200.RCCB200Pinhole if type(sd["model"]).__name__ == "PinholeModel" else rmcl_b200.RCCB200Spherical
            h = cls(gpu_map("cube29"))
            h.setModel(sd["model"])
        h.setTsb(sd["Tsb"]); h.setParams(1.0, 0.15)
        if sd["dirs"] is None:
            h.setDataset(sd["dataset_points"], sd["dataset_mask"])
        elif bind and k == 3:
            p, mk = torch.from_numpy(sd["dataset_points"].copy()).cuda(), torch.from_numpy(sd["dataset_mask"].copy()).cuda()
            h.bindDataset(p, mk)
            keep += [p, mk]
        else:
            h.setRanges(sd["ranges"])
        hs.append(h)
    return hs, keep


def _tbo(sensors):
    return np.stack([sd["Tbo"] for sd in sensors])


def _host_fed_equal(hs, Tbo, Tom, cp0, w, steps, iterations=5):
    import rmcl_b200
    T, cp = Tom, cp0
    for s, rec in enumerate(steps):
        Tn, Td, Cm = rmcl_b200.micp_correct_once(hs, Tbo, T, iterations, cp, merge_weights=w)
        assert Tn.tobytes() == rec["Tom_new"].tobytes(), s
        assert Td.tobytes() == rec["T_onew_oold"].tobytes(), s
        assert Cm.tobytes() == rec["Cmerged_o"].tobytes(), s
        T, cp = Tn, float(rec["convergence_progress"])


@pytest.mark.parametrize("ns", [1, 2, 4])
def test_chain_equals_host_fed_steps(po, synth, ns):
    """Per step, the chain's Tom_new / T_onew_oold / Cmerged_o equal host-fed b2_micp_correct_once calls bit for bit; each step's progress is within
    one float ulp of the numpy restatement; 1 sensor (spherical), 2 (+ pinhole, merge weight 0.35), 4 (+ closest point, + bound dataset)."""
    import rmcl_b200
    osc, sensors, Tom = _near_origin_case(po, synth)
    sensors = sensors[:ns]
    hs, keep = _handles(sensors, bind=True)
    Tbo = _tbo(sensors)
    w = None if ns == 1 else [sd["weight"] for sd in sensors]
    valid = int(sum(int((sd["dataset_mask"] > 0).sum()) for sd in sensors))
    for n, cp0 in ((1, 0.0), (3, 0.0), (4, 0.25)):
        T, cp, steps = rmcl_b200.micp_correct(hs, Tbo, Tom, n_corrections=n, iterations=5, convergence_progress=cp0, merge_weights=w)
        assert len(steps) == n
        _host_fed_equal(hs, Tbo, Tom, cp0, w, steps)
        assert T.tobytes() == steps[-1]["Tom_new"].tobytes() and cp == steps[-1]["convergence_progress"]
        Tprev = Tom
        for rec in steps:
            assert rec["valid_measurements"] == valid and rec["total_measurements"] == sum(len(sd["dataset_mask"]) for sd in sensors)
            want = progress_np(po, Tprev, rec["T_onew_oold"], int(rec["Cmerged_o"]["n_meas"]), valid)
            assert _ulp_close(rec["convergence_progress"], want), (rec["convergence_progress"], want)
            Tprev = rec["Tom_new"]
        assert steps[-1]["convergence_progress"] > 0.1


def test_chain_against_oracle(po, synth):
    """Against the oracle's chain (chain_ref.oracle_chain, FP64 sums): pose within 1e-5 per step, n_meas equal.  Near the map origin the progress
    passes 0.1 and the narrowed gate drops the ghost returns: n_meas differs from the same chain with adaptive_max_dist = 0 (progress 0)."""
    import rmcl_b200
    osc, sensors, Tom = _near_origin_case(po, synth)
    sensors = sensors[:2]
    hs, _ = _handles(sensors)
    Tbo = _tbo(sensors)
    w = [sd["weight"] for sd in sensors]
    got = {}
    for adaptive in (True, False):
        T, cp, steps = rmcl_b200.micp_correct(hs, Tbo, Tom, n_corrections=3, iterations=5, merge_weights=w, adaptive_max_dist=adaptive)
        Tr, cpr, ref = chain_ref.oracle_chain(po, osc, sensors, Tom, n_corrections=3, iterations=5, adaptive_max_dist=adaptive)
        for s in range(3):
            assert int(steps[s]["Cmerged_o"]["n_meas"]) == int(ref[s]["Cmerged_o"]["n_meas"]), (adaptive, s)
            assert np.abs(steps[s]["Tom_new"]["t"] - ref[s]["Tom_new"]["t"]).max() <= TOL_DT
            assert quat_close(steps[s]["Tom_new"]["R"], ref[s]["Tom_new"]["R"], TOL_DT)
            assert abs(steps[s]["convergence_progress"] - ref[s]["convergence_progress"]) <= 1e-4
            assert steps[s]["valid_measurements"] == ref[s]["valid_measurements"]
        got[adaptive] = steps
    assert got[True][0]["convergence_progress"] > 0.1 and (got[False]["convergence_progress"] == 0).all()
    assert got[True][2]["Cmerged_o"]["n_meas"] < got[False][2]["Cmerged_o"]["n_meas"] - 50


def test_measurement_counts(po, synth):
    """valid_measurements = mask ones of the datasets, total_measurements = dataset sizes, for set_ranges, set_dataset and bind_dataset."""
    import torch
    import rmcl_b200
    osc, sensors, Tom = _near_origin_case(po, synth)
    sd = sensors[0]
    hs, _ = _handles([sd])
    h = hs[0]
    n = len(sd["dataset_mask"])
    want = int((sd["dataset_mask"] > 0).sum())
    assert 0 < want < n
    _, _, st = rmcl_b200.micp_correct([h], _tbo([sd]), Tom, n_corrections=2)
    assert (st["valid_measurements"] == want).all() and (st["total_measurements"] == n).all()
    mask = (np.arange(n) % 3 != 0).astype(np.uint8) * sd["dataset_mask"]
    h.setDataset(sd["dataset_points"], mask * 7)                                       # any value > 0 counts
    _, _, st = rmcl_b200.micp_correct([h], _tbo([sd]), Tom, n_corrections=1)
    assert st[0]["valid_measurements"] == int((mask > 0).sum()) and st[0]["total_measurements"] == n
    p, mk = torch.from_numpy(sd["dataset_points"].copy()).cuda(), torch.from_numpy(mask.copy()).cuda()
    h.bindDataset(p, mk)
    _, _, st = rmcl_b200.micp_correct([h], _tbo([sd]), Tom, n_corrections=1)
    assert st[0]["valid_measurements"] == int((mask > 0).sum())


def test_chain_edges(po, synth):
    """iterations = 0, empty sensors, steps_out = NULL, refusal with calls in flight, exec mode 0."""
    import torch
    import rmcl_b200
    osc, sensors, Tom = _near_origin_case(po, synth)
    sensors = sensors[:2]
    hs, _ = _handles(sensors)
    Tbo = _tbo(sensors)
    w = [sd["weight"] for sd in sensors]
    # iterations = 0: find only, Tom kept, progress 0
    T, cp, st = rmcl_b200.micp_correct(hs, Tbo, Tom, n_corrections=3, iterations=0, convergence_progress=0.4, merge_weights=w)
    assert T.tobytes() == Tom.tobytes() and cp == 0.0 and (st["convergence_progress"] == 0).all() and (st["Cmerged_o"]["n_meas"] == 0).all()
    assert all(s["Tom_new"].tobytes() == Tom.tobytes() for s in st) and quat_close(st[0]["T_onew_oold"]["R"], [0, 0, 0, 1], 0)
    # an empty closest-point sensor next to the others changes no bit; all sensors empty keeps Tom
    he = rmcl_b200.CPCB200(gpu_map("cube29"))
    he.setTsb(sensors[0]["Tsb"]); he.setParams(1.0, 0.15)
    he.setDataset(np.zeros((0, 3), np.float32), np.zeros(0, np.uint8))
    a = rmcl_b200.micp_correct(hs, Tbo, Tom, n_corrections=3, merge_weights=w)
    b = rmcl_b200.micp_correct([hs[0], he, hs[1]], np.stack([Tbo[0], Tbo[0], Tbo[1]]), Tom, n_corrections=3, merge_weights=[w[0], 1.0, w[1]])
    assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1] and a[2]["Cmerged_o"].tobytes() == b[2]["Cmerged_o"].tobytes()
    T, cp, st = rmcl_b200.micp_correct([he], Tbo[:1], Tom, n_corrections=2, convergence_progress=0.3)
    assert T.tobytes() == Tom.tobytes() and cp == 0.0 and (st["valid_measurements"] == 0).all() and (st["total_measurements"] == 0).all()
    # steps_out = NULL: same state as with records
    lib = rmcl_b200.load_library()
    harr = (C.c_void_p * 2)(*[h._h for h in hs])
    Tb, wa = np.ascontiguousarray(Tbo), np.ascontiguousarray(w, np.float64)
    T2, cp2 = np.array(Tom, copy=True), C.c_double(0.0)
    assert lib.b2_micp_correct(harr, C.c_void_p(Tb.ctypes.data), C.c_void_p(wa.ctypes.data), C.c_uint32(2), C.c_void_p(T2.ctypes.data), C.byref(cp2),
                               C.c_int(1), C.c_uint32(3), C.c_uint32(5), None) == 0
    assert T2.tobytes() == a[0].tobytes() and cp2.value == a[1]
    # refused while a call is in flight on the lead handle: outputs untouched, no pending CUDA error
    hs[0].correctOnceAsync(Tom, Tbo[0], 5, 0.0)
    T3, cp3 = np.array(Tom, copy=True), C.c_double(0.125)
    st3 = np.zeros(3, rmcl_b200.MICP_STEP_DTYPE)
    st3["convergence_progress"] = 7.0
    rc = lib.b2_micp_correct(harr, C.c_void_p(Tb.ctypes.data), C.c_void_p(wa.ctypes.data), C.c_uint32(2), C.c_void_p(T3.ctypes.data), C.byref(cp3),
                             C.c_int(1), C.c_uint32(3), C.c_uint32(5), C.c_void_p(st3.ctypes.data))
    assert rc == -1 and T3.tobytes() == Tom.tobytes() and cp3.value == 0.125 and (st3["convergence_progress"] == 7.0).all()
    assert lib.b2_peek_cuda_error().decode() == ""
    hs[0].correctOnceWait()
    # exec mode 0 on the lead handle runs the mode-1 chain
    res = {}
    for mode in (1, 0):
        hs[0].setExecMode(mode)
        res[mode] = rmcl_b200.micp_correct(hs, Tbo, Tom, n_corrections=3, merge_weights=w)
    assert res[0][0].tobytes() == res[1][0].tobytes() and res[0][2].tobytes() == res[1][2].tobytes()
    hs[0].setExecMode(2)
    torch.cuda.synchronize()


def test_chain_exchange_fallback(po, synth):
    """The 10 000 km cube of test_exchange_range_fallback: the first step's fixed-point exchange gives up, the later steps leave at once, and the
    library re-runs the chain cooperatively from the first step without a record.  One re-run is counted; the result equals the same chain in
    exec mode 1."""
    import rmcl_b200
    from oracle import pyoracle
    V, F = synth.cube(29)
    V = (V * np.float32(5e5)).astype(np.float32)
    osc, gm = pyoracle.Scene(V, F), rmcl_b200.Map(V, F, device=0)
    m = synth.SphericalModel(np.radians(-60.0), np.radians(120.0) / 31, 32, -np.pi, 2 * np.pi / 64, 64, 1.0, 1e8)
    o, d = po.model_rays(m)
    Tsb = synth.make_transform((0, 0, 0), (0, 0, 0))
    Tgt = synth.make_transform((1e3, -2e3, 5e2), (0, 0, 0.2))
    ranges = osc.simulate(Tgt, Tsb, o, d, m.range_max)["ranges"]
    Tbo = np.stack([synth.make_transform()])
    Tom = synth.compose(Tgt, synth.make_transform((30.0, -20.0, 10.0), (0, 0, 1e-5)))
    h = rmcl_b200.RCCB200Spherical(gm)
    h.setTsb(Tsb); h.setModel(m); h.setParams(200.0, 200.0); h.setRanges(ranges)
    lib, cnt = rmcl_b200.load_library(), C.c_ulonglong(0)
    out2 = rmcl_b200.micp_correct([h], Tbo, Tom, n_corrections=3)
    lib.b2_rcc_debug_reruns(h._h, C.byref(cnt))
    assert cnt.value == 1
    h.setExecMode(1)
    out1 = rmcl_b200.micp_correct([h], Tbo, Tom, n_corrections=3)
    lib.b2_rcc_debug_reruns(h._h, C.byref(cnt))
    assert cnt.value == 1
    assert out1[0].tobytes() == out2[0].tobytes() and out1[2].tobytes() == out2[2].tobytes() and out2[2]["Cmerged_o"]["n_meas"].min() > 1500
    h.setExecMode(2)
    out3 = rmcl_b200.micp_correct([h], Tbo, Tom, n_corrections=3)            # the handle is consistent afterwards
    lib.b2_rcc_debug_reruns(h._h, C.byref(cnt))
    assert cnt.value == 2 and out3[0].tobytes() == out2[0].tobytes()
