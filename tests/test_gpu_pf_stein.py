"""GPU tests of the Stein variational step (b2_pf_stein_update, PCDSensorUpdaterB200.steinUpdate) against the product's functions compiled
for the host (tests/pf_stein_ref.py, pf_stein_ref/stein_emul.cu).  The host functions' relation to the float64 definition is pinned by
tests/test_pf_stein.py.

Tolerances.
  * device vs host-compiled product: exact (poses and the result record, bytes), after 1 and after 10 iterations.  The host runs every
    pair of the move, so the 10^6-particle case and n_ref 0 at 10^5 particles are compared after one iteration.
  * convergence (building:1000000, dist_sigma 0.2 m, 10 000 particles from N(true pose, 0.3 m, 10 deg), 30 iterations, no resampling):
    the mean translation and yaw errors fall to at most a third, the RMS spread to at most half; no particle crosses a wall.
  * control: without beams the spread does not shrink (at least 0.99 of its start)."""
import ctypes as C
import math

import numpy as np
import pytest

import dfield_ref as DR
import pf_stein_ref as S
from conftest import gpu_map, mesh

pytestmark = pytest.mark.gpu

_FIELDS = {}


def _setup(name):
    """(map, device field, grid, index, bricks, host walls) for name with h 0.05, trunc 1"""
    import rmcl_b200
    if name not in _FIELDS:
        gmap = gpu_map(name)
        f = rmcl_b200.DistanceField(gmap, 0.05, 1.0)
        V, F = mesh(name)
        lo, hi = DR.default_box(V, 1.0)
        g = DR.Grid(lo, hi, 0.05, 1.0)
        index, bricks = f.download()
        _FIELDS[name] = (gmap, f, g, index, bricks, S.Scene(V, F))
    return _FIELDS[name]


def _beams(k, seed=3):
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    B = np.zeros(k, synth.RANGE_MEAS_DTYPE)
    a = rng.uniform(-np.pi, np.pi, k)
    el = rng.uniform(-0.3, 0.3, k)
    B["dir"] = np.stack([np.cos(a) * np.cos(el), np.sin(a) * np.cos(el), np.sin(el)], 1).astype(np.float32)
    B["range"] = rng.uniform(0.5, 8.0, k).astype(np.float32)
    B["orig"] = [0.05, 0.0, 0.2]
    return B


def _poses(name, n, seed=5):
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    T0 = synth.indoor_gt_pose() if name.startswith("indoor") else synth.building_gt_pose()
    P = synth.transforms(n)
    P["t"] = np.asarray(T0["t"], np.float32) + (rng.normal(0, 0.5, (n, 3)) * [1, 1, 0.05]).astype(np.float32)
    yaw = 2 * math.atan2(float(T0["R"][2]), float(T0["R"][3])) + rng.normal(0, 0.3, n)
    yaw[: min(n, 2)] = [np.pi, -np.pi][: min(n, 2)]
    P["R"][:, 2] = np.sin(yaw / 2)
    P["R"][:, 3] = np.cos(yaw / 2)
    P["stamp"] = np.arange(n)
    if n >= 33:
        P[10:14] = P[9]
        P["t"][20, 0] = np.nan
        P["R"][21, 2] = np.inf
    return P


def _tensor(P):
    import torch
    return torch.from_numpy(np.ascontiguousarray(P).view(np.float32).reshape(-1, 8).copy()).cuda()


def _host(Pd):
    from rmcl_b200 import synth
    return Pd.cpu().numpy().reshape(-1).view(synth.TRANSFORM_DTYPE)


def _cfg(iterations, n_ref):
    import rmcl_b200
    c = rmcl_b200.SteinConfig.defaults()
    c.iterations, c.n_ref = iterations, n_ref
    return c


@pytest.mark.parametrize("name,n,n_ref,n_beams,iters", [
    ("indoor:500000", 1, 0, 180, 10), ("indoor:500000", 33, 0, 1, 10), ("indoor:500000", 33, 4096, 0, 10), ("indoor:500000", 4097, 0, 180, 10),
    ("indoor:500000", 4097, 4096, 1000, 10), ("indoor:500000", 100_000, 4096, 180, 10), ("indoor:500000", 100_000, 0, 180, 1),
    ("building:1000000", 1, 4096, 1000, 10), ("building:1000000", 33, 4096, 180, 10), ("building:1000000", 4097, 0, 0, 10),
    ("building:1000000", 4097, 4096, 180, 1), ("building:1000000", 100_000, 4096, 1000, 1), ("building:1000000", 1_000_000, 4096, 180, 1)])
def test_device_equals_the_host_compiled_product(name, n, n_ref, n_beams, iters):
    import rmcl_b200
    from rmcl_b200 import synth
    gmap, f, g, index, bricks, scene = _setup(name)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    up.setDistanceField(f)
    P, B, Tsb = _poses(name, n), _beams(n_beams), synth.scenario_tsb()
    prm = rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.2
    cfg = _cfg(iters, n_ref)
    Pd = _tensor(P)
    res = up.steinUpdate(Pd, Tsb, B, cfg, prm, seed=1234, step=7)
    want, rec = scene.update(g, index, bricks, P, Tsb, B, 0.2, cfg, 1234, 7)
    got = _host(Pd)
    diff = np.flatnonzero(got.view(np.uint32).reshape(n, 8) != want.view(np.uint32).reshape(n, 8))
    assert got.tobytes() == want.tobytes(), f"{len(diff)} words differ, first particles {np.unique(diff // 8)[:5]}"
    assert np.array(res["bandwidth"], np.float32).tobytes() == np.array(rec.bandwidth, np.float32).tobytes()
    assert (res["n_ref"], res["n_blocked"]) == (rec.n_ref, rec.n_blocked)
    assert np.float32(res["rms_step_t"]) == np.float32(rec.rms_step_t) and np.float32(res["rms_step_r"]) == np.float32(rec.rms_step_r)
    moved = (got["t"][:, :2] != P["t"][:, :2]).any(1).sum()
    print(f"{name} n {n} n_ref {n_ref} beams {n_beams} x{iters}: moved {moved}, blocked {rec.n_blocked}, h {np.round(rec.bandwidth[:], 4)}, "
          f"rms {rec.rms_step_t:.4f} m {rec.rms_step_r:.4f} rad")


def _c3():
    import rmcl_b200
    from rmcl_b200 import synth
    gmap, f, *_ = _setup("building:1000000")
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gmap)
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(m); h.find(Tgt)
    return gmap, f, Tsb, Tgt, synth.pf_beams(h.modelView()["points"], 180)


def _spread_set(Tgt, n=10_000, seed=21):
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    P = synth.transforms(n)
    P["t"] = np.asarray(Tgt["t"], np.float32)
    P["t"][:, :2] += rng.normal(0, 0.3, (n, 2)).astype(np.float32)
    yaw = 2 * math.atan2(float(Tgt["R"][2]), float(Tgt["R"][3])) + rng.normal(0, math.radians(10.0), n)
    P["R"][:, 2], P["R"][:, 3] = np.sin(yaw / 2), np.cos(yaw / 2)
    return P


def _errors(P, Tgt):
    c = S.chart64(P)
    yaw_gt = 2 * math.atan2(float(Tgt["R"][2]), float(Tgt["R"][3]))
    et = np.hypot(c[:, 0] - float(Tgt["t"][0]), c[:, 1] - float(Tgt["t"][1])).mean()
    ey = np.abs(S.wrap64(c[:, 2] - yaw_gt)).mean()
    spread = np.sqrt(((c[:, :2] - c[:, :2].mean(0)) ** 2).sum(1).mean())
    return et, ey, spread


def test_convergence_toward_the_true_pose_without_crossing_walls():
    import rmcl_b200
    gmap, f, Tsb, Tgt, beams = _c3()
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    up.setDistanceField(f)
    prm = rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.2
    P0 = _spread_set(Tgt)
    Pd = _tensor(P0)
    e0 = _errors(P0, Tgt)
    res = up.steinUpdate(Pd, Tsb, beams, _cfg(30, 4096), prm, seed=5)
    P1 = _host(Pd)
    e1 = _errors(P1, Tgt)
    print(f"start: {e0[0]:.3f} m, {math.degrees(e0[1]):.2f} deg, spread {e0[2]:.3f} m; after 30: {e1[0]:.3f} m, {math.degrees(e1[1]):.2f} deg, "
          f"spread {e1[2]:.3f} m; blocked {res['n_blocked']}, h {np.round(res['bandwidth'], 4)}")
    assert e1[0] <= e0[0] / 3 and e1[1] <= e0[1] / 3 and e1[2] <= e0[2] / 2
    # no particle on the other side of a wall from its start
    a, b = P0["t"].astype(np.float32), P1["t"].astype(np.float32)
    d = b - a
    L = np.linalg.norm(d.astype(np.float64), axis=1)
    k = L > 1e-4
    t, face, _, _ = gmap.intersect(a[k], (d[k] / L[k, None]).astype(np.float32))
    assert not (t < L[k] - 1e-4).any()


def test_without_beams_the_spread_does_not_shrink():
    import rmcl_b200
    gmap, f, Tsb, Tgt, beams = _c3()
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    up.setDistanceField(f)
    P0 = _spread_set(Tgt)
    Pd = _tensor(P0)
    up.steinUpdate(Pd, Tsb, beams[:0], _cfg(30, 4096), None, seed=5)
    e0, e1 = _errors(P0, Tgt), _errors(_host(Pd), Tgt)
    print(f"no beams: spread {e0[2]:.3f} -> {e1[2]:.3f} m")
    assert e1[2] >= 0.99 * e0[2]


def test_two_handles_on_two_streams_agree():
    import rmcl_b200
    import torch
    gmap, f, *_ = _setup("indoor:500000")
    from rmcl_b200 import synth
    P, B = _poses("indoor:500000", 50_000), _beams(180)
    outs = []
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    ups = [rmcl_b200.PCDSensorUpdaterB200(gmap) for _ in streams]
    Pds = [_tensor(P) for _ in streams]
    torch.cuda.synchronize()
    for up, s, Pd in zip(ups, streams, Pds):
        up.setDistanceField(f)
        up.setStream(s.cuda_stream)
        outs.append(up.steinUpdate(Pd, synth.scenario_tsb(), B, _cfg(5, 4096), None, seed=3))
    torch.cuda.synchronize()
    assert _host(Pds[0]).tobytes() == _host(Pds[1]).tobytes() and outs[0] == outs[1]


def test_refusals_and_no_ops():
    import rmcl_b200
    from rmcl_b200 import synth
    gmap, f, *_ = _setup("indoor:500000")
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    P, B, Tsb = _poses("indoor:500000", 100), _beams(10), synth.scenario_tsb()
    Pd = _tensor(P)
    with pytest.raises(rmcl_b200.B2Error):
        up.steinUpdate(Pd, Tsb, B)                        # no field
    up.setDistanceField(f)
    bad = []
    for field, v in [("step_t", 0.0), ("step_r", -1.0), ("min_bandwidth_t", float("nan")), ("min_bandwidth_r", float("inf")), ("w_rand", 1.0),
                     ("w_rand", -0.1)]:
        c = rmcl_b200.SteinConfig.defaults()
        setattr(c, field, v)
        bad.append((c, None))
    p0 = rmcl_b200.PFParams.defaults()
    p0.dist_sigma = 0.0
    bad.append((rmcl_b200.SteinConfig.defaults(), p0))
    n0 = rmcl_b200.kernel_launch_count()
    for c, p in bad:
        with pytest.raises(rmcl_b200.B2Error) as e:
            up.steinUpdate(Pd, Tsb, B, c, p)
        assert e.value.code == -1
    assert rmcl_b200.kernel_launch_count() == n0 and _host(Pd).tobytes() == P.tobytes()
    lib = rmcl_b200.load_library()
    prm, cfg = rmcl_b200.PFParams.defaults(), rmcl_b200.SteinConfig.defaults()
    T = np.ascontiguousarray(Tsb)
    args = lambda h, fh, poses, n, beams, nb, c: (h, fh, poses, C.c_uint32(n), C.c_void_p(T.ctypes.data), beams, C.c_uint32(nb), C.byref(prm), c,
                                                 C.c_uint64(1), C.c_uint32(0), None)
    assert lib.b2_pf_stein_update(*args(up._h, None, C.c_void_p(Pd.data_ptr()), 100, None, 0, C.byref(cfg))) == -1
    assert lib.b2_pf_stein_update(*args(up._h, f._h, None, 100, None, 0, C.byref(cfg))) == -1
    assert lib.b2_pf_stein_update(*args(up._h, f._h, C.c_void_p(Pd.data_ptr()), 100, None, 5, C.byref(cfg))) == -1
    assert lib.b2_pf_stein_update(*args(up._h, f._h, C.c_void_p(Pd.data_ptr()), 100, None, 0, None)) == -1
    # n == 0 and iterations == 0: B2_OK, nothing launched, a zeroed record
    assert up.steinUpdate(Pd[:0], Tsb, B)["n_ref"] == 0
    assert up.steinUpdate(Pd, Tsb, B, _cfg(0, 4096)) == {"bandwidth": (0.0, 0.0, 0.0), "n_ref": 0, "n_blocked": 0, "rms_step_t": 0.0, "rms_step_r": 0.0}
    assert rmcl_b200.kernel_launch_count() == n0 and _host(Pd).tobytes() == P.tobytes()
    # with 0 beams: the steps are the repulsion only; the record is filled
    r = up.steinUpdate(Pd, Tsb, B[:0], _cfg(1, 0))
    assert r["n_ref"] == 100 and r["rms_step_t"] > 0
