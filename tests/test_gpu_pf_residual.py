"""GPU tests of residual resampling (b2_pf_resample_residual: k_pf_residual_stats, k_pf_residual_counts, the scan, k_pf_residual_find and
k_pf_residual_expand) against the C restatement of tests/pf_residual_ref, fed the device's weight_sum and weight_max.  Every stamp is its
particle's index, so the parentage of each slot can be read off the output.

Tolerances (as test_gladiator_resample_gpu).  The draws, the counts and everything copied from the parent are exact.  The normals go through
device logf / sinf / cosf and are within 4e-6 of the host's; slot k's translation moves by at most 4e-6 times its noise scale
s = min_noise / (L / L_max), plus the rounding of |t| (8e-6 at |t| <= 64).  R goes through device atan2f / asinf / sinf / cosf (2e-6, as for
Gladiator) and the angle noise.  n_meas is a truncated product next to an ulp of pow(): +-1, with more than 99.9 % exact."""
import ctypes as C

import numpy as np
import pytest

import pf_residual_ref as ref
from conftest import gpu_map
from test_pf_residual import CFG, FAMILIES, particles

pytestmark = pytest.mark.gpu
EPS = float(np.finfo(np.float32).eps)
_up = None


def _updater():
    global _up
    if _up is None:
        import rmcl_b200
        _up = rmcl_b200.PCDSensorUpdaterB200(gpu_map("cube29"))
    return _up


def _case(n, family, seed):
    P, A = particles(n, family, seed=seed)
    A["likelihood"]["n_meas"] %= 1000
    return P, A


def _dev(P, A):
    import torch
    return (torch.from_numpy(P.view(np.float32).reshape(-1, 8).copy()).cuda(), torch.from_numpy(A.view(np.float32).reshape(-1, 9).copy()).cuda())


def _out(n, fill=-7.0):
    import torch
    return torch.full((n, 8), fill, dtype=torch.float32, device="cuda"), torch.full((n, 9), fill, dtype=torch.float32, device="cuda")


def _np(Pt, At):
    import torch
    from rmcl_b200 import synth
    torch.cuda.synchronize()
    return Pt.cpu().numpy().view(synth.TRANSFORM_DTYPE).reshape(-1), At.cpu().numpy().view(synth.PARTICLE_ATTR_DTYPE).reshape(-1)


def _check(gP, gA, rP, rA, A, L_max, cfg=CFG):
    assert np.array_equal(gP["stamp"], rP["stamp"])
    for f in ("mean", "sigma"):
        assert np.array_equal(gA["likelihood"][f], rA["likelihood"][f])
    assert np.array_equal(gA["state_sigma"], rA["state_sigma"])
    if len(gP) == 0:
        return
    s = L_max / A["likelihood"]["mean"][rP["stamp"]].astype(np.float64)           # 1 / L_max_normed of each slot's parent
    st = s * max(cfg.min_noise_tx, cfg.min_noise_ty, cfg.min_noise_tz)
    sr = s * max(cfg.min_noise_roll, cfg.min_noise_pitch, cfg.min_noise_yaw)
    dt = np.abs(gP["t"].astype(np.float64) - rP["t"]).max(1)
    assert np.all(dt <= 8e-6 + 4e-6 * st + 4 * EPS * np.abs(rP["t"]).max(1)), float((dt - 4e-6 * st).max())
    dR = np.abs(gP["R"].astype(np.float64) - rP["R"]).max(1)
    assert np.all(dR <= 2e-6 + 4e-6 * sr), float(dR.max())
    dn = np.abs(gA["likelihood"]["n_meas"].astype(np.int64) - rA["likelihood"]["n_meas"].astype(np.int64))
    assert dn.max() <= 1 and (dn != 0).sum() <= max(1, len(dn) // 1000)


def _run(up, P, A, M, seed=77, step=3, cfg=CFG, first=0, n_local=None, fill=-7.0):
    Pd, Ad = _dev(P, A)
    n_local = M - first if n_local is None else n_local
    Pn, An = _out(n_local, fill)
    r = up.resampleResidual(Pd, Ad, Pn, An, cfg, seed=seed, step=step, first=first, n_new=M)
    gP, gA = _np(Pn, An)
    return r, gP, gA


def _compare(n, M, family, seed=1):
    P, A = _case(n, family, seed)
    r, gP, gA = _run(_updater(), P, A, M)
    S = float(r["weight_sum"])
    seq = 0.0
    for v in A["likelihood"]["mean"].astype(np.float64):
        seq += v
    assert abs(S - seq) <= 2 * n * 2.0 ** -53 * S
    assert float(r["weight_max"]) == max(0.0, float(A["likelihood"]["mean"].max()))
    want = ref.resample(P, A, M, CFG, 77, 3, S=S, L_max=float(r["weight_max"]))
    assert int(r["n_particles"]) == want["n_particles"] and int(r["draws"]) == want["draws"]
    k = want["n_particles"]
    _check(gP[:k], gA[:k], want["P"][:k], want["A"][:k], A, float(r["weight_max"]))
    assert np.all(gP[k:].view(np.float32) == -7.0) and np.all(gA[k:].view(np.float32) == -7.0)
    return r


def _sizes(n):
    return sorted({m for m in (1, n - 1, n, n + 1, 2 * n + 1, 20 * n) if m >= 1})


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("n,M", [(n, M) for n in (1, 31, 32, 33, 255, 256, 257, 4097, 50000) for M in _sizes(n)] + [(50000, 1000000)])
def test_device_matches_restatement(n, M, family):
    _compare(n, M, family)


def test_three_chunks_and_the_draw_bound():
    """one particle holds 1/5 of the weight among 30 000 (every other count is 0): about 5 hits of p = 1/30 000 fill the set, over several
    chunks of 60 000 draws.  With 1/30 of the weight the 480 000 draws of D_max run out first."""
    n = 30000
    for share, seed in ((5, 3), (30, 3)):
        P, A = _case(n, 0.0, seed)
        A["likelihood"]["mean"] = np.float32((share - 1) / (n - 1))
        A["likelihood"]["mean"][1234] = 1.0
        r = _compare_arrays(P, A, n)
        if share == 5:
            assert int(r["n_particles"]) == n and ref.chunks(n, n, int(r["draws"])) >= 3, (int(r["draws"]), ref.chunks(n, n, int(r["draws"])))
        else:
            assert int(r["draws"]) == ref.d_max(n, n) and 0 < int(r["n_particles"]) < n and ref.chunks(n, n, int(r["draws"])) == 8


def _compare_arrays(P, A, M):
    r, gP, gA = _run(_updater(), P, A, M)
    want = ref.resample(P, A, M, CFG, 77, 3, S=float(r["weight_sum"]), L_max=float(r["weight_max"]))
    assert int(r["n_particles"]) == want["n_particles"] and int(r["draws"]) == want["draws"]
    k = want["n_particles"]
    _check(gP[:k], gA[:k], want["P"][:k], want["A"][:k], A, float(r["weight_max"]))
    assert np.all(gP[k:].view(np.float32) == -7.0)
    return r


def test_equal_weights_below_one_copy_fill_nothing():
    r = _compare(5000, 4999, 0.5)
    assert int(r["draws"]) == ref.d_max(5000, 4999) and int(r["n_particles"]) == 0


@pytest.mark.parametrize("bad", [0.0, -1e-3, float("nan"), float("inf")])
def test_invalid_weights_fill_nothing(bad):
    P, A = _case(1000, "uniform", 2)
    if bad == 0.0:
        A["likelihood"]["mean"] = 0.0
    else:
        A["likelihood"]["mean"][500] = bad
    r, gP, gA = _run(_updater(), P, A, 1000)
    assert int(r["n_particles"]) == 0 and int(r["draws"]) == 0
    assert np.all(gP.view(np.float32) == -7.0) and np.all(gA.view(np.float32) == -7.0)


@pytest.mark.parametrize("ranks", [1, 2, 3, 7])
@pytest.mark.parametrize("n,M,family", [(4097, 20000, "lognormal"), (30000, 30000, 0.0)])
def test_slices_concatenate_to_the_whole(ranks, n, M, family):
    P, A = _case(n, family, 4)
    if family == 0.0:                                 # the draw bound ends the loop with part of the set filled
        A["likelihood"]["mean"] = np.float32(29 / (n - 1))
        A["likelihood"]["mean"][77] = 1.0
    up = _updater()
    whole, wP, wA = _run(up, P, A, M, fill=-3.0)
    assert 0 < int(whole["n_particles"]) <= M
    cuts = np.linspace(0, M, ranks + 1).astype(int)
    parts = [_run(up, P, A, M, first=int(a), n_local=int(b - a), fill=-3.0) for a, b in zip(cuts[:-1], cuts[1:])]
    for r, _, _ in parts:
        assert r.tobytes() == whole.tobytes()
    assert b"".join(p[1].tobytes() for p in parts) == wP.tobytes()
    assert b"".join(p[2].tobytes() for p in parts) == wA.tobytes()
    k = int(whole["n_particles"])
    assert np.all(wP[k:].view(np.float32) == -3.0) and np.all(wA[k:].view(np.float32) == -3.0)


@pytest.mark.parametrize("n", [1, 255, 257, 4097, 50000, 300001])
def test_weight_sum_is_the_estimate_sum(n):
    P, A = _case(n, "lognormal", 6)
    up = _updater()
    Pd, Ad = _dev(P, A)
    Pn, An = _out(1)
    r = up.resampleResidual(Pd, Ad, Pn, An, CFG, n_new=1)
    est = up.estimateStats(Pd, Ad, max_induction_particles=n)
    assert float(r["weight_sum"]) / n == float(est["likelihood"]["mean"])
    assert float(r["weight_max"]) == float(est["likelihood"]["max"])


def test_reproducible():
    P, A = _case(4097, "half_zero", 8)
    up = _updater()
    a = _run(up, P, A, 50000, seed=5, step=9)
    b = _run(up, P, A, 50000, seed=5, step=9)
    c = _run(up, P, A, 50000, seed=5, step=10)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    assert a[1].tobytes() != c[1].tobytes()


def test_refusals_leave_outputs_untouched():
    import rmcl_b200
    from rmcl_b200.api import _devptr
    from rmcl_b200.synth import RESIDUAL_RESULT_DTYPE
    up = _updater()
    lib = rmcl_b200.load_library()
    P, A = _case(300, "uniform", 1)
    Pd, Ad = _dev(P, A)
    Pn, An = _out(600)
    P0, A0 = _np(Pn, An)
    out = np.zeros((), RESIDUAL_RESULT_DTYPE)
    cfg = rmcl_b200.GladiatorConfig.defaults()
    chk = rmcl_b200.api._chk

    def call(h=True, p=Pd, a=Ad, n=300, n_new=600, first=0, n_local=600, pn=Pn, an=An, c=True, o=True, off_p=0, off_a=0):
        ptr = lambda t, off: None if t is None else C.c_void_p(_devptr(t).value + off)
        return chk(lib.b2_pf_resample_residual(up._h if h else None, ptr(p, 0), ptr(a, 0), C.c_uint32(n), C.c_uint32(n_new), C.c_uint32(first), C.c_uint32(n_local),
                                               ptr(pn, off_p), ptr(an, off_a), C.byref(cfg) if c else None, C.c_uint64(1), C.c_uint32(0),
                                               C.c_void_p(out.ctypes.data) if o else None))

    def refused(what, **kw):
        before = rmcl_b200.kernel_launch_count()
        with pytest.raises(rmcl_b200.B2Error) as e:
            call(**kw)
        assert e.value.code == -1 and what in str(e.value), str(e.value)
        assert rmcl_b200.kernel_launch_count() == before
        gP, gA = _np(Pn, An)
        assert gP.tobytes() == P0.tobytes() and gA.tobytes() == A0.tobytes()
        assert lib.b2_peek_cuda_error().decode() == ""

    refused("'h'", h=False)
    refused("poses_dev", p=None)
    refused("attrs_dev", a=None)
    refused("poses_new_dev", pn=None)
    refused("attrs_new_dev", an=None)
    refused("cfg", c=False)
    refused("out_host", o=False)
    refused("both must be > 0", n=0)
    refused("both must be > 0", n_new=0)
    refused("exceed", first=1, n_local=600)
    refused("exceed", first=601, n_local=0)
    refused("overlaps", p=Pn, n=300, pn=Pn, off_p=32 * 299, n_local=1, first=0)         # output inside the input poses
    refused("overlaps", an=Ad, off_a=36 * 299, n_local=1)                               # output attrs on the last input attrs
    refused("overlaps", pn=An, off_p=0, n_local=1)                                      # poses_new on attrs_new
    refused("overlaps", an=Pd, n_local=2)                                               # attrs_new on the input poses


def test_whole_cycle_on_the_device():
    """initialise 50 000 particles, sensor update, residual resampling into the node's 1 000 000-slot buffer, then motion and sensor update
    of the grown set: nothing leaves the device, and the estimate of the grown set is finite"""
    import torch
    import rmcl_b200
    from rmcl_b200 import synth
    gmap = gpu_map("building:200000")
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gmap)
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(m); h.find(Tgt)
    beams = synth.pf_beams(h.modelView()["points"], 180)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    gx, gy, gz = (float(v) for v in Tgt["t"])
    n, n_max = 50_000, 1_000_000
    P = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    A = torch.empty((n, 9), dtype=torch.float32, device="cuda")
    up.initSamplesUniform(P, A, [gx - 3.0, gy - 3.0, gz, 0.0, 0.0, -np.pi], [gx + 3.0, gy + 3.0, gz, 0.0, 0.0, np.pi], 7)
    prm = rmcl_b200.PFParams.defaults()
    up.update(P, A, Tsb, beams, prm)
    Pn = torch.empty((n_max, 8), dtype=torch.float32, device="cuda")
    An = torch.empty((n_max, 9), dtype=torch.float32, device="cuda")
    r = up.resampleResidual(P, A, Pn, An, rmcl_b200.GladiatorConfig.defaults(), seed=7, step=0)
    k = int(r["n_particles"])
    assert k >= 10 and float(r["weight_sum"]) > 0.0
    P2, A2 = Pn[:k], An[:k]
    up.motionUpdate(P2, A2, synth.make_transform((0.05, 0.0, 0.0), (0.0, 0.0, 0.01)), 0.02)
    up.update(P2, A2, Tsb, beams, prm)
    est = up.estimateStats(P2, A2, max_induction_particles=k)
    assert np.all(np.isfinite(est["position"])) and np.all(np.isfinite(est["orientation"])) and np.all(np.isfinite(est["covariance"]))
    L = A2[:, 0].cpu().numpy()
    assert np.all(np.isfinite(L)) and L.max() > 0.0
    print(f"residual: 50 000 -> {k} particles in {int(r['draws'])} draws")
