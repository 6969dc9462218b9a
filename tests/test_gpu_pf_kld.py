"""GPU tests of KLD-sampling (b2_pf_resample_kld: k_pf_residual_stats, k_pf_kld_weights and the weight scan, then per chunk k_pf_kld_draw,
k_pf_kld_flags, the flag scan, k_pf_kld_stop and k_pf_kld_expand) against the C restatement of tests/pf_kld_ref, fed the device's
weight_sum and weight_max.  Every stamp is its particle's index, so the parentage of each slot can be read off the output.

n_particles, bins, the parents and everything copied from the parent are exact; t, R and n_meas are within the tolerances of
test_gpu_pf_residual (the copy is residual's, whose normals go through device logf / sinf / cosf)."""
import math
import os
import subprocess

import numpy as np
import pytest

import pf_kld_ref as ref
from conftest import gpu_map
from test_gpu_pf_residual import _check, _dev, _np, _out
from test_pf_residual import CFG, particles

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_MIN = 100
_up = None


def _updater():
    global _up
    if _up is None:
        import rmcl_b200
        _up = rmcl_b200.PCDSensorUpdaterB200(gpu_map("cube29"))
    return _up


def _kld(**kw):
    import rmcl_b200
    c = rmcl_b200.KLDConfig.defaults()
    c.n_min = N_MIN
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _case(n, seed, spread=20.0, family="lognormal"):
    """n particles with |t| <= spread (z within 1 m), all headings, likelihoods of `family`, n_meas < 1000"""
    P, A = particles(n, family, seed=seed)
    P["t"][:, :2] *= np.float32(spread / 20.0)
    P["t"][:, 2] *= np.float32(1.0 / 20.0)
    A["likelihood"]["n_meas"] %= 1000
    return P, A


def _run(up, P, A, n_max, kld, seed=77, step=3, first=0, n_local=None, fill=-7.0, dev=None):
    Pd, Ad = dev if dev is not None else _dev(P, A)
    n_local = n_max - first if n_local is None else n_local
    Pn, An = _out(n_local, fill)
    r = up.resampleKLD(Pd, Ad, Pn, An, kld, CFG, seed=seed, step=step, first=first, n_max=n_max)
    gP, gA = _np(Pn, An)
    return r, gP, gA


def _compare(P, A, n_max, kld, up=None):
    up = up or _updater()
    Pd, Ad = _dev(P, A)
    r, gP, gA = _run(up, P, A, n_max, kld, dev=(Pd, Ad))
    Pr, Ar = _out(1)
    rr = up.resampleResidual(Pd, Ad, Pr, Ar, CFG, n_new=1)
    assert float(r["weight_sum"]) == float(rr["weight_sum"]) and float(r["weight_max"]) == float(rr["weight_max"])   # the shared statistics
    assert float(r["weight_max"]) == max(0.0, float(A["likelihood"]["mean"].max()))
    want = ref.resample(P, A, n_max, kld, CFG, 77, 3, S=float(r["weight_sum"]), L_max=float(r["weight_max"]))
    assert (int(r["n_particles"]), int(r["bins"])) == (want["n_particles"], want["bins"])
    k = want["n_particles"]
    assert np.array_equal(gP["stamp"][:k], want["parents"])
    _check(gP[:k], gA[:k], want["P"][:k], want["A"][:k], A, float(r["weight_max"]))
    assert np.all(gP[k:].view(np.float32) == -7.0) and np.all(gA[k:].view(np.float32) == -7.0)
    return r


@pytest.mark.parametrize("n_max", [N_MIN, 2 ** 16 - 1, 2 ** 16 + 1, 1_000_000])
@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 1000, 65537, 1_000_000])
def test_device_matches_restatement(n, n_max):
    P, A = _case(n, n)
    r = _compare(P, A, n_max, _kld())
    if n >= 65537 and n_max == 1_000_000:                          # a spread set: the bound outruns the draws, over five chunks
        assert int(r["n_particles"]) == n_max and ref.chunks(N_MIN, n_max, n_max) == 5


@pytest.mark.parametrize("family", ["uniform", "dominant", "half_zero"])
def test_families_and_a_stop_in_a_later_chunk(family):
    """poses within 5 m: about 14 000 bins, whose bound stops the draws in the fourth chunk (family uniform)"""
    P, A = _case(1_000_000, 5, spread=5.0, family=family)
    r = _compare(P, A, 1_000_000, _kld())
    if family == "uniform":
        assert 458_752 < int(r["n_particles"]) < 983_040, int(r["n_particles"])


def test_settings():
    P, A = _case(200_000, 8, spread=8.0)
    for kw in ({"res_z": 0.1}, {"res_yaw": math.radians(1.0)}, {"res_yaw": 2 * math.pi / 32768}, {"res_yaw": 7.0}, {"epsilon": 0.2, "z": 3.0},
               {"n_min": 70_000}, {"res_xy": 0.05}):
        _compare(P, A, 300_000, _kld(**kw))


@pytest.mark.parametrize("ranks", [1, 2, 3, 5, 7])
def test_slices_concatenate_to_the_whole(ranks):
    P, A = _case(65537, 4, spread=3.0)                             # about 5 000 bins: the bound stops the draws in the third chunk
    n_max, kld = 400_000, _kld()
    up = _updater()
    whole, wP, wA = _run(up, P, A, n_max, kld, fill=-3.0)
    k = int(whole["n_particles"])
    assert 196_608 < k < n_max, k
    cuts = np.linspace(0, n_max, ranks + 1).astype(int)
    parts = [_run(up, P, A, n_max, kld, first=int(a), n_local=int(b - a), fill=-3.0) for a, b in zip(cuts[:-1], cuts[1:])]
    for r, _, _ in parts:
        assert r.tobytes() == whole.tobytes()
    assert b"".join(p[1].tobytes() for p in parts) == wP.tobytes()
    assert b"".join(p[2].tobytes() for p in parts) == wA.tobytes()
    assert np.all(wP[k:].view(np.float32) == -3.0) and np.all(wA[k:].view(np.float32) == -3.0)


def test_repeatable_across_calls_and_handles():
    import rmcl_b200
    P, A = _case(100_000, 6, spread=6.0)
    up = _updater()
    a = _run(up, P, A, 500_000, _kld(), seed=5, step=9)
    b = _run(up, P, A, 500_000, _kld(), seed=5, step=9)
    c = _run(rmcl_b200.PCDSensorUpdaterB200(gpu_map("cube29")), P, A, 500_000, _kld(), seed=5, step=9)
    d = _run(up, P, A, 500_000, _kld(), seed=5, step=10)
    assert all(x.tobytes() == y.tobytes() == z.tobytes() for x, y, z in zip(a, b, c))
    assert a[1].tobytes() != d[1].tobytes()


@pytest.mark.parametrize("bad", [0.0, -1e-3, float("nan"), float("inf")])
def test_invalid_sets_write_nothing(bad):
    P, A = _case(1000, 2)
    if bad == 0.0:
        A["likelihood"]["mean"] = 0.0
    else:
        A["likelihood"]["mean"][500] = bad
    r, gP, gA = _run(_updater(), P, A, 5000, _kld())
    assert int(r["n_particles"]) == 0 and int(r["bins"]) == 0
    assert np.all(gP.view(np.float32) == -7.0) and np.all(gA.view(np.float32) == -7.0)


def test_refusals_leave_outputs_untouched():
    import ctypes as C
    import rmcl_b200
    from rmcl_b200.api import _devptr
    from rmcl_b200.synth import KLD_RESULT_DTYPE
    up = _updater()
    lib = rmcl_b200.load_library()
    P, A = _case(300, 1)
    Pd, Ad = _dev(P, A)
    Pn, An = _out(600)
    P0, A0 = _np(Pn, An)
    out = np.zeros((), KLD_RESULT_DTYPE)
    cfg = rmcl_b200.GladiatorConfig.defaults()
    chk = rmcl_b200.api._chk

    def call(h=True, p=Pd, a=Ad, n=300, n_max=600, first=0, n_local=600, pn=Pn, an=An, c=True, k=True, o=True, off_p=0, off_a=0, **kw):
        kc = _kld(**kw)
        ptr = lambda t, off: None if t is None else C.c_void_p(_devptr(t).value + off)
        return chk(lib.b2_pf_resample_kld(up._h if h else None, ptr(p, 0), ptr(a, 0), C.c_uint32(n), C.c_uint32(n_max), C.c_uint32(first), C.c_uint32(n_local),
                                          ptr(pn, off_p), ptr(an, off_a), C.byref(cfg) if c else None, C.byref(kc) if k else None, C.c_uint64(1), C.c_uint32(0),
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
    refused("kld", k=False)
    refused("out_host", o=False)
    refused("both must be > 0", n=0)
    refused("both must be > 0", n_max=0)
    refused("n_min", n_min=0)
    refused("n_min", n_min=601)
    refused("exceed", first=1, n_local=600)
    refused("exceed", first=601, n_local=0)
    refused("overlaps", p=Pn, pn=Pn, off_p=32 * 299, n_local=1)
    refused("overlaps", an=Ad, off_a=36 * 299, n_local=1)
    refused("overlaps", pn=An, n_local=1)
    refused("overlaps", an=Pd, n_local=2)
    for f, v in (("res_xy", 0.0), ("res_xy", -0.5), ("res_xy", float("nan")), ("res_xy", float("inf")), ("epsilon", 0.0), ("epsilon", float("inf")),
                 ("epsilon", -0.01)):
        refused("must be finite and > 0", **{f: v})
    for v in (-0.1, float("nan"), float("inf")):
        refused("res_z", res_z=v)
    for v in (float("nan"), float("inf"), -float("inf")):
        refused("z = ", z=v)
    for v in (0.0, -0.1, float("nan"), float("inf"), 2 * math.pi / 40000):
        refused("yaw sectors", res_yaw=v)
    call()                                                          # the same arguments, valid: it runs
    assert int(out["n_particles"]) >= N_MIN


def test_the_set_shrinks_as_the_filter_converges():
    """The point of the feature, end to end on building:200000: a uniform initialisation of n_max particles around the true pose, then cycles
    of sensor update -> motion (standing still) -> resampleKLD into the other n_max buffer.  The set must shrink at least 10x from the first
    resampling to the last (on an H100: 50 730 -> 1 480), and the estimate must end within 0.1 m and 2 deg of the true pose (0.032 m, 0.33 deg).
    The sensor model is sharp (dist_sigma 0.05 m), so that the likelihoods, which are the weights as they are, separate the particles: with the
    default 2 m every L / L_max stays close to 1 and the drawn set keeps its spread."""
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
    yaw = math.radians(30.0)
    n_max = 1_000_000
    bufs = [(torch.empty((n_max, 8), dtype=torch.float32, device="cuda"), torch.empty((n_max, 9), dtype=torch.float32, device="cuda")) for _ in range(2)]
    up.initSamplesUniform(*bufs[0], [gx - 2.0, gy - 2.0, gz, 0.0, 0.0, yaw - 1.0], [gx + 2.0, gy + 2.0, gz, 0.0, 0.0, yaw + 1.0], 7)
    prm, kld = rmcl_b200.PFParams.defaults(), rmcl_b200.KLDConfig.defaults()
    prm.dist_sigma = 0.05
    still = synth.make_transform((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))
    n, cur, sizes = n_max, 0, []
    for step in range(30):
        P, A = bufs[cur][0][:n], bufs[cur][1][:n]
        up.update(P, A, Tsb, beams, prm)
        up.motionUpdate(P, A, still, 0.02)
        r = up.resampleKLD(P, A, *bufs[1 - cur], kld, rmcl_b200.GladiatorConfig.defaults(), seed=11, step=step)
        n, cur = int(r["n_particles"]), 1 - cur
        assert n >= kld.n_min
        sizes.append((n, int(r["bins"])))
    P, A = bufs[cur][0][:n], bufs[cur][1][:n]
    up.update(P, A, Tsb, beams, prm)
    est = up.estimateStats(P, A, max_induction_particles=n)
    x, y, z, w = (float(v) for v in est["orientation"])
    e_yaw = math.atan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z)) - yaw
    e_yaw = abs((e_yaw + math.pi) % (2 * math.pi) - math.pi)
    e_t = math.hypot(float(est["position"][0]) - gx, float(est["position"][1]) - gy)
    print(f"kld: (n_particles, bins) per cycle {sizes}; translation error {e_t:.3f} m, yaw error {math.degrees(e_yaw):.2f} deg")
    assert sizes[0][0] >= 10 * sizes[-1][0], sizes
    assert e_t < 0.1 and e_yaw < math.radians(2.0), (e_t, math.degrees(e_yaw))


def test_cpp_classes_match_python(tmp_path):
    """tests/pf_kld_cpp/pf_kld_cpp.cpp, compiled here against include/rmcl_b200/rcc_b200.hpp, resamples device particles through
    PCDSensorUpdaterB200::resampleKLD with its kld_config: byte for byte what the Python path gives, record included"""
    import rmcl_b200
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "pf_kld_cpp")
    lib_dir = os.path.dirname(rmcl_b200.lib_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "pf_kld_cpp", "pf_kld_cpp.cpp"), "-L" + lib_dir, "-lrmcl_b200",
                           "-L" + os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + lib_dir])
    P, A = _case(20_000, 12, spread=1.5)                           # about 1 300 bins: fewer particles than slots
    n_max = 150_000
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(np.array([len(P), n_max], np.uint32).tobytes())
        f.write(P.tobytes()); f.write(A.tobytes())
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "REFUSED" in r.stdout and "n_min" in r.stdout
    Pd, Ad = _dev(P, A)
    Pn, An = _out(n_max, 0.0)
    rec = _updater().resampleKLD(Pd, Ad, Pn, An, rmcl_b200.KLDConfig.defaults(), rmcl_b200.GladiatorConfig.defaults(), seed=77, step=3)
    gP, gA = _np(Pn, An)
    assert 0 < int(rec["n_particles"]) < n_max
    assert np.fromfile(out, np.uint8).tobytes() == rec.tobytes() + gP.tobytes() + gA.tobytes()
