"""GPU tests of the particle set's pose estimate (b2_pf_estimate_stats: k_pf_estimate_moments, k_pf_estimate_cov) against the float64 model
of tests/pf_estimate_ref, with pass 2 of the model fed the device's float Tbm.

Tolerances.
  * exact: nparticles, the AABB (float min / max), the likelihood min and max, and shift -- comparisons only, no rounding.
  * likelihood mean and sigma: FP64 sums in another order.  The mean is within 1e-12 relative; sigma^2 = sum_sq / k - mean^2 within
    1e-12 (sum_sq / k + mean^2), the size of the two terms whose difference it is.
  * translation: sum L t / sum L in FP64 in another order, then rounded to float: within one float ulp of the model's float value.
  * rotation: the device and numpy solve M = sum w q q^T perturbed by FP64 reordering, |dM| <= 64 eps64 |M|; by Davis-Kahan the top
    eigenvector moves by at most |dM| / gap, plus the rounding of four components to float (4 eps32).  Where the gap is too small to say
    anything (yaw spread over the whole circle), only the maximiser property q^T M q >= lambda_max - 8 eps32 |M| is checked.
  * covariance: the model's deviation is float64 of the same float inputs; the device's is float.  With |dt| <= 16 eps32 (|t|max + |Tbm.t|)
    and |dangle| <= 8e-6 per particle (tests/test_pf_estimate.py bounds the product's deviation function so), each entry is within
    sum w (da |v_b| + |v_a| db + da db), plus FP64 reordering."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import pf_estimate_ref as er
from conftest import gpu_map
from test_pf_init import RVIZ_COV, _gauss_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS32 = float(np.finfo(np.float32).eps)
EPS64 = float(np.finfo(np.float64).eps)


def _updater(name="cube29"):
    import rmcl_b200
    return rmcl_b200.PCDSensorUpdaterB200(gpu_map(name))


def _dev(P, A):
    import torch
    return (torch.from_numpy(np.ascontiguousarray(P).view(np.float32).reshape(-1, 8).copy()).cuda(),
            torch.from_numpy(np.ascontiguousarray(A).view(np.float32).reshape(-1, 9).copy()).cuda())


def _np(P, A):
    import torch
    from rmcl_b200 import synth
    torch.cuda.synchronize()
    return P.cpu().numpy().view(synth.TRANSFORM_DTYPE).reshape(-1), A.cpu().numpy().view(synth.PARTICLE_ATTR_DTYPE).reshape(-1)


def _random_set(n, seed, yaw=0.5, spread=20.0, decades=6):
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    P = np.zeros(n, synth.TRANSFORM_DTYPE)
    ang = rng.uniform(-1, 1, (n, 3)) * [0.05, 0.05, yaw]
    P["R"] = _quats(ang)
    P["t"] = rng.normal(size=(n, 3)) * [spread, spread, 0.3] + [5.0, -3.0, 0.5]
    A = np.zeros(n, synth.PARTICLE_ATTR_DTYPE)
    A["likelihood"]["mean"] = 10.0 ** rng.uniform(-decades, 0, n)
    return P, A


def _quats(ang):
    r, p, y = (ang[:, i] / 2 for i in range(3))
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    return np.stack([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy], 1)


def _tbm(rec):
    from rmcl_b200 import synth
    T = np.zeros((), synth.TRANSFORM_DTYPE)
    T["t"], T["R"] = rec["position"], rec["orientation"]
    assert np.array_equal(T["t"].astype(np.float64), rec["position"], equal_nan=True) and np.array_equal(T["R"].astype(np.float64), rec["orientation"], equal_nan=True)
    return T


def check(rec, P, A, rotation_gap=True, covariance=True):
    """the device record against the model over the same particles -> the model's record"""
    k = len(P)
    m, _, d = er.estimate_np(P, A, Tbm_pass2=_tbm(rec))
    assert int(rec["nparticles"]) == k
    for f in ("trans_bb_min", "trans_bb_max", "shift"):
        assert np.array_equal(rec[f], m[f]), f
    assert rec["likelihood"]["min"] == m["likelihood"]["min"] and rec["likelihood"]["max"] == m["likelihood"]["max"]
    mean = float(m["likelihood"]["mean"])
    assert abs(float(rec["likelihood"]["mean"]) - mean) <= 1e-12 * abs(mean)
    assert abs(float(rec["likelihood"]["sigma"]) ** 2 - float(m["likelihood"]["sigma"]) ** 2) <= 1e-12 * (d["L_sum_sq"] / k + mean * mean)
    if not (d["L_sum"] > 0 and np.isfinite(d["L_sum"])):
        assert np.all(np.isnan(rec["position"])) and np.all(np.isnan(rec["orientation"])) and np.all(np.isnan(rec["covariance"]))
        return m
    mt = m["position"].astype(np.float32)
    assert np.all(np.abs(rec["position"] - m["position"]) <= np.spacing(np.abs(mt)).astype(np.float64)), (rec["position"], m["position"])
    M = d["M"]
    lams = np.linalg.eigvalsh(M)
    nM = float(np.abs(lams).max())
    q = rec["orientation"]
    assert abs(np.linalg.norm(q) - 1.0) <= 4 * EPS32
    assert q @ M @ q >= lams[-1] - 8 * EPS32 * nM
    assert q[3] >= 0.0
    gap = lams[-1] - lams[-2]
    if rotation_gap:
        assert gap > 1e-6 * nM
        tol = 64 * EPS64 * nM / gap + 4 * EPS32
        assert np.linalg.norm(q - np.sign(q @ d["q"]) * d["q"]) <= tol, (q, d["q"], tol)
    if covariance:
        Vd = d["V"]
        assert np.abs(Vd[:, 3:]).max() < 3.0                                      # no angle near the +-pi wrap
        dt = 16 * EPS32 * (float(np.abs(P["t"]).max()) + float(np.abs(rec["position"]).max()))
        delta = np.array([dt] * 3 + [8e-6] * 3)
        aV = np.abs(Vd)
        w = np.abs(d["w"])
        tol = np.einsum("n,ni,nj->ij", w, aV, np.broadcast_to(delta, aV.shape)) + np.einsum("n,ni,nj->ij", w, np.broadcast_to(delta, aV.shape), aV) + \
            np.outer(delta, delta) * w.sum() + 1e-12 * np.einsum("n,ni,nj->ij", w, aV, aV)
        Cd = rec["covariance"].reshape(6, 6)
        assert np.all(np.abs(Cd - m["covariance"].reshape(6, 6)) <= tol), np.abs(Cd - m["covariance"].reshape(6, 6)).max()
        assert np.array_equal(Cd, Cd.T)
    return m


@pytest.mark.parametrize("k", [1, 255, 256, 257, 50_000, 1_000_003])
def test_counts_around_the_launch_geometry(k):
    """one particle, around one block of 256, the node's default induction slice, and far beyond the 4 n_sm grid cap"""
    up = _updater()
    P, A = _random_set(k, seed=k)
    Pd, Ad = _dev(P, A)
    rec = up.estimateStats(Pd, Ad, max_induction_particles=10 ** 7)
    check(rec, P, A, rotation_gap=k > 1)
    if k == 1:
        assert np.array_equal(rec["position"], P["t"][0].astype(np.float64))
        assert np.abs(rec["orientation"] - er.canonical(P["R"][0].astype(np.float64))).max() <= EPS32


def test_induction_slice():
    """max_induction_particles below n estimates the first max_induction_particles; above n, all n"""
    up = _updater()
    P, A = _random_set(70_001, seed=3)
    Pd, Ad = _dev(P, A)
    rec = up.estimateStats(Pd, Ad)                                                  # the node's default, 50 000
    check(rec, P[:50_000], A[:50_000])
    rec = up.estimateStats(Pd, Ad, max_induction_particles=1000)
    check(rec, P[:1000], A[:1000])
    rec = up.estimateStats(Pd, Ad, max_induction_particles=10 ** 6)
    check(rec, P, A)


def test_converged_and_spread_sets_from_the_initialisers():
    """a converged set from initSamples, a spread one from initSamplesUniform with yaw in +-0.5 rad, and the whole yaw circle (maximiser only)"""
    import torch
    up = _updater()
    n = 200_003
    Pd = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    Ad = torch.empty((n, 9), dtype=torch.float32, device="cuda")
    C, pose = _gauss_case()
    up.initSamples(Pd, Ad, pose, C * 0.01, 5)
    check(up.estimateStats(Pd, Ad, 10 ** 6), *_np(Pd, Ad))
    up.initSamplesUniform(Pd, Ad, [-30, -20, 0, -0.05, -0.05, -0.5], [30, 20, 1, 0.05, 0.05, 0.5], 6)
    P, A = _np(Pd, Ad)
    A = A.copy()
    A["likelihood"]["mean"] = np.random.default_rng(1).uniform(0.0, 1.0, n).astype(np.float32)
    Pd2, Ad2 = _dev(P, A)
    check(up.estimateStats(Pd2, Ad2, 10 ** 6), P, A)
    up.initSamplesUniform(Pd, Ad, [-30, -20, 0, 0, 0, -np.pi], [30, 20, 0, 0, 0, np.pi], 7)
    check(up.estimateStats(Pd, Ad, 10 ** 6), *_np(Pd, Ad), rotation_gap=False, covariance=False)


def _scene():
    import rmcl_b200
    from rmcl_b200 import synth
    gmap = gpu_map("building:200000")
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gmap)
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(m); h.find(Tgt)
    beams = synth.pf_beams(h.modelView()["points"], 180)
    return gmap, Tsb, Tgt, beams


def test_likelihoods_from_a_sensor_update():
    """weights from a real update() on the synthetic building span orders of magnitude: dist_sigma is narrow (0.05 m) and the particles are
    up to 5 m, 1 m in height and 0.2 rad in roll and pitch off, so that the beams to the floor miss too (the likelihood is a mean over the
    beams, so a particle only drops far when almost all of its beams do)"""
    import rmcl_b200
    import torch
    gmap, Tsb, Tgt, beams = _scene()
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    n = 100_000
    Pd = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    Ad = torch.empty((n, 9), dtype=torch.float32, device="cuda")
    gx, gy, gz = (float(v) for v in Tgt["t"])
    up.initSamplesUniform(Pd, Ad, [gx - 5.0, gy - 5.0, gz - 1.0, -0.2, -0.2, -0.4], [gx + 5.0, gy + 5.0, gz + 1.0, 0.2, 0.2, 0.4], 12)
    prm = rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.05
    up.update(Pd, Ad, Tsb, beams, prm)
    P, A = _np(Pd, Ad)
    L = A["likelihood"]["mean"][:50_000]
    pos = L[L > 0]
    assert pos.max() / pos.min() > 1e2, (pos.min(), pos.max())
    print(f"likelihoods of the induction slice: {pos.min():.3g} .. {pos.max():.3g}, {int((L == 0).sum())} zero")
    check(up.estimateStats(Pd, Ad), P[:50_000], A[:50_000])


def test_equal_weights_dominant_particle_and_zero_sum():
    up = _updater()
    P, A = _random_set(30_000, seed=9)
    A["likelihood"]["mean"] = 0.3
    rec = check(up.estimateStats(*_dev(P, A)), P, A)
    assert rec["likelihood"]["max"] == rec["likelihood"]["min"] == np.float64(np.float32(0.3))
    # one particle carries all the weight but for 1e-30 on the others: its pose, and a covariance of (almost) nothing
    A["likelihood"]["mean"] = 1e-30
    A["likelihood"]["mean"][12_345] = 1.0
    rec = up.estimateStats(*_dev(P, A))
    check(rec, P, A, rotation_gap=False)
    assert np.array_equal(rec["position"], P["t"][12_345].astype(np.float64))
    assert np.abs(rec["orientation"] - er.canonical(P["R"][12_345].astype(np.float64))).max() <= EPS32
    assert np.abs(rec["covariance"]).max() <= 1e-9
    # L_sum = 0 (decision E3): NaN pose and covariance, the rest filled in, B2_OK
    A["likelihood"]["mean"] = 0.0
    rec = up.estimateStats(*_dev(P, A))
    check(rec, P, A)
    assert rec["likelihood"]["max"] == 0.0 and rec["likelihood"]["mean"] == 0.0 and rec["likelihood"]["sigma"] == 0.0 and rec["nparticles"] == 30_000


def test_refusals_leave_the_output_untouched():
    import rmcl_b200
    from rmcl_b200 import synth
    from rmcl_b200.api import _devptr
    up = _updater()
    lib = rmcl_b200.load_library()
    P, A = _random_set(300, seed=2)
    Pd, Ad = _dev(P, A)
    out = np.full(synth.PARTICLE_STATS_DTYPE.itemsize, 0x5a, np.uint8)
    before_bytes = out.tobytes()
    chk = rmcl_b200.api._chk
    p = C.c_void_p(out.ctypes.data)

    def refused(fn, what):
        before = rmcl_b200.kernel_launch_count()
        with pytest.raises(rmcl_b200.B2Error) as e:
            fn()
        assert e.value.code == -1 and what in str(e.value), str(e.value)
        assert rmcl_b200.kernel_launch_count() == before
        assert out.tobytes() == before_bytes
        assert lib.b2_peek_cuda_error().decode() == ""

    refused(lambda: chk(lib.b2_pf_estimate_stats(up._h, _devptr(Pd), _devptr(Ad), C.c_uint32(0), p)), "n = 0")
    refused(lambda: chk(lib.b2_pf_estimate_stats(up._h, None, _devptr(Ad), C.c_uint32(300), p)), "poses_dev")
    refused(lambda: chk(lib.b2_pf_estimate_stats(up._h, _devptr(Pd), None, C.c_uint32(300), p)), "attrs_dev")
    refused(lambda: chk(lib.b2_pf_estimate_stats(up._h, _devptr(Pd), _devptr(Ad), C.c_uint32(300), None)), "out_host")
    refused(lambda: chk(lib.b2_pf_estimate_stats(None, _devptr(Pd), _devptr(Ad), C.c_uint32(300), p)), "'h'")
    with pytest.raises(rmcl_b200.B2Error):
        up.estimateStats(Pd, Ad, max_induction_particles=0)
    with pytest.raises(ValueError):
        up.estimateStats(Pd, Ad[:299])


def test_back_to_back_calls_are_bit_identical():
    up = _updater()
    P, A = _random_set(1_000_003, seed=21)
    Pd, Ad = _dev(P, A)
    a = up.estimateStats(Pd, Ad, 10 ** 7)
    b = up.estimateStats(Pd, Ad, 10 ** 7)
    assert a.tobytes() == b.tobytes()
    other = _updater()                                                              # a second handle: its own scratch, same result
    assert other.estimateStats(Pd, Ad, 10 ** 7).tobytes() == a.tobytes()


@pytest.mark.parametrize("cov", ["full", "rviz"])
def test_round_trip_on_the_device(cov):
    """initSamples(pose, C) -> estimateStats at 10^6 particles gives back pose and C within 5 standard errors (tests/test_pf_estimate.py
    states why the full covariance has no correlation between the angles)"""
    import torch
    from test_pf_estimate import _angle_diagonal, _roundtrip_ok
    up = _updater()
    C0, pose = _gauss_case()
    Cv = _angle_diagonal(C0) if cov == "full" else RVIZ_COV
    n = 1_000_000
    Pd = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    Ad = torch.empty((n, 9), dtype=torch.float32, device="cuda")
    up.initSamples(Pd, Ad, pose, Cv, 11)
    rec = up.estimateStats(Pd, Ad, max_induction_particles=n)
    ok, worst = _roundtrip_ok(rec, pose, Cv, n)
    assert ok, worst
    check(rec, *_np(Pd, Ad))
    print(f"{cov}: worst ratio to the standard error {worst:.2f}")


def test_cpp_classes_match_python(tmp_path):
    """tests/pf_estimate_cpp: PCDSensorUpdaterB200::estimateStats + fillParticleStats into a message-shaped struct, byte for byte the Python
    path's record"""
    import rmcl_b200
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "pf_estimate_cpp")
    lib_dir = os.path.dirname(rmcl_b200.lib_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "pf_estimate_cpp", "pf_estimate_cpp.cpp"), "-L" + lib_dir, "-lrmcl_b200",
                           "-L" + os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + lib_dir])
    P, A = _random_set(60_000, seed=33)
    src = str(tmp_path / "particles.bin")
    with open(src, "wb") as f:
        f.write(P.tobytes()); f.write(A.tobytes())
    out = str(tmp_path / "stats.bin")
    r = subprocess.run([exe, src, out, "50000"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "REFUSED" in r.stdout and "n = 0" in r.stdout
    want = _updater().estimateStats(*_dev(P, A))
    assert open(out, "rb").read() == want.tobytes()


def _tracking(seed):
    """initSamples 0.5 m and 0.2 rad off the true pose of the building map, then ten rounds of motion (standing still), sensor update,
    estimate and Gladiator resampling on one handle -> the ten estimates' (translation, yaw) errors and the last particle set"""
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    gmap, Tsb, Tgt, beams = _scene()
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    n = 100_000
    Pd = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    Ad = torch.empty((n, 9), dtype=torch.float32, device="cuda")
    yaw_gt = 2.0 * np.arctan2(float(Tgt["R"][2]), float(Tgt["R"][3]))
    start = synth.make_transform(np.asarray(Tgt["t"], np.float64) + [0.3, 0.4, 0.0], (0.0, 0.0, yaw_gt + 0.2))
    up.initSamples(Pd, Ad, start, RVIZ_COV, seed)
    glad, prm = rmcl_b200.GladiatorConfig.defaults(), rmcl_b200.PFParams.defaults()
    still = synth.make_transform()
    errs, recs = [], []
    for step in range(10):
        up.motionUpdate(Pd, Ad, still, 0.01)
        up.update(Pd, Ad, Tsb, beams, prm)
        rec = up.estimateStats(Pd, Ad)
        recs.append(rec)
        dt = float(np.linalg.norm(rec["position"][:2] - np.asarray(Tgt["t"][:2], np.float64)))
        q = rec["orientation"]
        dyaw = abs((2.0 * np.arctan2(q[2], q[3]) - yaw_gt + np.pi) % (2 * np.pi) - np.pi)
        errs.append((dt, dyaw))
        Pn, An = torch.empty_like(Pd), torch.empty_like(Ad)
        up.resample(Pd, Ad, Pn, An, glad, seed=seed, step=step)
        Pd, Ad = Pn, An
    return errs, b"".join(r.tobytes() for r in recs), _np(Pd, Ad)


def test_tracking_cycle_on_one_handle():
    """a seeded tracking cycle: bit-identical across two runs, and the estimate's error after ten rounds below half the initial offset
    (0.25 m, 0.1 rad)"""
    e1, r1, (P1, A1) = _tracking(77)
    e2, r2, (P2, A2) = _tracking(77)
    assert r1 == r2 and P1.tobytes() == P2.tobytes() and A1.tobytes() == A2.tobytes()
    print("estimate error per round (m, rad): " + ", ".join(f"({a:.3f}, {b:.3f})" for a, b in e1))
    assert e1[-1][0] < 0.25 and e1[-1][1] < 0.1, e1
