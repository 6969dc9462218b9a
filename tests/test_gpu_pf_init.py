"""GPU tests of the particle set initialisers (b2_pf_init_uniform / b2_pf_init_gaussian, k_pf_init_uniform / k_pf_init_gaussian) against
the reference of tests/pf_init_ref on the same seed, and of a whole particle-filter cycle started from the device.

Tolerances.  The Philox words are integers, so everything the kernels compute without a transcendental function is bit-exact: the
uniform translations (one subtraction, one multiplication, one addition, one min, each individually rounded), the attributes and the
stamps.  Quaternions go through device sinf/cosf, within 2 ulp of glibc: 2e-6 per component, as in test_gladiator_resample_gpu.

The Gaussian draws go through device logf/sinf/cosf as well: each normal is within 4e-6 of the host's (test_gladiator_resample_gpu
asserts this bound for the same Box-Muller code).  With e = 4e-6 and s = the largest row sum of |L|:
  * x = L N differs by at most s e, plus the rounding of six products and six sums: 12 ulp(|x|max), bounded by 12 * 2^-23 |x|max;
  * t = R_pose x_t + t_pose: the rotation keeps lengths, so |dt| <= sqrt(3) (s e + 12 ulp) per component, plus the rounding of the rotation
    and the addition, a few ulp of |t|max;
  * each quaternion component is a sum of products of cos and sin of half angles, so it moves by at most 3 * dx/2 through the angles,
    plus the 2e-6 of the device functions, plus the pose product's rounding (a few ulp of 1)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import pf_init_ref as ref
from conftest import gpu_map
from test_pf_init import BOX_MAX, BOX_MIN, RVIZ_COV, _gauss_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = float(np.finfo(np.float32).eps)


def _updater():
    import rmcl_b200
    return rmcl_b200.PCDSensorUpdaterB200(gpu_map("cube29"))


def _tensors(n, fill=None):
    import torch
    P = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    A = torch.empty((n, 9), dtype=torch.float32, device="cuda")
    if fill is not None:
        P.fill_(fill); A.fill_(fill)
    return P, A


def _np(P, A):
    import torch
    from rmcl_b200 import synth
    torch.cuda.synchronize()
    return P.cpu().numpy().view(synth.TRANSFORM_DTYPE).reshape(-1), A.cpu().numpy().view(synth.PARTICLE_ATTR_DTYPE).reshape(-1)


def _uniform(up, first, n, seed, lo=BOX_MIN, hi=BOX_MAX):
    P, A = _tensors(n)
    up.initSamplesUniform(P, A, lo, hi, seed, first=first)
    return _np(P, A)


def _gaussian(up, first, n, pose, cov, seed):
    P, A = _tensors(n)
    up.initSamples(P, A, pose, cov, seed, first=first)
    return _np(P, A)


def _check_uniform(gP, gA, rP, rA):
    assert np.array_equal(gP["t"], rP["t"])                                            # bit-exact
    assert np.abs(gP["R"].astype(np.float64) - rP["R"]).max() <= 2e-6                  # device sinf / cosf
    assert gA.tobytes() == rA.tobytes() and np.array_equal(gP["stamp"], rP["stamp"])


def _gauss_tols(L, rP):
    s = float(np.abs(L.astype(np.float64)).sum(1).max())
    xmax = 10.0 * float(np.sqrt((L.astype(np.float64) ** 2).sum(1)).max())             # |N| <= 5.6 for u1 >= 2^-25 (Box-Muller), per component
    dx = s * 4e-6 + 12 * EPS * xmax
    tol_t = np.sqrt(3.0) * dx + 8 * EPS * float(np.abs(rP["t"]).max())
    tol_R = 1.5 * dx + 2e-6 + 8 * EPS
    return tol_t, tol_R


def _check_gaussian(gP, gA, rP, rA, L):
    tol_t, tol_R = _gauss_tols(L, rP)
    assert np.abs(gP["t"].astype(np.float64) - rP["t"]).max() <= tol_t
    assert np.abs(gP["R"].astype(np.float64) - rP["R"]).max() <= tol_R
    assert gA.tobytes() == rA.tobytes() and np.array_equal(gP["stamp"], rP["stamp"])


def test_uniform_matches_reference():
    up = _updater()
    n = 1_000_003                                                                      # partial last block
    gP, gA = _uniform(up, 0, n, seed=4242)
    rP, rA = ref.init_uniform(0, n, BOX_MIN, BOX_MAX, seed=4242)
    _check_uniform(gP, gA, rP, rA)
    lo, hi = ref.box32(BOX_MIN, BOX_MAX)
    assert np.all(gP["t"] >= lo[:3]) and np.all(gP["t"] <= hi[:3]) and np.all(gP["t"][:, 2] == lo[2])


@pytest.mark.parametrize("cov", ["full", "rviz"])
def test_gaussian_matches_reference(cov):
    up = _updater()
    C, pose = _gauss_case()
    if cov == "rviz":
        C = RVIZ_COV
    n = 1_000_003
    gP, gA = _gaussian(up, 0, n, pose, C, seed=99)
    rP, rA = ref.init_gaussian(0, n, pose, C, seed=99)
    _check_gaussian(gP, gA, rP, rA, ref.chol6(C)[0])
    assert np.all(np.isfinite(gP["t"])) and np.all(np.isfinite(gP["R"]))


@pytest.mark.parametrize("n", [1, 255, 256, 257])
def test_small_counts(n):
    up = _updater()
    C, pose = _gauss_case()
    _check_uniform(*_uniform(up, 7, n, seed=5), *ref.init_uniform(7, n, BOX_MIN, BOX_MAX, seed=5))
    _check_gaussian(*_gaussian(up, 7, n, pose, C, seed=5), *ref.init_gaussian(7, n, pose, C, seed=5), ref.chol6(C)[0])


def test_shards_concatenate_and_seeds_differ():
    up = _updater()
    C, pose = _gauss_case()
    n = 100_003
    cuts = [0, 1, 256, 40_000, 100_002, n]
    for run in (lambda f, m, s: _uniform(up, f, m, s), lambda f, m, s: _gaussian(up, f, m, pose, C, s)):
        whole = run(0, n, 77)
        parts = [run(a, b - a, 77) for a, b in zip(cuts[:-1], cuts[1:])]
        for k in (0, 1):
            assert np.concatenate([p[k] for p in parts]).tobytes() == whole[k].tobytes()
        again = run(0, n, 77)
        assert again[0].tobytes() == whole[0].tobytes() and again[1].tobytes() == whole[1].tobytes()
        other = run(0, n, 78)
        assert np.all(other[0]["t"][:, :2] != whole[0]["t"][:, :2], axis=1).mean() > 0.999
    # the two kinds draw from different counters: over the unit box the uniform x, y are the first two words (r >> 8) 2^-24; had the
    # Gaussian kind read the same words, its x (identity pose and covariance) would be their first Box-Muller normal
    from rmcl_b200 import synth
    u = _uniform(up, 0, 1000, 77, lo=[0] * 6, hi=[1] * 6)[0]
    g = _gaussian(up, 0, 1000, synth.make_transform(), np.eye(6), 77)[0]
    u0, u1 = (u["t"][:, k].astype(np.float64) + 2.0 ** -25 for k in (0, 1))
    same_words = np.sqrt(-2.0 * np.log(u0)) * np.cos(2.0 * np.pi * u1)
    assert np.mean(np.abs(same_words - g["t"][:, 0]) < 1e-3) < 0.01


def test_refusals_leave_outputs_untouched():
    import ctypes as C
    import rmcl_b200
    from rmcl_b200.api import _devptr
    up = _updater()
    lib = rmcl_b200.load_library()
    C6, pose = _gauss_case()
    P, A = _tensors(300, fill=-7.0)
    P0, A0 = _np(P, A)

    def refused(fn, *args, what=""):
        before = rmcl_b200.kernel_launch_count()
        with pytest.raises(rmcl_b200.B2Error) as e:
            fn(*args)
        assert e.value.code == -1 and what in str(e.value), str(e.value)
        assert rmcl_b200.kernel_launch_count() == before
        gP, gA = _np(P, A)
        assert gP.tobytes() == P0.tobytes() and gA.tobytes() == A0.tobytes()
        assert lib.b2_peek_cuda_error().decode() == ""

    lo, hi = list(BOX_MIN), list(BOX_MAX)
    refused(up.initSamplesUniform, P, A, lo, hi, 1, 2**32 - 299, what="2^32")
    refused(up.initSamples, P, A, pose, C6, 1, 2**32 - 1, what="2^32")
    bad = list(lo); bad[1] = 31.0                                                             # y: min > max
    refused(up.initSamplesUniform, P, A, bad, hi, 1, what="min > max")
    bad = list(lo); bad[4] = float("nan")
    refused(up.initSamplesUniform, P, A, bad, hi, 1, what="pitch")
    bad = list(hi); bad[0] = float("inf")
    refused(up.initSamplesUniform, P, A, lo, bad, 1, what="not finite")
    bad = list(hi); bad[0] = 1e300                                                            # finite double, infinite float
    refused(up.initSamplesUniform, P, A, lo, bad, 1, what="not finite")
    bad = list(lo); bad[0] = -3e38; bad2 = list(hi); bad2[0] = 3e38                            # extent overflows float
    refused(up.initSamplesUniform, P, A, bad, bad2, 1, what="overflows")
    neg = np.array(RVIZ_COV); neg[1, 1] = -0.25
    refused(up.initSamples, P, A, pose, neg, 1, what="column 1")
    nan = np.array(RVIZ_COV); nan[3, 3] = np.nan
    refused(up.initSamples, P, A, pose, nan, 1, what="(3,3)")
    zc = np.array(RVIZ_COV); zc[4, 2] = zc[2, 4] = 0.01
    refused(up.initSamples, P, A, pose, zc, 1, what="column 2")
    # null pointers through the C ABI
    box_lo, box_hi = np.array(lo, np.float64), np.array(hi, np.float64)
    T = np.ascontiguousarray(pose).reshape(1)
    cov = np.ascontiguousarray(C6, np.float64).reshape(36)
    p = lambda a: C.c_void_p(a.ctypes.data)
    chk = rmcl_b200.api._chk
    refused(lambda: chk(lib.b2_pf_init_uniform(up._h, None, _devptr(A), C.c_uint32(0), C.c_uint32(300), p(box_lo), p(box_hi), C.c_uint64(1))), what="poses_dev")
    refused(lambda: chk(lib.b2_pf_init_uniform(up._h, _devptr(P), None, C.c_uint32(0), C.c_uint32(300), p(box_lo), p(box_hi), C.c_uint64(1))), what="attrs_dev")
    refused(lambda: chk(lib.b2_pf_init_uniform(up._h, _devptr(P), _devptr(A), C.c_uint32(0), C.c_uint32(300), None, p(box_hi), C.c_uint64(1))), what="bb_min")
    refused(lambda: chk(lib.b2_pf_init_gaussian(up._h, _devptr(P), _devptr(A), C.c_uint32(0), C.c_uint32(300), None, p(cov), C.c_uint64(1))), what="pose")
    refused(lambda: chk(lib.b2_pf_init_gaussian(up._h, _devptr(P), _devptr(A), C.c_uint32(0), C.c_uint32(300), p(T), None, C.c_uint64(1))), what="cov_rowmajor")
    refused(lambda: chk(lib.b2_pf_init_gaussian(None, _devptr(P), _devptr(A), C.c_uint32(0), C.c_uint32(300), p(T), p(cov), C.c_uint64(1))), what="h")
    # n == 0: accepted without a launch, even with null particle pointers
    before = rmcl_b200.kernel_launch_count()
    chk(lib.b2_pf_init_uniform(up._h, None, None, C.c_uint32(5), C.c_uint32(0), p(box_lo), p(box_hi), C.c_uint64(1)))
    chk(lib.b2_pf_init_gaussian(up._h, None, None, C.c_uint32(2**32 - 1), C.c_uint32(0), p(T), p(cov), C.c_uint64(1)))
    assert rmcl_b200.kernel_launch_count() == before
    # the last valid index is accepted
    Q, B = _tensors(1)
    up.initSamplesUniform(Q, B, lo, hi, 3, first=2**32 - 1)
    _check_uniform(*_np(Q, B), *ref.init_uniform(2**32 - 1, 1, lo, hi, seed=3))


def test_cpp_classes_match_python(tmp_path):
    """tests/pf_init_cpp/pf_init_cpp.cpp, compiled here against include/rmcl_b200/rcc_b200.hpp, fills device memory through
    PCDSensorUpdaterB200::initSamplesUniform / initSamples: byte for byte what the Python path gives"""
    import rmcl_b200
    from rmcl_b200 import synth
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "pf_init_cpp")
    lib_dir = os.path.dirname(rmcl_b200.lib_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "pf_init_cpp", "pf_init_cpp.cpp"), "-L" + lib_dir, "-lrmcl_b200",
                           "-L" + os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + lib_dir])
    n, first, seed = 5000, 123, 2024
    out = str(tmp_path / "particles.bin")
    r = subprocess.run([exe, out, str(n), str(first), str(seed)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "REFUSED" in r.stdout and "column 2" in r.stdout
    blob = np.fromfile(out, np.uint8)
    assert len(blob) == 2 * 68 * n
    up = _updater()
    pi = 3.14159265358979
    u = _uniform(up, first, n, seed, lo=[-5.0, -4.0, 0.5, -0.1, 0.0, -pi], hi=[5.0, 4.0, 0.5, 0.1, 0.0, pi])
    pose = np.zeros((), synth.TRANSFORM_DTYPE)
    pose["t"] = [2.0, -1.0, 0.0]
    pose["R"] = [0.0, 0.0, 0.38268343, 0.92387953]
    g = _gaussian(up, first, n, pose, RVIZ_COV, seed)
    want = b"".join(a.tobytes() for a in (*u, *g))
    assert blob.tobytes() == want


def _pf_cycle(seed):
    """global uniform initialisation of 100 000 particles in a box around the true pose of the building map (x, y +-3 m, yaw over +-pi; z,
    roll, pitch fixed), then ten rounds of sensor update (beams traced from the true pose), likelihoodStats and Gladiator resampling"""
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
    n = 100_000
    P, A = _tensors(n)
    up.initSamplesUniform(P, A, [gx - 3.0, gy - 3.0, gz, 0.0, 0.0, -np.pi], [gx + 3.0, gy + 3.0, gz, 0.0, 0.0, np.pi], seed)
    P0 = _np(P, A)[0].copy()
    glad = rmcl_b200.GladiatorConfig.defaults()
    prm = rmcl_b200.PFParams.defaults()
    for step in range(10):
        up.update(P, A, Tsb, beams, prm)
        up.likelihoodStats(A)
        Pn, An = torch.empty_like(P), torch.empty_like(A)
        up.resample(P, A, Pn, An, glad, seed=seed, step=step)
        P, A = Pn, An
    P1, A1 = _np(P, A)
    return P0, P1, A1, Tgt


def _near_share(P, Tgt):
    d = np.linalg.norm(P["t"][:, :2].astype(np.float64) - np.asarray(Tgt["t"][:2], np.float64), axis=1)
    yaw = 2.0 * np.arctan2(P["R"][:, 2].astype(np.float64), P["R"][:, 3].astype(np.float64))
    yaw_gt = 2.0 * np.arctan2(float(Tgt["R"][2]), float(Tgt["R"][3]))
    dyaw = np.abs((yaw - yaw_gt + np.pi) % (2 * np.pi) - np.pi)
    return float(np.mean((d <= 0.25) & (dyaw <= 0.1)))


def test_global_localisation_cycle_on_the_device():
    """the whole cycle on one handle from a device initialisation: bit-identical across two runs, and the share of particles within 0.25 m
    and 0.1 rad of the true pose grows at least 5x over ten rounds"""
    P0, P1, A1, Tgt = _pf_cycle(31)
    Q0, Q1, B1, _ = _pf_cycle(31)
    assert P0.tobytes() == Q0.tobytes() and P1.tobytes() == Q1.tobytes() and A1.tobytes() == B1.tobytes()
    s0, s1 = _near_share(P0, Tgt), _near_share(P1, Tgt)
    assert s0 > 0.0
    assert s1 >= 5.0 * s0, (s0, s1)
    print(f"share within 0.25 m / 0.1 rad of the true pose: {s0:.5f} initially, {s1:.5f} after ten rounds")
