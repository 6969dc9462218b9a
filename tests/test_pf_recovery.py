"""The recovery from a kidnapping (b2_pf_recovery_observe / b2_pf_recovery_inject, PCDSensorUpdaterB200.recovery*) on the CPU.

* The product's pf_recovery_one, compiled for the host over its host-built BVH, is byte-identical in poses, attributes and counts to the C
  restatement of decision, candidates and acceptance (tests/pf_recovery_ref/) on synth.terrain, a tilted plane and a small building, with
  and without the surface, for p in {0, 0.01, 0.3, 1} and max_tries in {1, 16, 64}.
* The product's pf_recovery_filter equals a float64 transcription of the recurrence, bit for bit.
* Statistics: the replaced fraction, uniformity of the candidates in box mode, ground under every candidate taken in surface mode, nothing
  taken off the terrain's footprint; failed particles are left byte for byte as they were.
* The C++ mirror compiles against the header."""
import math
import os
import subprocess

import numpy as np
import pytest

from pf_recovery_ref import ProductRecovery, RefRecovery, filter64, product_filter
from rmcl_b200 import synth
from rmcl_b200.api import SurfaceConfig
from rmcl_b200.synth import PARTICLE_ATTR_DTYPE, RECOVERY_STATE_DTYPE, TRANSFORM_DTYPE
from test_pf_surface import PLANE_A, PLANE_B, PLANE_BOUND, PLANE_HALF, TERRAIN_TRIS, _plane

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILDING_FACES = 4000
# the terrain's footprint: the floor's two rectangles and the bump field fill [0, 64] x [0, 32]
TERRAIN_XY = (0.0, 0.0, 64.0, 32.0)
_SCENES = {}


def scene_mesh(name):
    if name == "terrain":
        return synth.terrain(TERRAIN_TRIS)
    if name == "plane":
        return _plane()
    return synth.building(BUILDING_FACES)


def _scenes(name):
    if name not in _SCENES:
        V, F = scene_mesh(name)
        _SCENES[name] = (ProductRecovery(V, F), RefRecovery(V, F), (V, F))
    return _SCENES[name]


def scene_box(name):
    """a box that reaches 2 m beyond the map on every side, z from 0 to 0.5 m, roll and pitch 0, yaw [-pi, pi)"""
    V = scene_mesh(name)[0]
    lo, hi = V.min(0).astype(np.float64), V.max(0).astype(np.float64)
    return [lo[0] - 2.0, lo[1] - 2.0, 0.0, 0.0, 0.0, -math.pi], [hi[0] + 2.0, hi[1] + 2.0, 0.5, 0.0, 0.0, math.pi]


def particles(n, seed, lo=(-5.0, -5.0, 0.0), hi=(5.0, 5.0, 1.0)):
    """n particles with random poses, stamps and attributes (likelihood > 0, so a replaced one is told apart by its zero attributes)"""
    rng = np.random.default_rng(seed)
    P, A = np.zeros(n, TRANSFORM_DTYPE), np.zeros(n, PARTICLE_ATTR_DTYPE)
    P["t"] = rng.uniform(lo, hi, (n, 3)).astype(np.float32)
    q = rng.normal(size=(n, 4))
    P["R"] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    P["stamp"] = rng.integers(1, 2**32, n, dtype=np.uint64).astype(np.uint32)
    A["likelihood"]["mean"] = rng.uniform(0.1, 1.0, n)
    A["likelihood"]["sigma"] = rng.uniform(0.0, 0.1, n)
    A["likelihood"]["n_meas"] = rng.integers(1, 5000, n)
    A["state_sigma"] = rng.uniform(0.0, 1.0, (n, 6))
    return P, A


def replaced_mask(A):
    return A.view(np.uint8).reshape(len(A), 36).any(1) == 0


P_VALUES = [0.0, 0.01, 0.3, 1.0]
TRIES = [1, 16, 64]


@pytest.mark.parametrize("max_tries", TRIES)
@pytest.mark.parametrize("p", P_VALUES)
@pytest.mark.parametrize("surface", [True, False], ids=["surface", "box"])
@pytest.mark.parametrize("name", ["terrain", "plane", "building"])
def test_product_matches_restatement(name, surface, p, max_tries):
    prod, ref, _ = _scenes(name)
    P, A = particles(3000, seed=int(p * 100) + max_tries)
    lo, hi = scene_box(name)
    cfg = SurfaceConfig.defaults() if surface else None
    kw = dict(surface=cfg, max_tries=max_tries, seed=41, step=5, first=1000)
    Pp, Ap, cp = prod.inject(P, A, p, lo, hi, **kw)
    Pr, Ar, cr = ref.inject(P, A, p, lo, hi, **kw)
    assert Pp.tobytes() == Pr.tobytes() and Ap.tobytes() == Ar.tobytes() and cp == cr
    rep = replaced_mask(Ap)
    assert cp[0] == int(rep.sum())
    assert Pp[~rep].tobytes() == P[~rep].tobytes() and Ap[~rep].tobytes() == A[~rep].tobytes()
    assert (Pp["stamp"][rep] == 0).all()
    if p == 0.0:
        assert cp == (0, 0)
    if not surface and p > 0.0:
        assert cp[1] == 0


def test_draws_are_keyed_by_global_index_and_step():
    """slices concatenate to the whole; another step or seed draws afresh"""
    prod, _, _ = _scenes("terrain")
    P, A = particles(4000, seed=3)
    lo, hi = scene_box("terrain")
    cfg = SurfaceConfig.defaults()
    Pw, Aw, cw = prod.inject(P, A, 0.3, lo, hi, surface=cfg, seed=8, step=2)
    P1, A1, c1 = prod.inject(P[:1500], A[:1500], 0.3, lo, hi, surface=cfg, seed=8, step=2)
    P2, A2, c2 = prod.inject(P[1500:], A[1500:], 0.3, lo, hi, surface=cfg, seed=8, step=2, first=1500)
    assert np.concatenate([P1, P2]).tobytes() == Pw.tobytes() and np.concatenate([A1, A2]).tobytes() == Aw.tobytes()
    assert (c1[0] + c2[0], c1[1] + c2[1]) == cw
    for kw in (dict(seed=8, step=3), dict(seed=9, step=2)):
        Po, _, _ = prod.inject(P, A, 0.3, lo, hi, surface=cfg, **kw)
        assert Po.tobytes() != Pw.tobytes()


def _state(w_avg=0.0, w_slow=0.0, w_fast=0.0, p=0.0):
    s = np.zeros((), RECOVERY_STATE_DTYPE)
    s["w_avg"], s["w_slow"], s["w_fast"], s["p_inject"] = w_avg, w_slow, w_fast, p
    return s


def _check_filter(S, n, a_s, a_f, st):
    got = product_filter(S, n, a_s, a_f, st)
    want = filter64(S, n, a_s, a_f, st)
    assert np.array([float(got[k]) for k in ("w_avg", "w_slow", "w_fast", "p_inject")]).tobytes() == np.array(want).tobytes(), (S, n, a_s, a_f, st, got, want)
    return got


def test_filter_matches_float64_recurrence():
    rng = np.random.default_rng(11)
    for a_s, a_f in ((0.001, 0.1), (0.05, 0.05), (0.0, 1.0), (0.0, 0.0), (1.0, 1.0), (0.3, 0.7)):
        st = _state()
        for k in range(300):
            n = int(rng.integers(1, 2_000_000))
            S = float(rng.uniform(0.0, 1.0)) * n * float(rng.choice([1.0, 1e-3, 1e-30]))
            st = _check_filter(S, n, a_s, a_f, st)
            if k % 50 == 49:
                st = _state(w_avg=float(st["w_avg"]))                   # the injection's reset: both averages restart from w_avg
    # w_slow == 0 takes w_avg as it is; NaN, infinite and negative S leave the record (w_avg is still reported)
    st = _check_filter(3.0, 4, 0.001, 0.1, _state())
    assert float(st["w_slow"]) == float(st["w_fast"]) == 0.75 and float(st["p_inject"]) == 0.0
    before = _check_filter(1.0, 4, 0.001, 0.1, st)
    for S in (float("nan"), float("inf"), -1.0, -1e-300):
        after = _check_filter(S, 4, 0.001, 0.1, before)
        assert [float(after[k]) for k in ("w_slow", "w_fast", "p_inject")] == [float(before[k]) for k in ("w_slow", "w_fast", "p_inject")]
    # equal rates never inject; a fast average above the slow one never injects
    st = _state()
    for S in (1.0, 0.5, 0.1, 0.9):
        st = _check_filter(S, 1, 0.2, 0.2, st)
        assert float(st["p_inject"]) == 0.0
    # two observes with rates 0 and 1 set p = 1 - b / a (the GPU tests set p this way)
    st = _check_filter(0.8, 1, 0.0, 1.0, _state())
    st = _check_filter(0.2, 1, 0.0, 1.0, st)
    assert float(st["w_slow"]) == 0.8 and abs(float(st["p_inject"]) - 0.75) <= 1e-15
    # S == 0 with a zero record: w_slow stays 0, p 0
    st = _check_filter(0.0, 10, 0.001, 0.1, _state())
    assert float(st["w_slow"]) == 0.0 and float(st["p_inject"]) == 0.0


@pytest.mark.parametrize("p", [0.01, 0.3])
def test_replaced_fraction_is_binomial(p):
    prod, _, _ = _scenes("plane")
    n = 200_000
    P, A = particles(n, seed=5)
    lo, hi = scene_box("plane")
    _, Ap, (rep, fail) = prod.inject(P, A, p, lo, hi, max_tries=1, seed=17, step=4)
    assert fail == 0 and rep == int(replaced_mask(Ap).sum())
    assert abs(rep - n * p) <= 5.0 * math.sqrt(n * p * (1.0 - p))


def _rpy(R):
    q = np.asarray(R, np.float64)
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    roll = np.arctan2(2 * (w * x + y * z), 1 - 2 * (x * x + y * y))
    pitch = np.arcsin(np.clip(2 * (w * y - z * x), -1, 1))
    yaw = np.arctan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))
    return np.stack([roll, pitch, yaw], 1)


def test_box_candidates_are_uniform():
    """every dimension of the taken candidates passes a Kolmogorov-Smirnov test for the uniform distribution over the box (the angles read
    back from the quaternion; their float rounding is far below what the test can see at this n)"""
    from scipy import stats
    prod, _, _ = _scenes("plane")
    n = 50_000
    P, A = particles(n, seed=6)
    lo, hi = [-3.0, 1.0, 0.25, -0.5, -0.4, -math.pi], [7.0, 2.5, 0.75, 0.5, 0.4, math.pi]
    Pp, Ap, (rep, _) = prod.inject(P, A, 1.0, lo, hi, max_tries=1, seed=23, step=0)
    assert rep == n
    v = np.concatenate([Pp["t"].astype(np.float64), _rpy(Pp["R"])], 1)
    for k in range(6):
        pv = stats.kstest(v[:, k], "uniform", args=(lo[k], hi[k] - lo[k])).pvalue
        assert pv > 1e-4, (k, pv)


def test_surface_candidates_stand_on_ground():
    """on the tilted plane every taken particle lies on the plane within PLANE_BOUND with its z-axis on the normal; on the terrain none is
    taken off the footprint, and with max_tries 64 nearly every chosen one finds ground"""
    prod, _, _ = _scenes("plane")
    n = 20_000
    P, A = particles(n, seed=7)
    lo, hi = [-PLANE_HALF - 4.0, -PLANE_HALF - 4.0, 0.0, 0.0, 0.0, -math.pi], [PLANE_HALF + 4.0, PLANE_HALF + 4.0, 0.0, 0.0, 0.0, math.pi]
    # the plane's height reaches 3 m at the corners: probe from 4 m above the candidate
    cfg = SurfaceConfig(4.0, 4.0, 0.0, 0.6, 1)
    Pp, Ap, (rep, fail) = prod.inject(P, A, 1.0, lo, hi, surface=cfg, max_tries=1, seed=29, step=1)
    m = replaced_mask(Ap)
    assert rep == int(m.sum()) and rep + fail == n
    area = (2 * PLANE_HALF) ** 2 / (2 * PLANE_HALF + 8.0) ** 2
    assert abs(rep - n * area) <= 5.0 * math.sqrt(n * area * (1 - area))
    t = Pp["t"][m].astype(np.float64)
    assert (np.abs(t[:, :2]) <= PLANE_HALF).all()
    assert np.abs(t[:, 2] - (PLANE_A * t[:, 0] + PLANE_B * t[:, 1])).max() <= PLANE_BOUND
    nrm = np.array([-PLANE_A, -PLANE_B, 1.0]) / math.sqrt(PLANE_A ** 2 + PLANE_B ** 2 + 1.0)
    q = Pp["R"][m].astype(np.float64)
    u, w = q[:, :3], q[:, 3:]
    ez = np.array([0.0, 0.0, 1.0])
    up = ez + 2.0 * np.cross(u, np.cross(u, ez) + w * ez)
    assert np.abs(up - nrm).max() <= 1e-5
    # terrain: nothing off the footprint, and 64 tries leave almost no particle without ground
    prod_t, _, _ = _scenes("terrain")
    lo, hi = scene_box("terrain")
    Pt, At, (rep, fail) = prod_t.inject(P, A, 1.0, lo, hi, surface=SurfaceConfig.defaults(), max_tries=64, seed=31, step=1)
    m = replaced_mask(At)
    x, y = Pt["t"][m, 0], Pt["t"][m, 1]
    assert ((x >= TERRAIN_XY[0]) & (x <= TERRAIN_XY[2]) & (y >= TERRAIN_XY[1]) & (y <= TERRAIN_XY[3])).all()
    assert rep + fail == n and fail <= n // 1000


def test_failed_particles_are_untouched():
    """with a box far off the map and the surface given, every chosen particle fails: all of them, poses, stamps and attributes, stay"""
    prod, ref, _ = _scenes("terrain")
    P, A = particles(5000, seed=9)
    lo, hi = [100.0, 100.0, 0.0, 0.0, 0.0, -math.pi], [120.0, 120.0, 0.5, 0.0, 0.0, math.pi]
    for scene in (prod, ref):
        Pp, Ap, (rep, fail) = scene.inject(P, A, 0.3, lo, hi, surface=SurfaceConfig.defaults(), max_tries=16, seed=2, step=0)
        assert rep == 0 and 0 < fail < 5000
        assert Pp.tobytes() == P.tobytes() and Ap.tobytes() == A.tobytes()


def test_cpp_mirror_compiles_against_the_header():
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    out = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"),
                          os.path.join(ROOT, "tests", "pf_recovery_cpp", "pf_recovery_cpp.cpp")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-4000:]
