"""CPU tests of residual resampling (b2_pf_resample_residual): the C restatement (tests/pf_residual_ref) against a literal Python
transcription of ResidualResamplerCPU::update's loop (rmcl_ros/src/rmcl/ResidualResamplerCPU.cpp:72-181) fed the same draws and normals;
the product's per-element functions compiled for the CPU against the restatement; properties of the draws; and the deviations of
SURVEY D31 (the draw bound and the invalid weight sums)."""
import ctypes as C
import ctypes.util

import numpy as np
import pytest
from scipy import stats as sps

import pf_residual_ref as ref
from rmcl_b200.api import GladiatorConfig
from rmcl_b200.synth import PARTICLE_ATTR_DTYPE, TRANSFORM_DTYPE

f32 = np.float32
CFG = GladiatorConfig(0.03, 0.03, 0.01, 0.002, 0.002, 0.01, 0.3, 0.2)
FAMILIES = ("uniform", "lognormal", "dominant", "half_zero")

_libm = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
for _f, _n in (("sinf", 1), ("cosf", 1), ("asinf", 1), ("sqrtf", 1), ("atan2f", 2)):
    getattr(_libm, _f).restype = C.c_float
    getattr(_libm, _f).argtypes = [C.c_float] * _n
_libm.pow.restype = C.c_double
_libm.pow.argtypes = [C.c_double, C.c_double]


def particles(n, family, seed=0):
    """n particles with stamp = index, |t| <= 20, unit quaternions, random n_meas / sigma / state_sigma, likelihoods of `family`"""
    rng = np.random.default_rng(seed)
    P, A = np.zeros(n, TRANSFORM_DTYPE), np.zeros(n, PARTICLE_ATTR_DTYPE)
    P["t"] = rng.uniform(-20, 20, (n, 3)).astype(np.float32)
    q = rng.normal(size=(n, 4))
    P["R"] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    P["stamp"] = np.arange(n, dtype=np.uint32)
    if family == "uniform":
        L = rng.uniform(0.0, 1.0, n)
    elif family == "lognormal":
        L = np.exp(rng.normal(0.0, 1.5, n))
    elif family == "dominant":
        L = rng.uniform(0.0, 1e-4, n)
        L[rng.integers(n)] = 1.0
    elif family == "half_zero":
        L = rng.uniform(0.0, 1.0, n)
        L[rng.permutation(n)[: n // 2]] = 0.0
    else:
        L = np.full(n, float(family))
    A["likelihood"]["mean"] = L.astype(np.float32)
    A["likelihood"]["sigma"] = rng.uniform(0, 1, n).astype(np.float32)
    A["likelihood"]["n_meas"] = rng.integers(0, 100000, n).astype(np.uint32)
    A["state_sigma"] = rng.uniform(0, 1, (n, 6)).astype(np.float32)
    return P, A


# ---- the reference's loop, transcribed: float32 scalars (each op rounded), libm for sinf / cosf / atan2f / asinf / sqrtf ----------------
def _qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return (aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
            aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz)


def _qconj(q):
    return (-q[0], -q[1], -q[2], q[3])


def _qrot(q, v):
    r = _qmul(_qmul(q, (v[0], v[1], v[2], f32(0))), _qconj(q))
    return r[:3]


def _tmul(a, b):
    R = _qmul(a[0], b[0])
    rt = _qrot(a[0], b[1])
    return R, (rt[0] + a[1][0], rt[1] + a[1][1], rt[2] + a[1][2])


def _tinv(a):
    Ri = _qconj(a[0])
    t = _qrot(Ri, a[1])
    return Ri, (-t[0], -t[1], -t[2])


def _euler(q):
    x, y, z, w = q
    two, one = f32(2), f32(1)
    roll = f32(_libm.atan2f(two * (w * x + y * z), one - two * (x * x + y * y)))
    sinp = two * (w * y - z * x)
    pitch = f32(np.copysign(f32(1.5707963267948966), sinp)) if abs(sinp) >= one else f32(_libm.asinf(sinp))
    yaw = f32(_libm.atan2f(two * (w * z + x * y), one - two * (y * y + z * z)))
    return roll, pitch, yaw


def _quat(roll, pitch, yaw):
    h = f32(0.5)
    cr, sr = f32(_libm.cosf(roll * h)), f32(_libm.sinf(roll * h))
    cp, sp = f32(_libm.cosf(pitch * h)), f32(_libm.sinf(pitch * h))
    cy, sy = f32(_libm.cosf(yaw * h)), f32(_libm.sinf(yaw * h))
    return (sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy)


def reference_loop(P, A, M, cfg, draws, N):
    """ResidualResamplerCPU::update with uniform_distribution(*rand_gen_) replaced by `draws` and Nd(*rand_gen_) by the slot's row of N.
    The loop also ends when the draws run out (the bound of SURVEY D31).  -> (n_particles, parents, insertions, P_new, A_new)"""
    n = len(A)
    weight_sum, weight_max = 0.0, 0.0
    for i in range(n):                                                                  # :78-84
        v = float(A["likelihood"]["mean"][i])
        weight_sum += v
        weight_max = max(weight_max, v)
    Pn, An = np.zeros(M, TRANSFORM_DTYPE), np.zeros(M, PARTICLE_ATTR_DTYPE)
    insertion_idx, it, par, ins = 0, 0, [], []
    while insertion_idx < M and it < len(draws):                                        # :102
        r = int(draws[it])
        it += 1
        pose = (tuple(f32(v) for v in P["R"][r]), tuple(f32(v) for v in P["t"][r]))
        L = float(A["likelihood"]["mean"][r])
        L_sum_normed, L_max_normed = L / weight_sum, L / weight_max
        n_expected = int(L_sum_normed * float(M))
        n_left = M - insertion_idx
        n_ins = n_expected if n_expected <= n_left else n_left
        for inner in range(n_ins):
            k = insertion_idx + inner
            Nk = N[k]
            noise = [f32(float(getattr(cfg, name)) / L_max_normed) for name in
                     ("min_noise_tx", "min_noise_ty", "min_noise_tz", "min_noise_roll", "min_noise_pitch", "min_noise_yaw")]
            t = tuple(pose[1][c] + Nk[c] * noise[c] for c in range(3))
            e = _euler(pose[0])
            e = tuple(e[c] + Nk[3 + c] * noise[3 + c] for c in range(3))
            new = (_quat(*e), t)
            d = _tmul(_tinv(pose), new)
            trans_dist = d[1][0] * d[1][0] + d[1][1] * d[1][1] + d[1][2] * d[1][2]     # l2normSquared
            q = d[0]
            rot_dist = f32(_libm.sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]))
            red = f32(_libm.pow(float(f32(cfg.likelihood_forget_per_meter)), float(trans_dist)) *
                      _libm.pow(float(f32(cfg.likelihood_forget_per_radian)), float(rot_dist)))
            Pn[k]["R"], Pn[k]["t"], Pn[k]["stamp"] = new[0], new[1], P["stamp"][r]
            An[k] = A[r]
            An[k]["likelihood"]["n_meas"] = np.uint32(int(f32(A["likelihood"]["n_meas"][r]) * red))
        par.append(r)
        ins.append(n_ins)
        insertion_idx += n_ins
    return insertion_idx, np.array(par, np.uint32), np.array(ins, np.uint64), Pn, An


def _sizes(n):
    return sorted({1, max(1, n // 2), n, 3 * n})


CASES = [(n, M, fam) for n in (1, 2, 7, 2000) for M in _sizes(n) for fam in FAMILIES]


@pytest.mark.parametrize("n,M,family", CASES)
def test_restatement_matches_reference_loop(n, M, family):
    P, A = particles(n, family, seed=n + M)
    seed, step = 77, 3
    draws = ref.parents(seed, step, 0, ref.d_max(n, M), n)
    N = ref.normals(seed, step, 0, M)
    cnt, par, ins, Pw, Aw = reference_loop(P, A, M, CFG, draws, N)
    got = ref.resample(P, A, M, CFG, seed, step, trace=ref.d_max(n, M))
    assert got["n_particles"] == cnt and got["draws"] == len(par)
    assert np.array_equal(got["parents"], par) and np.array_equal(got["ins"], ins)
    assert got["P"][:cnt].tobytes() == Pw[:cnt].tobytes() and got["A"][:cnt].tobytes() == Aw[:cnt].tobytes()
    # the same loop with the normals handed in
    got2 = ref.resample(P, A, M, CFG, seed, step, N=N)
    assert got2["P"].tobytes() == got["P"].tobytes() and got2["A"].tobytes() == got["A"].tobytes()


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("n,M", [(7, 21), (2000, 1000), (2000, 6000), (333, 50000)])
def test_product_functions_match_restatement(n, M, family):
    P, A = particles(n, family, seed=5)
    seed, step = 0x1234567890ABCDEF, 11
    S, _, L_max = ref.stats(A)
    dm = ref.d_max(n, M)
    par = ref.parents(seed, step, 0, dm, n)
    assert np.array_equal(ref.product_parents(seed, step, 0, dm, n), par)
    L = A["likelihood"]["mean"][par]
    cnt = ref.product_counts(L, S, M)
    want = np.minimum(np.floor(L.astype(np.float64) / S * float(M)), float(M)).astype(np.uint64)
    assert np.array_equal(cnt, want)
    r = ref.resample(P, A, M, CFG, seed, step, trace=dm)
    left = M - np.concatenate([[0], np.cumsum(r["ins"])[:-1]]).astype(np.uint64)
    assert np.array_equal(r["ins"], np.minimum(cnt[: r["draws"]], left))
    N = ref.normals(seed, step, 0, r["n_particles"])
    assert np.array_equal(ref.product_normals(seed, step, 0, r["n_particles"]), N)
    slot_par = np.repeat(r["parents"], r["ins"].astype(np.int64))
    Pp, Ap = ref.product_copies(P, A, slot_par, N, L_max, CFG)
    assert Pp.tobytes() == r["P"][: r["n_particles"]].tobytes() and Ap.tobytes() == r["A"][: r["n_particles"]].tobytes()


def test_parents_past_2_32_draws():
    """the draw index is 64-bit: counter words 0 and 3 carry lo / hi of j / 4"""
    d0 = (1 << 34) + 3
    assert np.array_equal(ref.product_parents(9, 2, d0, 4099, 1000003), ref.parents(9, 2, d0, 4099, 1000003))
    assert not np.array_equal(ref.parents(9, 2, d0, 64, 1000003), ref.parents(9, 2, d0 & 0xFFFFFFFF, 64, 1000003))


def test_zero_likelihood_parents_never_appear():
    P, A = particles(2000, "half_zero", seed=3)
    r = ref.resample(P, A, 4000, CFG, 1, 0)
    assert r["n_particles"] == 4000
    assert np.all(A["likelihood"]["mean"][r["P"]["stamp"]] > 0)


def test_single_nonzero_particle_fills_every_slot():
    P, A = particles(500, 0.0, seed=4)
    A["likelihood"]["mean"][137] = 0.25
    r = ref.resample(P, A, 1000, CFG, 2, 0, trace=16 * 1000)
    first = int(np.flatnonzero(r["parents"] == 137)[0])
    assert r["draws"] == first + 1 and r["n_particles"] == 1000
    assert np.all(r["ins"][:first] == 0) and r["ins"][first] == 1000
    assert np.all(r["P"]["stamp"] == 137)


def test_parent_draws_are_uniform():
    n = 97
    par = ref.parents(4242, 1, 0, 200000, n)
    _, p = sps.chisquare(np.bincount(par, minlength=n))
    assert p > 1e-4
    par = ref.parents(4242, 2, 1 << 33, 200000, n)
    _, p = sps.chisquare(np.bincount(par, minlength=n))
    assert p > 1e-4


def test_all_zero_likelihoods_fill_nothing():
    P, A = particles(100, 0.0)
    r = ref.resample(P, A, 100, CFG, 1, 0)
    assert r["n_particles"] == 0 and r["draws"] == 0
    assert not r["P"].tobytes().strip(b"\0") and not r["A"].tobytes().strip(b"\0")


def test_equal_weights_below_one_copy_exhaust_the_draws():
    P, A = particles(1000, 0.5)
    r = ref.resample(P, A, 999, CFG, 1, 0)
    assert r["draws"] == ref.d_max(1000, 999) and r["n_particles"] == 0


@pytest.mark.parametrize("bad", [-1e-3, float("nan"), float("inf")])
def test_invalid_likelihood_fills_nothing(bad):
    P, A = particles(100, "uniform")
    A["likelihood"]["mean"][42] = bad
    r = ref.resample(P, A, 100, CFG, 1, 0)
    assert r["n_particles"] == 0 and r["draws"] == 0


def test_slices_concatenate_to_the_whole():
    P, A = particles(300, "lognormal", seed=9)
    whole = ref.resample(P, A, 900, CFG, 5, 1)
    parts = [ref.resample(P, A, 900, CFG, 5, 1, first=a, n_local=b - a) for a, b in ((0, 128), (128, 129), (129, 900))]
    assert b"".join(p["P"].tobytes() for p in parts) == whole["P"].tobytes()
    assert b"".join(p["A"].tobytes() for p in parts) == whole["A"].tobytes()
