"""CPU tests of the particle set's pose estimate (RmclNode::estimateStats, rmcl_ros/src/nodes/rmcl_localization.cpp:642-731): the float64
model of tests/pf_estimate_ref on known answers, the round trip through initSamples (tests/pf_init_ref) that pins decision E2 against quirk
D13, and the product's eigen solver and deviation function compiled for the CPU against numpy."""
import numpy as np
import pytest

import pf_estimate_ref as er
import pf_init_ref as ref
from rmcl_b200 import synth
from test_pf_init import RVIZ_COV, _gauss_case

EPS32 = float(np.finfo(np.float32).eps)


def _set(q, t=None, L=None):
    q = np.asarray(q, np.float64).reshape(-1, 4)
    n = len(q)
    P = np.zeros(n, synth.TRANSFORM_DTYPE)
    P["R"] = q.astype(np.float32)
    P["t"] = np.zeros((n, 3)) if t is None else np.asarray(t, np.float32)
    A = np.zeros(n, synth.PARTICLE_ATTR_DTYPE)
    A["likelihood"]["mean"] = 1.0 if L is None else np.asarray(L, np.float32)
    return P, A


def _quat(axis, angle):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.concatenate([np.sin(angle / 2) * axis, [np.cos(angle / 2)]])


def test_symmetric_rotations_give_the_centre():
    """rotations placed symmetrically about a known q (q * exp(+-a u) for three axes u) give q; so do translations about t"""
    q0 = _quat([0.3, -0.2, 0.9], 1.1)
    qs, ts = [], []
    for u in np.eye(3):
        for s in (1.0, -1.0):
            qs.append(er.qmul(q0, _quat(u, s * 0.4)))
            ts.append(np.array([2.0, -1.0, 0.5]) + s * u)
    P, A = _set(qs, ts)
    r, T, _ = er.estimate_np(P, A)
    assert np.abs(r["orientation"] - er.canonical(q0)).max() <= 2 * EPS32
    assert np.abs(r["position"] - [2.0, -1.0, 0.5]).max() <= 2 * EPS32


def test_sign_flips_change_nothing():
    rng = np.random.default_rng(3)
    q = rng.normal(size=(200, 4)) * [0.1, 0.1, 0.3, 1.0]
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    L = rng.uniform(0.01, 1.0, 200)
    P, A = _set(q, rng.normal(size=(200, 3)), L)
    r, _, _ = er.estimate_np(P, A)
    flip = rng.random(200) < 0.5
    P["R"][flip] *= -1
    r2, _, _ = er.estimate_np(P, A)
    assert r.tobytes() == r2.tobytes()
    assert r["orientation"][3] > 0.0


def test_one_particle_with_all_the_weight_gives_its_pose():
    rng = np.random.default_rng(4)
    q = rng.normal(size=(50, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    L = np.zeros(50)
    L[17] = 0.7
    P, A = _set(q, rng.normal(size=(50, 3)) * 10, L)
    r, _, _ = er.estimate_np(P, A)
    assert np.array_equal(r["position"], P["t"][17].astype(np.float64))
    assert np.abs(r["orientation"] - er.canonical(P["R"][17].astype(np.float64))).max() <= EPS32
    assert np.abs(r["covariance"]).max() <= 1e-6                                   # the pose itself: a zero deviation


def test_zero_likelihood_sum_gives_nan_and_the_rest():
    """decision E3: every likelihood 0 -> pose and covariance NaN, likelihood statistics, AABB and nparticles filled in"""
    P, A = _set(np.tile([0.0, 0.0, 0.0, 1.0], (10, 1)), np.arange(30).reshape(10, 3), np.zeros(10))
    r, _, _ = er.estimate_np(P, A)
    assert np.all(np.isnan(r["position"])) and np.all(np.isnan(r["orientation"])) and np.all(np.isnan(r["covariance"]))
    assert r["likelihood"]["min"] == 0.0 and r["likelihood"]["max"] == 0.0 and r["likelihood"]["mean"] == 0.0 and r["likelihood"]["sigma"] == 0.0
    assert r["nparticles"] == 10 and np.array_equal(r["trans_bb_min"], [0, 1, 2]) and np.array_equal(r["trans_bb_max"], [27, 28, 29])


def test_rounding_only_negative_variance_gives_zero_sigma():
    """decision E4: equal likelihoods whose sum_sq / n - mean^2 rounds below zero give sigma 0, not NaN"""
    for v in (0.1, 0.3, 0.7, 1.1, 1e-3, 3.3):
        for n in (3, 7, 10, 1000):
            L = np.full(n, np.float32(v), np.float64)
            Ls, Lsq = L.sum(), (L * L).sum()
            var = Lsq / n - (Ls / n) ** 2
            P, A = _set(np.tile([0.0, 0.0, 0.0, 1.0], (n, 1)), None, L)
            s = er.estimate_np(P, A)[0]["likelihood"]["sigma"]
            assert s == (0.0 if var < 0 else np.sqrt(var)) and np.isfinite(s)


def _angle_diagonal(C):
    """the covariance with the correlations between the three angles removed (still positive definite)"""
    C = np.array(C)
    for i, j in ((3, 4), (3, 5), (4, 5)):
        C[i, j] = C[j, i] = 0.0
    assert np.all(np.linalg.eigvalsh(C) > 0)
    return C


def _roundtrip_ok(r, pose, C, n, floor=1e-6):
    """Tbm within 5 standard errors of `pose` in its own frame, and the covariance within 5 standard errors of C; components without
    variance get an absolute floor -> (ok, worst ratio)"""
    T = np.zeros((), synth.TRANSFORM_DTYPE)
    T["t"], T["R"] = r["position"], r["orientation"]
    off = er.deviation(pose, T.reshape(1))[0]
    se_mean = np.sqrt(np.diag(C) / n)
    d = np.sqrt(np.diag(C))
    se_cov = np.sqrt((np.outer(d * d, d * d) + C * C) / n)
    Cm = r["covariance"].reshape(6, 6)
    ratios = np.concatenate([np.where(se_mean > 0, np.abs(off) / np.maximum(se_mean, 1e-300), np.abs(off) / floor),
                             np.where(se_cov > 0, np.abs(Cm - C) / np.maximum(se_cov, 1e-300), np.abs(Cm - C) / floor).reshape(-1)])
    return bool(ratios.max() <= 5.0), float(ratios.max())


@pytest.mark.parametrize("cov", ["full", "rviz"])
def test_round_trip_through_init_samples(cov):
    """initSamples(pose, C) at 10^6 particles with equal weights gives back `pose` and C (decision E2 in the frame of quirk D13).  The full
    covariance keeps its translation and translation-angle correlations but not those between the angles: correlated Euler angles shift the
    Markley mean of the rotations by second-order terms (about C_pitch,yaw / 4 in the roll component), a property of the mean, not of the
    frame.  The map-frame alternative (t - Tbm.t, not rotated into Tbm) misses the full C."""
    C0, pose = _gauss_case()
    C = _angle_diagonal(C0) if cov == "full" else RVIZ_COV
    n = 1_000_000
    P, A = ref.init_gaussian(0, n, pose, C, seed=11)
    r, T, _ = er.estimate_np(P, A)
    ok, worst = _roundtrip_ok(r, pose, C, n)
    assert ok, worst
    assert 2.0 * np.arctan2(float(T["R"][2]), float(T["R"][3])) > 1.0          # the pose has a non-zero yaw (1.2 rad)
    if cov == "full":
        V = er.deviation(T, P)
        Vmap = np.concatenate([P["t"].astype(np.float64) - T["t"].astype(np.float64), V[:, 3:]], 1)
        rm = np.array(r, copy=True)
        rm["covariance"] = (Vmap.T @ Vmap / n).reshape(36)
        assert not _roundtrip_ok(rm, pose, C, n)[0]
        # and the correlated angles of the untouched covariance do move the mean, by far more than 5 standard errors
        P2, A2 = ref.init_gaussian(0, n, pose, C0, seed=11)
        assert not _roundtrip_ok(er.estimate_np(P2, A2)[0], pose, C0, n)[0]
    print(f"{cov}: worst ratio to the standard error {worst:.2f}")


def _psd_cases():
    rng = np.random.default_rng(8)
    out = []
    for _ in range(200):
        B = rng.normal(size=(4, 4))
        out.append(B @ B.T)
    for _ in range(50):
        u = rng.normal(size=4)
        out.append(rng.uniform(0.1, 10) * np.outer(u, u))                       # rank 1
    for _ in range(50):
        out.append(np.diag(rng.permutation([0.0, 1e-3, 0.5, 2.0]) * rng.uniform(0.5, 3)))
    for _ in range(50):                                                            # nearly degenerate top pair
        Q = np.linalg.qr(rng.normal(size=(4, 4)))[0]
        out.append(Q @ np.diag([1.0, 1.0 - 10.0 ** rng.uniform(-15, -6), 0.3, 0.1]) @ Q.T)
    out.append(np.zeros((4, 4)))
    out.append(np.eye(4))
    # the particle case: q q^T of quaternions about one rotation, weights summing to 1
    q = rng.normal(size=(1000, 4)) * [0.05, 0.05, 0.2, 1.0]
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w = rng.uniform(size=1000)
    out.append(np.einsum("n,ni,nj->ij", w / w.sum(), q, q))
    return out


def test_product_eigen_solver_matches_numpy():
    """the product's sym4_top_eigvec on the CPU returns a maximiser of q^T M q (>= lambda_max - tol, always), with unit length and the sign of
    decision E1; the angle to numpy's vector is checked where the eigen-gap allows it"""
    for it, M in enumerate(_psd_cases()):
        v, lam = er.product_eigvec(M)
        vn, ln = er.top_eigvec(M)
        lams = np.linalg.eigvalsh(M)
        norm = max(np.abs(lams).max(), 1e-300)
        tol = 64 * np.finfo(np.float64).eps * norm
        assert abs(np.linalg.norm(v) - 1.0) <= 1e-12, it
        assert v @ M @ v >= ln - tol, (it, v @ M @ v, ln)
        assert abs(lam - ln) <= tol, it
        assert np.array_equal(v, er.canonical(v)), it
        gap = lams[-1] - lams[-2]
        if gap > 1e-8 * norm:
            ang = np.linalg.norm(v - np.sign(v @ vn) * vn)                          # chord: ~ the angle, without arccos's loss near 1
            assert ang <= 64 * np.finfo(np.float64).eps * norm / gap + 1e-12, (it, ang)


def test_product_eigen_solver_nan_and_sign_rule():
    v, lam = er.product_eigvec(np.full((4, 4), np.nan))
    assert np.all(np.isnan(v)) and np.isnan(lam)
    M = np.diag([1.0, 2.0, 3.0, 4.0])
    M[0, 1] = M[1, 0] = np.inf
    assert np.all(np.isnan(er.product_eigvec(M)[0]))
    # w == 0: the first non-zero component is positive
    for u in ([0, -1, 0, 0], [-1, 0, 0, 0], [0, 0, -1, 0], [0.6, -0.8, 0, 0], [-0.6, 0.8, 0, 0]):
        u = np.asarray(u, np.float64)
        v, _ = er.product_eigvec(np.outer(u, u) * 3.0)
        assert np.abs(v - er.canonical(u)).max() <= 1e-15 and np.array_equal(v, er.canonical(v))


def test_product_deviation_matches_float64():
    """pf_deviation (float) against the float64 deviation: within a few float ulp of the translation's magnitude and of the angle"""
    C, pose = _gauss_case()
    P, _ = ref.init_gaussian(0, 20000, pose, _angle_diagonal(C), seed=2)
    for T in (pose, synth.make_transform((3.2, -6.9, 0.4), (0.05, -0.02, 1.15)), synth.make_transform((-20.0, 35.0, 1.0), (0.0, 0.0, -2.9))):
        v = er.product_deviation(T, P).astype(np.float64)
        d = er.deviation(T, P)
        tmag = np.abs(P["t"]).max() + np.abs(T["t"]).max()
        assert np.abs(v[:, :3] - d[:, :3]).max() <= 16 * EPS32 * tmag
        dang = np.abs(v[:, 3:] - d[:, 3:])
        dang = np.minimum(dang, 2 * np.pi - dang)                                 # +-pi wrap of roll / yaw
        assert dang.max() <= 8e-6, dang.max()
