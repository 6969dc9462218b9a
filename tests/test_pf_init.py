"""CPU tests of the reference for the particle set initialisers (tests/pf_init_ref): RmclNode::initSamplesUniform
(rmcl_ros/src/nodes/rmcl_localization.cpp:277-342) and RmclNode::initSamples(PoseWithCovarianceStamped) (:165-275).

The Cholesky factor is checked against numpy's, with the zero-variance rule (SURVEY quirk D14); the samples are checked for their
distribution: the uniform ones by a Kolmogorov-Smirnov test per free dimension, the Gaussian ones by their sample mean and covariance in the
frame of the message pose (quirk D13)."""
import numpy as np
import pytest
from scipy import stats

import pf_init_ref as ref
from rmcl_b200 import synth

RVIZ_COV = np.diag([0.25, 0.25, 0.0, 0.0, 0.0, 0.06853891909122467])     # rviz's /initialpose: z, roll and pitch without variance


def _spd(rng, scale=1.0):
    A = rng.normal(size=(6, 6))
    return scale * (A @ A.T / 6.0 + 0.05 * np.eye(6))


def _quat_mat(q):
    """(n, 4) x, y, z, w -> (n, 3, 3) float64"""
    x, y, z, w = (np.asarray(q, np.float64)[..., k] for k in range(4))
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)


def _euler(Rm):
    """ZYX Euler angles (roll, pitch, yaw) of rotation matrices (n, 3, 3)"""
    roll = np.arctan2(Rm[:, 2, 1], Rm[:, 2, 2])
    pitch = np.arcsin(np.clip(-Rm[:, 2, 0], -1.0, 1.0))
    yaw = np.arctan2(Rm[:, 1, 0], Rm[:, 0, 0])
    return np.stack([roll, pitch, yaw], 1)


def local_coords(P, pose):
    """Tlm^-1 * pose per particle -> (n, 6): t, then roll, pitch, yaw, in float64"""
    R0 = _quat_mat(np.asarray(pose["R"]).reshape(1, 4))[0]
    R0 = R0 / np.cbrt(np.linalg.det(R0))                     # the message quaternion is used as given; the test's is unit length
    t = (np.asarray(P["t"], np.float64) - np.asarray(pose["t"], np.float64).reshape(1, 3)) @ R0
    Rl = np.einsum("ji,njk->nik", R0, _quat_mat(P["R"]))
    return np.concatenate([t, _euler(Rl)], 1)


def _within_5se(X, C):
    """sample mean and covariance of X (n, 6) against 0 and C, within 5 standard errors entry by entry -> (ok, worst ratio)"""
    n = len(X)
    se_mean = np.sqrt(np.diag(C) / n)
    d = np.sqrt(np.diag(C))
    se_cov = np.sqrt((np.outer(d * d, d * d) + C * C) / n)
    m = X.mean(0)
    S = np.cov(X, rowvar=False)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.concatenate([np.where(se_mean > 0, np.abs(m) / se_mean, np.where(m == 0, 0, np.inf)),
                            np.where(se_cov > 0, np.abs(S - C) / se_cov, np.where(S == C, 0, np.inf)).reshape(-1)])
    return bool(r.max() <= 5.0), float(r.max())


def test_chol6_matches_numpy():
    rng = np.random.default_rng(1)
    for it in range(200):
        C = _spd(rng, scale=10.0 ** rng.uniform(-3, 2))
        L, rc = ref.chol6(C)
        assert rc == 0
        Ln = np.linalg.cholesky(C)
        assert np.abs(L - Ln).max() <= 2e-5 * np.abs(Ln).max(), it
        assert np.all(np.triu(L, 1) == 0)


def test_chol6_zero_variances_give_zero_columns():
    L, rc = ref.chol6(RVIZ_COV)
    assert rc == 0
    assert np.array_equal(L, np.diag(np.sqrt(np.diag(RVIZ_COV).astype(np.float32))))
    for diag in ([0, 1, 0, 2, 0, 3], [0] * 6, [1e-4, 0, 0, 0, 0, 0], [4, 0, 0, 0, 0, 0]):
        L, rc = ref.chol6(np.diag(diag))
        assert rc == 0 and np.array_equal(L, np.diag(np.sqrt(np.float32(diag))))
    # a zero variance between correlated components: the column is zero, the other rows are the factor of the rest
    C = _spd(np.random.default_rng(2))
    C[2, :] = 0.0
    C[:, 2] = 0.0
    L, rc = ref.chol6(C)
    assert rc == 0 and np.all(L[:, 2] == 0) and np.all(L[2, :] == 0)
    keep = [0, 1, 3, 4, 5]
    assert np.abs(L[np.ix_(keep, keep)] - np.linalg.cholesky(C[np.ix_(keep, keep)])).max() <= 1e-5
    # only the lower triangle is read
    U = np.array(RVIZ_COV)
    U[0, 5] = 7.0
    assert np.array_equal(ref.chol6(U)[0], ref.chol6(RVIZ_COV)[0])


def test_chol6_refusals():
    neg = np.array(RVIZ_COV)
    neg[1, 1] = -0.25
    assert ref.chol6(neg) == (None, 2)
    nan = np.array(RVIZ_COV)
    nan[3, 3] = np.nan
    assert ref.chol6(nan)[1] == 4
    nan_off = np.array(RVIZ_COV)
    nan_off[5, 1] = np.nan
    assert ref.chol6(nan_off)[1] == 2
    zero_cov = np.array(RVIZ_COV)
    zero_cov[4, 2] = zero_cov[2, 4] = 0.01                               # z has no variance but covaries with pitch
    assert ref.chol6(zero_cov) == (None, 3)
    inf = np.array(RVIZ_COV)
    inf[0, 0] = 1e300                                                     # finite double, infinite float
    assert ref.chol6(inf)[1] == 1


BOX_MIN = [-50.0, -20.0, 0.25, -0.5, 0.3, -np.pi]
BOX_MAX = [50.0, 30.0, 0.25, 0.5, 0.3, np.pi]


def test_uniform_in_box_and_uniform():
    n = 200_000
    P, A = ref.init_uniform(0, n, BOX_MIN, BOX_MAX, seed=7)
    lo, hi = ref.box32(BOX_MIN, BOX_MAX)
    t = P["t"]
    assert np.all(t >= lo[:3]) and np.all(t <= hi[:3])
    assert np.all(t[:, 2] == lo[2])                                      # degenerate dimension: exactly the bound
    ang = _euler(_quat_mat(P["R"]))
    assert np.all(ang >= lo[3:] - 2e-6) and np.all(ang <= hi[3:] + 2e-6)
    assert np.abs(ang[:, 1] - np.float64(lo[4])).max() <= 2e-6            # pitch fixed at 0.3
    for k, v in ((0, t[:, 0]), (1, t[:, 1]), (3, ang[:, 0]), (5, ang[:, 2])):
        ks = stats.kstest(np.asarray(v, np.float64), "uniform", args=(float(lo[k]), float(hi[k]) - float(lo[k])))
        assert ks.pvalue > 1e-3, (k, ks)
    assert np.all(A["likelihood"]["mean"] == 1.0) and np.all(A["likelihood"]["sigma"] == 0.0) and np.all(A["likelihood"]["n_meas"] == 0)
    assert np.all(A["state_sigma"] == 0.0) and np.all(P["stamp"] == 0)
    # the node's default box (rmcl_localization.hpp:153-154): z, roll and pitch exactly 0
    P, _ = ref.init_uniform(0, 10_000, [-50, -50, 0, 0, 0, -np.pi], [50, 50, 0, 0, 0, np.pi], seed=1)
    assert np.all(P["t"][:, 2] == 0) and np.all(P["R"][:, 0] == 0) and np.all(P["R"][:, 1] == 0)


def _gauss_case():
    """a full SPD covariance (variances 0.5 m^2 in t, 0.02 / 0.02 / 0.1 rad^2 in the angles, x widened 4x so that a rotated frame is
    visible) and a pose rotated 1.2 rad in yaw"""
    S = _spd(np.random.default_rng(5))
    d = np.sqrt(np.array([2.0, 0.5, 0.5, 0.02, 0.02, 0.1]) / np.diag(S))
    C = S * np.outer(d, d)
    assert np.all(np.linalg.eigvalsh(C) > 0) and np.abs(C - np.diag(np.diag(C))).max() > 0.01
    pose = synth.make_transform((3.0, -7.0, 0.5), (0.1, -0.05, 1.2))
    return C, pose


def test_gaussian_moments_in_the_pose_frame():
    """sample mean 0 and covariance C of Tlm^-1 * pose (t, Euler angles) within 5 standard errors; the same samples read in the map frame
    (t - t_pose, not rotated) miss C: the covariance acts in the pose frame (SURVEY quirk D13)"""
    C, pose = _gauss_case()
    n = 1_000_000
    P, A = ref.init_gaussian(0, n, pose, C, seed=11)
    X = local_coords(P, pose)
    ok, worst = _within_5se(X, C)
    assert ok, worst
    Xmap = np.concatenate([np.asarray(P["t"], np.float64) - np.asarray(pose["t"], np.float64).reshape(1, 3), X[:, 3:]], 1)
    assert not _within_5se(Xmap, C)[0]
    assert np.all(A["likelihood"]["mean"] == 1.0) and np.all(A["state_sigma"] == 0.0) and np.all(P["stamp"] == 0)


def test_gaussian_zero_variance_components_stay_exact():
    """rviz's covariance: z of the pose frame stays 0, so with an upright pose every particle keeps the pose's z, roll and pitch"""
    pose = synth.make_transform((1.0, 2.0, 0.0), (0.0, 0.0, 0.7))
    P, _ = ref.init_gaussian(0, 50_000, pose, RVIZ_COV, seed=3)
    assert np.all(np.isfinite(P["t"])) and np.all(np.isfinite(P["R"]))
    X = local_coords(P, pose)
    assert np.abs(X[:, 2]).max() <= 1e-6 and np.abs(X[:, 3:5]).max() <= 1e-6
    assert np.all(P["R"][:, 0] == 0) and np.all(P["R"][:, 1] == 0)


def test_given_normals_reproduce_the_draws():
    C, pose = _gauss_case()
    N = ref.init_normals(100, 5000, seed=9)
    a = ref.init_gaussian(100, 5000, pose, C, seed=9)
    b = ref.init_gaussian(100, 5000, pose, C, seed=12345, normals=N)
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    assert abs(float(N.mean())) < 0.02 and abs(float(N.std()) - 1.0) < 0.02


@pytest.mark.parametrize("kind", ["uniform", "gaussian"])
def test_shards_concatenate_to_the_whole(kind):
    C, pose = _gauss_case()

    def run(first, n):
        if kind == "uniform":
            return ref.init_uniform(first, n, BOX_MIN, BOX_MAX, seed=21)
        return ref.init_gaussian(first, n, pose, C, seed=21)
    whole = run(0, 10_007)
    cuts = [0, 1, 256, 3333, 10_006, 10_007]
    parts = [run(a, b - a) for a, b in zip(cuts[:-1], cuts[1:])]
    for k in (0, 1):
        assert np.concatenate([p[k] for p in parts]).tobytes() == whole[k].tobytes()
