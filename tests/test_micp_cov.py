"""b2_micp_pose_covariance without a GPU: the product's finaliser (micp_cov_finalize, compiled for the CPU) against a float64 numpy restatement,
and the frame of the restated information (SURVEY appendix I)."""
import numpy as np
import pytest

import micp_cov_ref as ref

TAU, DV = 1e-3, 1e2


def _rot(rng):
    q = rng.normal(size=4)
    return ref.quat_mat(q)


def _sums_for(lam, L, W, R2, rng, weights=(1.0,)):
    """per-sensor sums whose weighted total has S H S = Q diag(lam) Q^T, length scale L and pair count W"""
    Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    Hs = Q @ np.diag(lam) @ Q.T
    S_inv = np.diag([1.0, 1.0, 1.0, L, L, L])
    H = S_inv @ Hs @ S_inv
    H = 0.5 * (H + H.T)
    total = ref.pack(H, R2, L * L * W, W)
    # split the total among the sensors: sensor k carries share_k / w_k, so that sum_k w_k s_k = total
    share = rng.uniform(0.5, 1.5, len(weights))
    share /= share.sum()
    sums = np.stack([total * (share[k] / weights[k]) for k in range(len(weights))])
    sums[:, 23] = np.round(sums[:, 23])            # pair counts are integers
    return sums


def _compare(got, want):
    assert int(got["n_degenerate"]) == int(want["n_degenerate"]) and int(got["degenerate_mask"]) == int(want["degenerate_mask"])
    assert (got["n_pairs"] == want["n_pairs"]).all()
    np.testing.assert_allclose(got["information"], want["information"], rtol=1e-15, atol=0)
    for f in ("residual_sq_sum", "weight_sum", "length_scale"):
        np.testing.assert_allclose(got[f], want[f], rtol=1e-14)
    assert np.isnan(got["sigma2"]) == np.isnan(want["sigma2"])
    lam_w = want["eigenvalues"]
    lmax = max(abs(float(lam_w[5])), 1e-300)
    assert np.abs(got["eigenvalues"] - lam_w).max() <= 1e-12 * lmax, (got["eigenvalues"], lam_w)
    Vg, Vw = got["eigenvectors"].reshape(6, 6), want["eigenvectors"].reshape(6, 6)
    if lam_w[5] > 0:
        # simple eigenvalues: the same vector (both follow the sign rule); a cluster of equal eigenvalues: the same span
        i = 0
        while i < 6:
            j = i + 1
            while j < 6 and lam_w[j] - lam_w[j - 1] <= 1e-6 * lmax:
                j += 1
            if j == i + 1:
                assert np.abs(Vg[i] - Vw[i]).max() <= 1e-8, (i, Vg[i], Vw[i])
            else:
                Pg, Pw = Vg[i:j].T @ Vg[i:j], Vw[i:j].T @ Vw[i:j]
                assert np.abs(Pg - Pw).max() <= 1e-8, (i, j)
            i = j
    else:
        assert (Vg == 0).all() and (got["eigenvalues"] == 0).all()
    Cg, Cw = got["covariance"], want["covariance"]
    assert (np.isnan(Cg) == np.isnan(Cw)).all()
    fin = ~np.isnan(Cw)
    if fin.any():
        assert np.linalg.norm(Cg[fin] - Cw[fin]) <= 1e-10 * np.linalg.norm(Cw[fin])


CASES = {
    "full":  dict(lam=[0.7, 3.0, 10.0, 42.0, 180.0, 1000.0], W=5000.0),
    "one_deg": dict(lam=[1e-5, 3.0, 10.0, 42.0, 180.0, 1000.0], W=5000.0),
    "rank5": dict(lam=[0.0, 3.0, 10.0, 42.0, 180.0, 1000.0], W=800.0),
    "rank4": dict(lam=[0.0, 0.0, 10.0, 42.0, 180.0, 1000.0], W=800.0),
    "rank3": dict(lam=[0.0, 0.0, 0.0, 42.0, 180.0, 1000.0], W=800.0),
    "w_le_6": dict(lam=[0.5, 3.0, 10.0, 42.0, 180.0, 1000.0], W=6.0),
    "repeated": dict(lam=[2.0, 2.0, 10.0, 10.0, 10.0, 1000.0], W=900.0),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("weights", [(1.0,), (0.5, 2.0), (1.0, 0.35, 0.6, 2.0)])
def test_finalize_matches_numpy(case, weights):
    """micp_cov_finalize (product, on the CPU) = the numpy restatement: eigenvalues within 1e-12 of lambda_max, eigenvectors equal under the sign
    rule (spans for repeated eigenvalues), the covariance within 1e-10, masks and counts exact"""
    c = CASES[case]
    for seed in range(5):
        rng = np.random.default_rng(100 * seed + len(weights))
        L = float(rng.uniform(0.5, 8.0))
        sums = _sums_for(np.array(c["lam"]) * float(rng.uniform(0.1, 100.0)), L, c["W"], float(rng.uniform(1.0, 50.0)), rng, weights)
        got = ref.product_finalize(sums, weights, TAU, DV)
        want = ref.finalize_np(sums, weights, TAU, DV)
        _compare(got, want)
        if case in ("rank5", "rank4", "rank3"):
            assert int(got["n_degenerate"]) == 6 - int(case[-1])
        if float(got["weight_sum"]) <= 6.0:
            assert np.isnan(got["sigma2"]) and np.isnan(got["covariance"]).all()


def test_finalize_no_pairs():
    """W == 0: zero information and eigen data, NaN covariance and sigma2, all six directions degenerate; also with pairs of weight 0"""
    for sums, w in ((np.zeros((1, ref.NACC)), (1.0,)), (ref.pack(np.eye(6), 1.0, 1.0, 100.0)[None], (0.0,))):
        got = ref.product_finalize(sums, w, TAU, DV)
        _compare(got, ref.finalize_np(sums, w, TAU, DV))
        assert (got["information"] == 0).all() and (got["eigenvalues"] == 0).all() and (got["eigenvectors"] == 0).all()
        assert np.isnan(got["covariance"]).all() and np.isnan(got["sigma2"])
        assert int(got["n_degenerate"]) == 6 and int(got["degenerate_mask"]) == 0x3F
        assert int(got["n_pairs"][0]) == int(sums[0, 23])


def test_degenerate_variance_units():
    """a degenerate direction gets degenerate_variance m^2 along translation and degenerate_variance / L^2 rad^2 along rotation"""
    L = 4.0
    H = np.diag([100.0, 100.0, 0.0, 100.0 * L * L, 100.0 * L * L, 0.0])          # z and yaw carry no information
    got = ref.product_finalize(ref.pack(H, 10.0, L * L * 1000.0, 1000.0)[None], (1.0,), TAU, DV)
    C = got["covariance"].reshape(6, 6)
    assert int(got["degenerate_mask"]) == 0b11 and int(got["n_degenerate"]) == 2          # the two smallest eigenvalues
    np.testing.assert_allclose([C[2, 2], C[5, 5]], [DV, DV / (L * L)], rtol=1e-12)
    sigma2 = 10.0 / (1000.0 - 6.0)
    np.testing.assert_allclose([C[0, 0], C[3, 3]], [sigma2 / 100.0, sigma2 / (100.0 * L * L)], rtol=1e-12)


def test_information_moves_with_the_reference_frame():
    """Restatement property: moving the reference frame by X = (R_x, t_x) (Tbo_ref' = Tbo_ref * X) turns H into A H A^T with
    A = [[R_x^T, 0], [-R_x^T [t_x]x, R_x^T]]; this pins the frame and the (x y z roll pitch yaw) order of the restated information"""
    rng = np.random.default_rng(7)
    Tbo_ref, Tbo, Tsb, Tpre = (_transform(_rot(rng), rng.normal(size=3)) for _ in range(4))
    n = 500
    d = rng.normal(size=(n, 3)) * 5.0
    N = rng.normal(size=(n, 3)); N /= np.linalg.norm(N, axis=1, keepdims=True)
    r = rng.normal(size=n) * 0.05
    H0 = ref.information_np(d, N, r, *ref.frames(Tbo_ref, Tbo, Tsb, Tpre))[0]
    Rx, tx = _rot(rng), rng.normal(size=3)
    X = _transform(Rx, tx)
    moved = _compose(Tbo_ref, X)
    H1 = ref.information_np(d, N, r, *ref.frames(moved, Tbo, Tsb, Tpre))[0]
    Rx = ref.quat_mat(X["R"])                                                    # the rotation the record holds
    tx = np.asarray(X["t"], np.float64)
    tx_cross = np.array([[0, -tx[2], tx[1]], [tx[2], 0, -tx[0]], [-tx[1], tx[0], 0]])
    A = np.block([[Rx.T, np.zeros((3, 3))], [-Rx.T @ tx_cross, Rx.T]])
    want = A @ H0 @ A.T
    assert np.abs(H1 - want).max() <= 1e-5 * np.abs(want).max()
    assert np.allclose(np.trace(H0[:3, :3]), n)                                 # unit normals: the translation block's trace is the pair count


def _transform(R, t):
    from scipy.spatial.transform import Rotation
    T = np.zeros((), ref.TRANSFORM)
    T["R"] = Rotation.from_matrix(R).as_quat().astype(np.float32)
    T["t"] = np.asarray(t, np.float32)
    return T


def _compose(A, B):
    """A * B in float64, rounded to float"""
    Ra, Rb = ref.quat_mat(A["R"]), ref.quat_mat(B["R"])
    return _transform(Ra @ Rb, Ra @ np.asarray(B["t"], np.float64) + np.asarray(A["t"], np.float64))


def test_pretransform_and_gate_are_the_loops():
    """the emulated pre-transform is Tso * T_onew_oold * Tos of float Transforms, and the gate accepts exactly |r| < max_dist among the masked pairs"""
    rng = np.random.default_rng(3)
    Tbo, Tsb, Td = (_transform(_rot(rng), rng.normal(size=3) * 0.1) for _ in range(3))
    Tpre = ref.product_pretransform(Tbo, Tsb, Td)
    Tos = _compose(Tbo, Tsb)
    R = ref.quat_mat(Tos["R"])
    want = R.T @ ref.quat_mat(Td["R"]) @ R
    assert np.abs(ref.quat_mat(Tpre["R"]) - want).max() < 1e-5
    n = 2000
    d = rng.normal(size=(n, 3)).astype(np.float32)
    I = rng.normal(size=(n, 3)).astype(np.float32)
    N = rng.normal(size=(n, 3)); N = (N / np.linalg.norm(N, axis=1, keepdims=True)).astype(np.float32)
    dm, hits = (rng.random(n) < 0.9).astype(np.uint8), (rng.random(n) < 0.9).astype(np.uint8)
    ok, r = ref.product_gate(Tpre, d, dm, I, N, hits, 0.5)
    Rp, tp = ref.quat_mat(Tpre["R"]), np.asarray(Tpre["t"], np.float64)
    r64 = ((I - (d @ Rp.T + tp)) * N).sum(1)
    clear = np.abs(np.abs(r64) - 0.5) > 1e-4
    assert (ok[clear] == ((dm > 0) & (hits > 0) & (np.abs(r64) < 0.5))[clear]).all()
    assert np.abs(r[ok] - r64[ok]).max() < 1e-4
