"""TEST INFRASTRUCTURE ONLY: references for the MICP-L pose covariance (b2_micp_pose_covariance; SURVEY appendix I).

* finalize_np: a float64 numpy restatement of the finaliser (weights, scaling, numpy.linalg.eigh, the sign rule, the pseudo-inverse).
* frames / information_np: the Jacobian rows J = (n, q x n) of the accepted pairs in the reference body frame and their sums, in float64 from
  the float buffers.
* product_finalize / product_pretransform / product_gate: the product's own micp_cov_finalize, pre-transform and P2L gate
  (rmcl_b200/csrc/kernels.cuh) compiled for the CPU (micp_cov_ref/cov_emul.cu), built on first use into the per-user temporary directory of
  chain_ref."""
import ctypes as C
import os

import numpy as np

from chain_ref import _build

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_CSRC = os.path.join(_ROOT, "rmcl_b200", "csrc")
TRANSFORM = np.dtype([("R", np.float32, 4), ("t", np.float32, 3), ("stamp", np.uint32)])
# b2_micp_covariance (include/rmcl_b200.h)
COVARIANCE = np.dtype([("information", np.float64, 36), ("covariance", np.float64, 36), ("eigenvalues", np.float64, 6),
                       ("eigenvectors", np.float64, 36), ("sigma2", np.float64), ("residual_sq_sum", np.float64), ("weight_sum", np.float64),
                       ("length_scale", np.float64), ("n_pairs", np.uint64, 4), ("n_degenerate", np.uint32), ("degenerate_mask", np.uint32)])
assert COVARIANCE.itemsize == 984
NACC = 24
_UPPER = [(i, j) for i in range(6) for j in range(i, 6)]
_emul = None


def _emul_lib():
    global _emul
    if _emul is None:
        src = os.path.join(_HERE, "micp_cov_ref", "cov_emul.cu")
        deps = [src] + [os.path.join(_CSRC, f) for f in ("kernels.cuh", "icp_loop.cuh", "trace.cuh", "b2_math.cuh", "bvh8.h")] + \
               [os.path.join(_ROOT, "include", "rmcl_b200.h")]
        nvcc = os.environ.get("NVCC", "nvcc")
        _emul = _build("micp_cov_emul", deps, [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-fmad=false",
                                               "-Xcompiler", "-fPIC,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared", src])
        for f in ("emul_micp_cov_finalize", "emul_micp_cov_pretransform", "emul_micp_cov_gate"):
            getattr(_emul, f).restype = None
    return _emul


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _tf(a):
    a = np.ascontiguousarray(np.asarray(a).reshape(()))
    assert a.dtype.itemsize == 32, a.dtype
    return a


def pack(H, R2, Q2, W):
    """one sensor's 24 sums from its information H (6x6), sum r^2, sum |q|^2 and pair count"""
    return np.array([H[i, j] for i, j in _UPPER] + [R2, Q2, W], np.float64)


def unpack(s):
    H = np.zeros((6, 6))
    for e, (i, j) in enumerate(_UPPER):
        H[i, j] = H[j, i] = s[e]
    return H


def product_finalize(sums, weights, tau=1e-3, degenerate_variance=1e2):
    sums = np.ascontiguousarray(sums, np.float64).reshape(-1, NACC)
    w = np.ascontiguousarray(weights, np.float64).reshape(len(sums))
    out = np.zeros((), COVARIANCE)
    _emul_lib().emul_micp_cov_finalize(_p(sums), _p(w), C.c_uint32(len(sums)), C.c_double(tau), C.c_double(degenerate_variance), _p(out))
    return out


def product_pretransform(Tbo, Tsb, T_onew_oold):
    out = np.zeros((), TRANSFORM)
    _emul_lib().emul_micp_cov_pretransform(_p(_tf(Tbo)), _p(_tf(Tsb)), _p(_tf(T_onew_oold)), _p(out))
    return out


def product_gate(Tpre, d, dmask, I, N, hits, max_dist):
    """-> (accepted (bool), r (float32)) of the product's gate over the float buffers"""
    d, I, N = (np.ascontiguousarray(a, np.float32).reshape(-1, 3) for a in (d, I, N))
    dmask, hits = np.ascontiguousarray(dmask, np.uint8).reshape(-1), np.ascontiguousarray(hits, np.uint8).reshape(-1)
    n = len(d)
    ok, r = np.zeros(n, np.uint8), np.zeros(n, np.float32)
    _emul_lib().emul_micp_cov_gate(_p(_tf(Tpre)), C.c_uint32(n), _p(d), _p(dmask), _p(I), _p(N), _p(hits), C.c_float(max_dist), _p(ok), _p(r))
    return ok.astype(bool), r


def quat_mat(q):
    x, y, z, w = np.asarray(q, np.float64) / np.linalg.norm(np.asarray(q, np.float64))
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def frames(Tbo_ref, Tbo, Tsb, Tpre):
    """float64 (R_U, t_U, R_N): U = ~Tbo_ref * Tbo * Tsb takes a dataset point into the reference body frame, R_N = R_U R(Tpre)^T a model normal"""
    Rr, Rb, Rs = quat_mat(Tbo_ref["R"]), quat_mat(Tbo["R"]), quat_mat(Tsb["R"])
    tr, tb, ts = (np.asarray(T["t"], np.float64) for T in (Tbo_ref, Tbo, Tsb))
    RU = Rr.T @ Rb @ Rs
    tU = Rr.T @ (Rb @ ts + tb - tr)
    return RU, tU, RU @ quat_mat(Tpre["R"]).T


def information_np(d, N, r, RU, tU, RN):
    """float64 sums of the accepted pairs (d, N, r): -> (H 6x6, R2, Q2, W)"""
    d, N, r = np.asarray(d, np.float64).reshape(-1, 3), np.asarray(N, np.float64).reshape(-1, 3), np.asarray(r, np.float64).reshape(-1)
    q = d @ RU.T + tU
    n = N @ RN.T
    J = np.concatenate([n, np.cross(q, n)], 1)
    return J.T @ J, float((r * r).sum()), float((q * q).sum()), float(len(r))


def sign_rule(v):
    """largest-magnitude component positive (the first one on ties)"""
    m = int(np.argmax(np.abs(v)))
    return v if v[m] >= 0.0 else -v


def finalize_np(sums, weights, tau=1e-3, degenerate_variance=1e2):
    """the record of micp_cov_finalize, restated in float64 with numpy.linalg.eigh"""
    sums = np.asarray(sums, np.float64).reshape(-1, NACC)
    r = np.zeros((), COVARIANCE)
    H, R2, Q2, W = np.zeros((6, 6)), 0.0, 0.0, 0.0
    for k, (s, w) in enumerate(zip(sums, weights)):
        H += w * unpack(s)
        R2 += w * s[21]; Q2 += w * s[22]; W += w * s[23]
        r["n_pairs"][k] = int(s[23])
    r["information"] = H.reshape(36)
    r["residual_sq_sum"], r["weight_sum"] = R2, W
    r["sigma2"] = R2 / (W - 6.0) if W > 6.0 else np.nan
    if not W > 0.0:
        r["covariance"] = np.nan
        r["n_degenerate"], r["degenerate_mask"] = 6, 0x3F
        return r
    L = np.sqrt(Q2 / W)
    L = L if L > 0.0 else 1.0
    S = np.diag([1.0, 1.0, 1.0, 1.0 / L, 1.0 / L, 1.0 / L])
    lam, V = np.linalg.eigh(S @ H @ S)
    ev = np.stack([sign_rule(V[:, i]) for i in range(6)])
    deg = lam <= tau * lam[5]
    Cs = np.zeros((6, 6))
    for i in range(6):
        Cs += (degenerate_variance if deg[i] else r["sigma2"] / lam[i]) * np.outer(ev[i], ev[i])
    r["covariance"] = (S @ Cs @ S).reshape(36)
    r["eigenvalues"], r["eigenvectors"] = lam, ev.reshape(36)
    r["length_scale"] = L
    r["n_degenerate"], r["degenerate_mask"] = int(deg.sum()), int(sum(1 << i for i in range(6) if deg[i]))
    return r
