"""TEST INFRASTRUCTURE ONLY: references for the particle set's pose estimate (b2_pf_estimate_stats, RmclNode::estimateStats,
rmcl_ros/src/nodes/rmcl_localization.cpp:642-731).

* estimate_np: a float64 numpy model of estimateStats with the decisions recorded in SURVEY (E1-E4): likelihood statistics, the float
  AABB, the weighted Markley mean (numpy.linalg.eigh of sum w q q^T) rounded to a float Transform, and the covariance of (~Tbm * pose) about
  that Tbm.  Pass 2 can be fed another Tbm (the device's), so that a comparison isolates the float deviation arithmetic.
* product_eigvec / product_deviation: the product's own B2_DEV functions (rmcl_b200/csrc/kernels.cuh) compiled for the CPU
  (pf_estimate_ref/estimate_emul.cu), built on first use into the per-user temporary directory of chain_ref."""
import ctypes as C
import os

import numpy as np

from chain_ref import _build
from rmcl_b200.synth import PARTICLE_STATS_DTYPE, TRANSFORM_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(_HERE), "rmcl_b200", "csrc")
DBL_MAX = float(np.finfo(np.float64).max)
FLT_MAX = float(np.finfo(np.float32).max)
_emul = None


def _emul_lib():
    global _emul
    if _emul is None:
        src = os.path.join(_HERE, "pf_estimate_ref", "estimate_emul.cu")
        deps = [src] + [os.path.join(_CSRC, f) for f in ("kernels.cuh", "icp_loop.cuh", "trace.cuh", "b2_math.cuh", "bvh8.h")] + \
               [os.path.join(os.path.dirname(_HERE), "include", "rmcl_b200.h")]
        nvcc = os.environ.get("NVCC", "nvcc")
        _emul = _build("estimate_emul", deps, [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-fmad=false",
                                               "-Xcompiler", "-fPIC,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared", src])
        _emul.emul_sym4_top_eigvec.restype = None
        _emul.emul_pf_deviation.restype = None
    return _emul


def product_eigvec(M):
    """the product's sym4_top_eigvec on the CPU -> (v (4,), lambda)"""
    A = np.ascontiguousarray(M, np.float64).reshape(16)
    v, lam = np.zeros(4), np.zeros(1)
    _emul_lib().emul_sym4_top_eigvec(C.c_void_p(A.ctypes.data), C.c_void_p(v.ctypes.data), C.c_void_p(lam.ctypes.data))
    return v, float(lam[0])


def product_deviation(Tbm, P):
    """the product's pf_deviation on the CPU: (n, 6) float32 of (~Tbm * pose) as (t, roll, pitch, yaw)"""
    T = np.ascontiguousarray(np.asarray(Tbm).reshape(()))
    P = np.ascontiguousarray(P).reshape(-1)
    out = np.zeros((len(P), 6), np.float32)
    _emul_lib().emul_pf_deviation(C.c_void_p(T.ctypes.data), C.c_void_p(P.ctypes.data), C.c_uint32(len(P)), C.c_void_p(out.ctypes.data))
    return out


def qmul(a, b):
    ax, ay, az, aw = (a[..., i] for i in range(4))
    bx, by, bz, bw = (b[..., i] for i in range(4))
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], -1)


def qrot(q, v):
    p = np.concatenate([v, np.zeros(v.shape[:-1] + (1,))], -1)
    return qmul(qmul(q, p), q * np.array([-1.0, -1.0, -1.0, 1.0]))[..., :3]


def quat_to_euler(q):
    """the ZYX conversion of quat_to_euler (kernels.cuh) in float64, on (n, 4) x y z w -> (n, 3)"""
    x, y, z, w = (q[..., i] for i in range(4))
    roll = np.arctan2(2.0 * (w * x + y * z), 1.0 - 2.0 * (x * x + y * y))
    sinp = 2.0 * (w * y - z * x)
    pitch = np.where(np.abs(sinp) >= 1.0, np.copysign(np.pi / 2, sinp), np.arcsin(np.clip(sinp, -1.0, 1.0)))
    yaw = np.arctan2(2.0 * (w * z + x * y), 1.0 - 2.0 * (y * y + z * z))
    return np.stack([roll, pitch, yaw], -1)


def deviation(Tbm, P):
    """(~Tbm * pose) in float64 from the float records -> (n, 6): t, roll, pitch, yaw"""
    qb = np.asarray(Tbm["R"], np.float64).reshape(1, 4) * np.array([-1.0, -1.0, -1.0, 1.0])
    tb = np.asarray(Tbm["t"], np.float64).reshape(1, 3)
    q = np.asarray(P["R"], np.float64)
    t = np.asarray(P["t"], np.float64)
    d_q = qmul(np.broadcast_to(qb, q.shape), q)
    d_t = qrot(np.broadcast_to(qb, q.shape), t - tb)
    return np.concatenate([d_t, quat_to_euler(d_q)], 1)


def canonical(v):
    """sign of decision E1: w >= 0; when w == 0 the first non-zero component is positive"""
    v = np.array(v, np.float64)
    for i in (3, 0, 1, 2):
        if v[i] != 0.0:
            return v if v[i] > 0.0 else -v
    return v


def top_eigvec(M):
    lam, V = np.linalg.eigh(M)
    return canonical(V[:, -1]), float(lam[-1])


def estimate_np(P, A, Tbm_pass2=None):
    """-> (PARTICLE_STATS_DTYPE record, model's float Tbm, float64 internals dict) over all of P / A"""
    L = np.asarray(A["likelihood"]["mean"], np.float64)
    k = len(L)
    t = np.asarray(P["t"], np.float64)
    q = np.asarray(P["R"], np.float64)
    r = np.zeros((), PARTICLE_STATS_DTYPE)
    Ls, Lsq = float(L.sum()), float((L * L).sum())
    finite = L[~np.isnan(L)]
    r["likelihood"]["max"] = max(0.0, float(finite.max())) if len(finite) else 0.0
    r["likelihood"]["min"] = min(DBL_MAX, float(finite.min())) if len(finite) else DBL_MAX
    mean = Ls / k
    var = Lsq / k - mean * mean
    r["likelihood"]["mean"] = mean
    r["likelihood"]["sigma"] = 0.0 if var < 0.0 else np.sqrt(var)                 # decision E4
    r["shift"] = r["likelihood"]["min"]
    r["trans_bb_min"] = np.minimum(FLT_MAX, np.nanmin(t, 0)) if k else FLT_MAX
    r["trans_bb_max"] = np.maximum(-FLT_MAX, np.nanmax(t, 0)) if k else -FLT_MAX
    r["nparticles"] = k
    ok = Ls > 0.0 and np.isfinite(Ls)                                                # decision E3
    T = np.zeros((), TRANSFORM_DTYPE)
    if ok:
        w = L / Ls
        tm = (w[:, None] * t).sum(0)
        M = np.einsum("n,ni,nj->ij", w, q, q)
        qv, lam = top_eigvec(M)
    else:
        w = np.full(k, np.nan)
        tm, M, qv, lam = np.full(3, np.nan), np.full((4, 4), np.nan), np.full(4, np.nan), np.nan
    T["R"] = qv.astype(np.float32)
    T["t"] = tm.astype(np.float32)
    r["position"] = T["t"]
    r["orientation"] = T["R"]
    Tb = T if Tbm_pass2 is None else np.asarray(Tbm_pass2).reshape(())
    V = deviation(Tb, P)
    Cv = np.einsum("n,ni,nj->ij", w, V, V) if ok else np.full((6, 6), np.nan)
    r["covariance"] = Cv.reshape(36)
    return r, T, {"M": M, "lambda": lam, "q": qv, "t": tm, "w": w, "V": V, "L_sum": Ls, "L_sum_sq": Lsq}
