"""TEST INFRASTRUCTURE ONLY: reference for the particle set initialisers (b2_pf_init_uniform / b2_pf_init_gaussian), a thin ctypes layer
over pf_init_ref/pf_init_ref.c.  That file compiles the oracle's source (oracle/oracle.c) in, so Philox4x32-10, euler_to_quat and the
Transform product are the oracle's own.  The library is compiled on first use into the per-user temporary directory of chain_ref."""
import ctypes as C
import os

import numpy as np

from chain_ref import _build
from rmcl_b200.synth import PARTICLE_ATTR_DTYPE, TRANSFORM_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "pf_init_ref", "pf_init_ref.c")
        cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
        deps = [src, os.path.join(_ORACLE, "oracle.c"), os.path.join(_ORACLE, "oracle.h")]
        _lib = _build("pf_init_ref", deps, [cc, "-O2", "-fopenmp", "-ffp-contract=off", "-mavx2", "-mfma", "-fPIC", "-std=gnu11", "-shared", src, "-lm"])
        _lib.orc_pf_chol6.restype = C.c_int
    return _lib


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def chol6(cov):
    """-> (L (6,6) float32, 0) or (None, 1 + refused column)"""
    c = np.ascontiguousarray(cov, np.float64).reshape(36)
    L = np.zeros(36, np.float32)
    rc = lib().orc_pf_chol6(_p(c), _p(L))
    return (L.reshape(6, 6), 0) if rc == 0 else (None, rc)


def box32(bb_min, bb_max):
    return np.asarray(bb_min, np.float64).astype(np.float32), np.asarray(bb_max, np.float64).astype(np.float32)


def init_uniform(first, n, bb_min, bb_max, seed):
    """-> (poses TRANSFORM_DTYPE (n,), attrs PARTICLE_ATTR_DTYPE (n,)) of particles first .. first+n-1"""
    lo, hi = box32(bb_min, bb_max)
    P, A = np.zeros(n, TRANSFORM_DTYPE), np.zeros(n, PARTICLE_ATTR_DTYPE)
    lib().orc_pf_init_uniform(C.c_uint32(first), C.c_uint32(n), _p(lo), _p(hi), C.c_uint64(seed), _p(P), _p(A))
    return P, A


def init_normals(first, n, seed):
    """the (n, 6) N(0, I) draws of the Gaussian initialiser"""
    N = np.zeros((n, 6), np.float32)
    lib().orc_pf_init_normals(C.c_uint32(first), C.c_uint32(n), C.c_uint64(seed), _p(N))
    return N


def init_gaussian(first, n, pose, cov, seed, normals=None):
    """-> (poses, attrs); `normals` (n, 6) float32 replaces the draws.  Raises ValueError where the covariance is refused."""
    L, rc = chol6(cov)
    if L is None:
        raise ValueError(f"covariance refused at column {rc - 1}")
    T = np.ascontiguousarray(pose).reshape(())
    assert T.dtype.itemsize == 32
    if normals is not None:
        normals = np.ascontiguousarray(normals, np.float32).reshape(n, 6)
    P, A = np.zeros(n, TRANSFORM_DTYPE), np.zeros(n, PARTICLE_ATTR_DTYPE)
    lib().orc_pf_init_gaussian(C.c_uint32(first), C.c_uint32(n), _p(np.ascontiguousarray(L)), _p(T), C.c_uint64(seed), _p(normals), _p(P), _p(A))
    return P, A
