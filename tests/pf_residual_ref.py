"""TEST INFRASTRUCTURE ONLY: references for residual resampling (b2_pf_resample_residual, ResidualResamplerCPU::update,
rmcl_ros/src/rmcl/ResidualResamplerCPU.cpp:55-202).

* resample / parents / normals / stats: the C restatement with the library's keyed draws (pf_residual_ref/pf_residual_ref.c, which compiles
  the oracle's source in for Philox4x32-10, the Euler conversions and the Transform product).
* product_*: the product's per-element functions (rmcl_b200/csrc/kernels.cuh: residual_parent, residual_count, residual_normals,
  residual_copy) compiled for the CPU (pf_residual_ref/residual_emul.cu).
Both libraries are built on first use into the per-user temporary directory of chain_ref."""
import ctypes as C
import os

import numpy as np

from chain_ref import _build
from rmcl_b200.api import GladiatorConfig
from rmcl_b200.synth import PARTICLE_ATTR_DTYPE, TRANSFORM_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_CSRC = os.path.join(_ROOT, "rmcl_b200", "csrc")
_ref = None
_emul = None


def _ref_lib():
    global _ref
    if _ref is None:
        src = os.path.join(_HERE, "pf_residual_ref", "pf_residual_ref.c")
        cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
        deps = [src, os.path.join(_ROOT, "oracle", "oracle.c"), os.path.join(_ROOT, "oracle", "oracle.h")]
        _ref = _build("pf_residual_ref", deps, [cc, "-O2", "-fopenmp", "-ffp-contract=off", "-mavx2", "-mfma", "-fPIC", "-std=gnu11", "-shared", src, "-lm"])
        for f in ("orc_residual_parents", "orc_residual_normals", "orc_residual_stats", "orc_pf_resample_residual"):
            getattr(_ref, f).restype = None
    return _ref


def _emul_lib():
    global _emul
    if _emul is None:
        src = os.path.join(_HERE, "pf_residual_ref", "residual_emul.cu")
        deps = [src] + [os.path.join(_CSRC, f) for f in ("kernels.cuh", "icp_loop.cuh", "trace.cuh", "b2_math.cuh", "bvh8.h")] + \
               [os.path.join(_ROOT, "include", "rmcl_b200.h")]
        nvcc = os.environ.get("NVCC", "nvcc")
        _emul = _build("pf_residual_emul", deps, [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-fmad=false",
                                                  "-Xcompiler", "-fPIC,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared", src])
        for f in ("emul_residual_parents", "emul_residual_counts", "emul_residual_normals", "emul_residual_copies"):
            getattr(_emul, f).restype = None
    return _emul


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def d_max(n, M):
    return 16 * max(n, M)


def chunks(n, M, draws):
    """the number of chunks b2_pf_resample_residual runs to consume `draws` draws: sizes double from max(2n, 2^16) up to 2 max(n, M)"""
    nm = max(n, M)
    cap = min(2 * nm, 1 << 30)
    chunk, done, k = min(max(2 * n, 1 << 16), cap), 0, 0
    while done < draws:
        done += min(chunk, 16 * nm - done)
        chunk = min(2 * chunk, cap)
        k += 1
    return k


def stats(A):
    """-> (weight_sum summed in order, minimum from DBL_MAX, maximum from 0.0) of likelihood.mean in double"""
    A = np.ascontiguousarray(A)
    out = np.zeros(3)
    _ref_lib().orc_residual_stats(C.c_uint32(len(A)), _p(A), _p(out))
    return float(out[0]), float(out[1]), float(out[2])


def parents(seed, step, d0, count, n):
    out = np.zeros(count, np.uint32)
    _ref_lib().orc_residual_parents(C.c_uint64(seed), C.c_uint32(step), C.c_uint64(d0), C.c_uint64(count), C.c_uint32(n), _p(out))
    return out


def normals(seed, step, first, count):
    out = np.zeros((count, 6), np.float32)
    _ref_lib().orc_residual_normals(C.c_uint64(seed), C.c_uint32(step), C.c_uint32(first), C.c_uint32(count), _p(out))
    return out


def resample(P, A, n_new, cfg=None, seed=1234, step=0, first=0, n_local=None, S=None, L_max=None, N=None, trace=0):
    """The restated loop.  S / L_max default to stats(A) (the device passes its own); N (n_new, 6) float32 replaces the keyed normals.
    -> dict(n_particles, draws, P, A (n_local entries, untouched entries zero), parents, ins (the first `trace` draws))"""
    P, A = np.ascontiguousarray(P), np.ascontiguousarray(A)
    cfg = cfg or GladiatorConfig.defaults()
    S0, L_min, L_max0 = stats(A)
    S = S0 if S is None else S
    L_max = L_max0 if L_max is None else L_max
    n_local = n_new - first if n_local is None else n_local
    Pn, An = np.zeros(n_local, TRANSFORM_DTYPE), np.zeros(n_local, PARTICLE_ATTR_DTYPE)
    par, ins = np.zeros(max(trace, 1), np.uint32), np.zeros(max(trace, 1), np.uint64)
    res = np.zeros(2, np.uint64)
    if N is not None:
        N = np.ascontiguousarray(N, np.float32).reshape(n_new, 6)
    _ref_lib().orc_pf_resample_residual(C.c_uint32(len(P)), _p(P), _p(A), C.c_uint32(n_new), C.c_double(S), C.c_double(L_min), C.c_double(L_max), C.byref(cfg),
                                        C.c_uint64(seed), C.c_uint32(step), _p(N), C.c_uint32(first), C.c_uint32(n_local), _p(Pn), _p(An), _p(par), _p(ins),
                                        C.c_uint64(trace), _p(res))
    draws = int(res[1])
    k = min(trace, draws)
    return {"n_particles": int(res[0]), "draws": draws, "P": Pn, "A": An, "parents": par[:k], "ins": ins[:k]}


def product_parents(seed, step, d0, count, n):
    out = np.zeros(count, np.uint32)
    _emul_lib().emul_residual_parents(C.c_uint64(seed), C.c_uint32(step), C.c_uint64(d0), C.c_uint64(count), C.c_uint32(n), _p(out))
    return out


def product_counts(L, S, M):
    L = np.ascontiguousarray(L, np.float32)
    out = np.zeros(len(L), np.uint64)
    _emul_lib().emul_residual_counts(_p(L), C.c_uint64(len(L)), C.c_double(S), C.c_uint64(M), _p(out))
    return out


def product_normals(seed, step, first, count):
    out = np.zeros((count, 6), np.float32)
    _emul_lib().emul_residual_normals(C.c_uint64(seed), C.c_uint32(step), C.c_uint32(first), C.c_uint32(count), _p(out))
    return out


def product_copies(P, A, par, N, L_max, cfg=None):
    """copy i of parent par[i] with the normals N[i] -> (poses, attrs)"""
    cfg = cfg or GladiatorConfig.defaults()
    par = np.ascontiguousarray(par, np.uint32)
    N = np.ascontiguousarray(N, np.float32).reshape(len(par), 6)
    Pn, An = np.zeros(len(par), TRANSFORM_DTYPE), np.zeros(len(par), PARTICLE_ATTR_DTYPE)
    _emul_lib().emul_residual_copies(_p(np.ascontiguousarray(P)), _p(np.ascontiguousarray(A)), _p(par), _p(N), C.c_uint32(len(par)), C.c_double(L_max),
                                     C.byref(cfg), _p(Pn), _p(An))
    return Pn, An
