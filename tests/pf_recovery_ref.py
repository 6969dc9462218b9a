"""TEST INFRASTRUCTURE ONLY: references for the recovery (b2_pf_recovery_observe / b2_pf_recovery_inject, PCDSensorUpdaterB200.recovery*).

* RefRecovery.inject: the C restatement of decision, candidates and acceptance (pf_recovery_ref/pf_recovery_ref.c) over the surface rule of
  pf_surface_ref.c and the oracle's closest hit.
* ProductRecovery.inject / product_filter: the product's pf_recovery_one and pf_recovery_filter (rmcl_b200/csrc/kernels.cuh) compiled for
  the CPU over the product's host-built BVH (pf_recovery_ref/recovery_emul.cu).
* filter64: the record's recurrence transcribed in float64 Python.
Both libraries are built on first use into the per-user temporary directory of chain_ref."""
import ctypes as C
import math
import os

import numpy as np

from chain_ref import _build
from rmcl_b200.synth import RECOVERY_STATE_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_CSRC = os.path.join(_ROOT, "rmcl_b200", "csrc")
_ref = None
_emul = None


def _ref_lib():
    global _ref
    if _ref is None:
        src = os.path.join(_HERE, "pf_recovery_ref", "pf_recovery_ref.c")
        cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
        deps = [src, os.path.join(_HERE, "pf_surface_ref", "pf_surface_ref.c"), os.path.join(_ROOT, "oracle", "oracle.c"), os.path.join(_ROOT, "oracle", "oracle.h")]
        _ref = _build("pf_recovery_ref", deps, [cc, "-O2", "-fopenmp", "-ffp-contract=off", "-mavx2", "-mfma", "-fPIC", "-std=gnu11", "-shared", src, "-lm"])
        _ref.orc_scene_create.restype = C.c_void_p
        _ref.orc_scene_destroy.argtypes = [C.c_void_p]
        _ref.orc_pf_recovery.restype = None
    return _ref


def _emul_lib():
    global _emul
    if _emul is None:
        src = os.path.join(_HERE, "pf_recovery_ref", "recovery_emul.cu")
        deps = [src] + [os.path.join(_CSRC, f) for f in ("kernels.cuh", "icp_loop.cuh", "trace.cuh", "b2_math.cuh", "bvh8.h", "bvh_build.cpp")] + \
               [os.path.join(_ROOT, "include", "rmcl_b200.h")]
        nvcc = os.environ.get("NVCC", "nvcc")
        _emul = _build("pf_recovery_emul", deps, [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-fmad=false",
                                                  "-Xcompiler", "-fPIC,-fopenmp,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared", src,
                                                  os.path.join(_CSRC, "bvh_build.cpp"), "-lgomp"])
        _emul.emul_recovery_scene.restype = C.c_void_p
        _emul.emul_recovery_scene_free.argtypes = [C.c_void_p]
        _emul.emul_pf_recovery.restype = None
        _emul.emul_recovery_filter.restype = None
    return _emul


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _mesh(V, F):
    return np.ascontiguousarray(V, np.float32).reshape(-1, 3), np.ascontiguousarray(F, np.uint32).reshape(-1, 3)


def box32(bb_min, bb_max):
    return np.asarray(bb_min, np.float64).astype(np.float32), np.asarray(bb_max, np.float64).astype(np.float32)


class _Scene:
    def inject(self, P, A, p, bb_min, bb_max, surface=None, max_tries=16, seed=1234, step=0, first=0):
        """-> (poses, attrs, (n_replaced, n_failed)) after the injection with probability p; the inputs are not changed"""
        P, A = np.array(P, copy=True), np.array(A, copy=True)
        lo, hi = box32(bb_min, bb_max)
        counts = np.zeros(2, np.uint64)
        self._run(surface, first, len(P), float(p), lo, hi, max_tries, seed, step, P, A, counts)
        return P, A, (int(counts[0]), int(counts[1]))


class RefRecovery(_Scene):
    """the C restatement over the oracle's scene"""

    def __init__(self, V, F):
        self.V, self.F = _mesh(V, F)
        self._s = _ref_lib().orc_scene_create(_p(self.V), C.c_uint32(len(self.V)), _p(self.F), C.c_uint32(len(self.F)))
        assert self._s

    def __del__(self):
        if getattr(self, "_s", None):
            _ref_lib().orc_scene_destroy(self._s)

    def _run(self, surface, first, n, p, lo, hi, max_tries, seed, step, P, A, counts):
        _ref_lib().orc_pf_recovery(C.c_void_p(self._s) if surface is not None else None, C.byref(surface) if surface is not None else None, C.c_uint32(first),
                                   C.c_uint32(n), C.c_double(p), _p(lo), _p(hi), C.c_uint32(max_tries), C.c_uint64(seed), C.c_uint32(step), _p(P), _p(A), _p(counts))


class ProductRecovery(_Scene):
    """the product's pf_recovery_one on the CPU"""

    def __init__(self, V, F):
        self.V, self.F = _mesh(V, F)
        self._s = _emul_lib().emul_recovery_scene(_p(self.V), C.c_uint32(len(self.V)), _p(self.F), C.c_uint32(len(self.F)))
        assert self._s

    def __del__(self):
        if getattr(self, "_s", None):
            _emul_lib().emul_recovery_scene_free(self._s)

    def _run(self, surface, first, n, p, lo, hi, max_tries, seed, step, P, A, counts):
        _emul_lib().emul_pf_recovery(C.c_void_p(self._s), C.byref(surface) if surface is not None else None, C.c_uint32(first), C.c_uint32(n), C.c_double(p),
                                     _p(lo), _p(hi), C.c_uint32(max_tries), C.c_uint64(seed), C.c_uint32(step), _p(P), _p(A), _p(counts))


def product_filter(S, n, alpha_slow, alpha_fast, state):
    """the product's pf_recovery_filter on a copy of `state` (RECOVERY_STATE_DTYPE)"""
    st = np.array(state, RECOVERY_STATE_DTYPE, copy=True).reshape(())
    _emul_lib().emul_recovery_filter(C.c_double(S), C.c_uint32(n), C.c_double(alpha_slow), C.c_double(alpha_fast), _p(st))
    return st


def filter64(S, n, alpha_slow, alpha_fast, state):
    """float64 transcription of the recurrence: -> the new (w_avg, w_slow, w_fast, p_inject)"""
    w_avg = S / n
    _, w_slow, w_fast, p = (float(state[k]) for k in ("w_avg", "w_slow", "w_fast", "p_inject"))
    if math.isfinite(w_avg) and w_avg >= 0.0:
        w_slow = w_avg if w_slow == 0.0 else w_slow + alpha_slow * (w_avg - w_slow)
        w_fast = w_avg if w_fast == 0.0 else w_fast + alpha_fast * (w_avg - w_fast)
        p = max(0.0, 1.0 - w_fast / w_slow) if w_slow > 0.0 else 0.0
    return w_avg, w_slow, w_fast, p
