"""TEST INFRASTRUCTURE ONLY: references for KLD-sampling (b2_pf_resample_kld; Fox, IJRR 2003; SURVEY appendix G).

* resample / table / keys / bounds / prefix / parents: the C restatement (pf_kld_ref/pf_kld_ref.c, which compiles the residual restatement
  and through it the oracle's source in for Philox4x32-10, the normals and the copy).
* product_*: the product's per-element functions (rmcl_b200/csrc/kernels.cuh: kld_weight, kld_parent, kld_key, kld_bound, kld_stop)
  compiled for the CPU (pf_kld_ref/kld_emul.cu).
Both libraries are built on first use by native.py."""
import ctypes as C

import numpy as np

import native
from rmcl_b200.api import GladiatorConfig, KLDConfig
from rmcl_b200.synth import PARTICLE_ATTR_DTYPE, TRANSFORM_DTYPE

_ref = None
_emul = None


def _ref_lib():
    global _ref
    if _ref is None:
        _ref = native.restatement("pf_kld_ref/pf_kld_ref.c")
        for f in ("orc_kld_table", "orc_kld_keys", "orc_kld_bounds", "orc_kld_prefix", "orc_kld_parents", "orc_pf_resample_kld"):
            getattr(_ref, f).restype = None
        _ref.orc_kld_sectors.restype = C.c_uint32
        _ref.orc_kld_sectors.argtypes = [C.c_float]
    return _ref


def _emul_lib():
    global _emul
    if _emul is None:
        _emul = native.emulator()
        for f in ("emul_kld_prefix", "emul_kld_parents", "emul_kld_keys", "emul_kld_bounds", "emul_kld_stop"):
            getattr(_emul, f).restype = None
    return _emul


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def sectors(res_yaw):
    """K of res_yaw (0 when outside [1, 32768])"""
    return int(_ref_lib().orc_kld_sectors(float(res_yaw)))


def chunks(n_min, n_max, draws):
    """the number of chunks b2_pf_resample_kld runs to make `draws` draws: sizes double from max(n_min, 2^16) up to n_max draws in all"""
    c, done, k = min(max(n_min, 1 << 16), n_max), 0, 0
    while done < draws:
        done += min(c, n_max - done)
        c = min(2 * c, 1 << 30)
        k += 1
    return k


def table(K):
    out = np.zeros((K, 2), np.float32)
    _ref_lib().orc_kld_table(C.c_uint32(K), _p(out))
    return out


def keys(P, res_xy, res_z, K):
    P = np.ascontiguousarray(P)
    cs = table(K)
    out = np.zeros(len(P), np.uint64)
    _ref_lib().orc_kld_keys(_p(P), C.c_uint64(len(P)), C.c_float(res_xy), C.c_float(res_z), _p(cs), C.c_uint32(K), _p(out))
    return out


def bounds(k, epsilon, z, n_min):
    k = np.ascontiguousarray(k, np.uint64)
    out = np.zeros(len(k), np.uint64)
    _ref_lib().orc_kld_bounds(_p(k), C.c_uint64(len(k)), C.c_double(epsilon), C.c_double(z), C.c_uint32(n_min), _p(out))
    return out


def prefix(A, L_max):
    A = np.ascontiguousarray(A)
    out = np.zeros(len(A), np.uint64)
    _ref_lib().orc_kld_prefix(C.c_uint32(len(A)), _p(A), C.c_double(L_max), _p(out))
    return out


def parents(seed, step, d0, count, W):
    W = np.ascontiguousarray(W, np.uint64)
    out = np.zeros(count, np.uint32)
    _ref_lib().orc_kld_parents(C.c_uint64(seed), C.c_uint32(step), C.c_uint64(d0), C.c_uint64(count), _p(W), C.c_uint32(len(W)), _p(out))
    return out


def resample(P, A, n_max, kld=None, cfg=None, seed=1234, step=0, first=0, n_local=None, S=None, L_max=None):
    """The restated resampler.  S / L_max default to the residual restatement's statistics of A (the device passes its own).
    -> dict(n_particles, bins, P, A (n_local entries, untouched entries zero), parents, keys (of the draws made))"""
    import pf_residual_ref
    P, A = np.ascontiguousarray(P), np.ascontiguousarray(A)
    kld = kld or KLDConfig.defaults()
    cfg = cfg or GladiatorConfig.defaults()
    S0, L_min, L_max0 = pf_residual_ref.stats(A)
    S = S0 if S is None else S
    L_max = L_max0 if L_max is None else L_max
    n_local = n_max - first if n_local is None else n_local
    Pn, An = np.zeros(n_local, TRANSFORM_DTYPE), np.zeros(n_local, PARTICLE_ATTR_DTYPE)
    par, key = np.zeros(n_max, np.uint32), np.zeros(n_max, np.uint64)
    res = np.zeros(2, np.uint64)
    _ref_lib().orc_pf_resample_kld(C.c_uint32(len(P)), _p(P), _p(A), C.c_uint32(n_max), C.c_double(S), C.c_double(L_min), C.c_double(L_max), C.byref(cfg),
                                   C.byref(kld), C.c_uint64(seed), C.c_uint32(step), C.c_uint32(first), C.c_uint32(n_local), _p(Pn), _p(An), _p(par), _p(key),
                                   _p(res))
    k = int(res[0])
    return {"n_particles": k, "bins": int(res[1]), "P": Pn, "A": An, "parents": par[:k], "keys": key[:k]}


def product_prefix(L, L_max):
    L = np.ascontiguousarray(L, np.float32)
    out = np.zeros(len(L), np.uint64)
    _emul_lib().emul_kld_prefix(_p(L), C.c_uint32(len(L)), C.c_double(L_max), _p(out))
    return out


def product_parents(seed, step, d0, count, W):
    W = np.ascontiguousarray(W, np.uint64)
    out = np.zeros(count, np.uint32)
    _emul_lib().emul_kld_parents(C.c_uint64(seed), C.c_uint32(step), C.c_uint64(d0), C.c_uint64(count), _p(W), C.c_uint32(len(W)), _p(out))
    return out


def product_keys(P, res_xy, res_z, K, cs=None):
    P = np.ascontiguousarray(P)
    cs = table(K) if cs is None else np.ascontiguousarray(cs, np.float32)
    out = np.zeros(len(P), np.uint64)
    _emul_lib().emul_kld_keys(_p(P), C.c_uint64(len(P)), C.c_float(res_xy), C.c_float(res_z), _p(cs), C.c_uint32(K), _p(out))
    return out


def product_bounds(k, epsilon, z, n_min):
    k = np.ascontiguousarray(k, np.uint64)
    out = np.zeros(len(k), np.uint64)
    _emul_lib().emul_kld_bounds(_p(k), C.c_uint64(len(k)), C.c_double(epsilon), C.c_double(z), C.c_uint32(n_min), _p(out))
    return out


def product_stop(j, k, epsilon, z, n_min, n_max):
    j, k = np.ascontiguousarray(j, np.uint64), np.ascontiguousarray(k, np.uint64)
    out = np.zeros(len(j), np.uint8)
    _emul_lib().emul_kld_stop(_p(j), _p(k), C.c_uint64(len(j)), C.c_double(epsilon), C.c_double(z), C.c_uint32(n_min), C.c_uint64(n_max), _p(out))
    return out.astype(bool)
