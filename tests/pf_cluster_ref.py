"""TEST INFRASTRUCTURE ONLY: references for the filter's pose hypotheses (b2_pf_cluster_stats; SURVEY appendix H).

* neighbours / cluster / clusters: the C restatement (pf_cluster_ref/pf_cluster_ref.c: sorted keys, binary search, sequential union-find),
  fed the bin keys and integer weights of the KLD restatement (pf_kld_ref).
* product_neighbours / product_offsets: the product's kld_key_neighbour / kld_key_offset (rmcl_b200/csrc/kernels.cuh) compiled for the CPU
  (pf_cluster_ref/cluster_emul.cu).
Both libraries are built on first use by native.py."""
import ctypes as C

import numpy as np

import native
import pf_kld_ref

NONE_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)
NONE = np.uint32(0xFFFFFFFF)
_ref = None
_emul = None


def _ref_lib():
    global _ref
    if _ref is None:
        _ref = native.restatement("pf_cluster_ref/pf_cluster_ref.c")
        _ref.orc_cluster_neighbours.restype = None
        _ref.orc_pf_cluster.restype = None
    return _ref


def _emul_lib():
    global _emul
    if _emul is None:
        _emul = native.emulator()
        _emul.emul_cluster_neighbours.restype = None
        _emul.emul_cluster_offsets.restype = None
    return _emul


def _p(a):
    return C.c_void_p(a.ctypes.data)


def neighbours(keys, dx, dy, dz, ds, K, has_z):
    keys = np.ascontiguousarray(keys, np.uint64)
    out = np.zeros(len(keys), np.uint64)
    _ref_lib().orc_cluster_neighbours(_p(keys), C.c_uint64(len(keys)), C.c_int(dx), C.c_int(dy), C.c_int(dz), C.c_int(ds), C.c_uint32(K), C.c_int(has_z), _p(out))
    return out


def product_neighbours(keys, dx, dy, dz, ds, K, has_z):
    keys = np.ascontiguousarray(keys, np.uint64)
    out = np.zeros(len(keys), np.uint64)
    _emul_lib().emul_cluster_neighbours(_p(keys), C.c_uint64(len(keys)), C.c_int(dx), C.c_int(dy), C.c_int(dz), C.c_int(ds), C.c_uint32(K), C.c_int(has_z), _p(out))
    return out


def product_offsets(keys, K, has_z):
    keys = np.ascontiguousarray(keys, np.uint64)
    out = np.zeros((len(keys), 81 if has_z else 27), np.uint64)
    _emul_lib().emul_cluster_offsets(_p(keys), C.c_uint64(len(keys)), C.c_uint32(K), C.c_int(has_z), _p(out))
    return out


def make_key(ix, iy, iz, s):
    """the bin key of cell (ix, iy, iz) and yaw sector s"""
    return np.uint64((int(ix) + 524288) << 44 | (int(iy) + 524288) << 24 | (int(iz) + 128) << 16 | int(s))


def cluster(keys, w, K, has_z):
    """The restated clustering of particles with bin keys `keys` (NONE_KEY: no bin) and integer weights `w`.
    -> dict(labels, n_clusters, bins, n_clustered, weight_total, weight_int, key, cbins, members), the last four per cluster in rank order"""
    keys, w = np.ascontiguousarray(keys, np.uint64), np.ascontiguousarray(w, np.uint64)
    n = len(keys)
    labels = np.zeros(n, np.uint32)
    cw, ck, cb, cm = (np.zeros(max(n, 1), np.uint64) for _ in range(4))
    res = np.zeros(4, np.uint64)
    _ref_lib().orc_pf_cluster(C.c_uint32(n), _p(keys), _p(w), C.c_uint32(K), C.c_int(has_z), _p(labels), _p(cw), _p(ck), _p(cb), _p(cm), _p(res))
    m = int(res[0])
    return {"labels": labels, "n_clusters": m, "bins": int(res[1]), "n_clustered": int(res[2]), "weight_total": int(res[3]),
            "weight_int": cw[:m], "key": ck[:m], "cbins": cb[:m], "members": cm[:m]}


def weights(A, L_max):
    """the integer weights w_i = (uint64)((double)L_i / L_max * 2^32) of the KLD restatement"""
    W = pf_kld_ref.prefix(A, L_max)
    return np.diff(W, prepend=np.uint64(0))


def clusters(P, A, cfg, S=None, L_max=None):
    """The restated b2_pf_cluster_stats but for the records' stats.  S / L_max default to the residual restatement's statistics of A (the
    device passes its own).  None: the set is refused (0 clusters)."""
    import pf_residual_ref
    P, A = np.ascontiguousarray(P), np.ascontiguousarray(A)
    S0, L_min, L_max0 = pf_residual_ref.stats(A)
    S = S0 if S is None else S
    L_max = L_max0 if L_max is None else L_max
    if not (np.isfinite(S) and S > 0.0 and L_min >= 0.0):
        return None
    K = pf_kld_ref.sectors(cfg.res_yaw)
    return cluster(pf_kld_ref.keys(P, cfg.res_xy, cfg.res_z, K), weights(A, L_max), K, cfg.res_z > 0.0)
