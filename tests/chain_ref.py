"""TEST INFRASTRUCTURE ONLY: references for chained MICP-L corrections (b2_micp_correct).

* oracle_progress / oracle_chain: convergence progress (micp_localization.cpp:988-1007) as a C restatement (chain_ref/progress_ref.c) and
  the chain of correct() (:847-854) as a loop over the oracle's multi-sensor correctOnce (oracle/: orc_micp_correct_once_multi) fed with it.
* product_progress / product_gate: the product's own update (rmcl_b200/csrc/icp_loop.cuh) compiled for the CPU (chain_ref/progress_emul.cu).
* progress_np: a numpy restatement of the same update.
"""
import ctypes as C

import numpy as np

import native
from rmcl_b200.synth import CROSS_STATS_DTYPE as CROSS_STATS, TRANSFORM_DTYPE as TRANSFORM

# one b2_micp_step record (include/rmcl_b200.h)
MICP_STEP = np.dtype([("Tom_new", TRANSFORM), ("T_onew_oold", TRANSFORM), ("Cmerged_o", CROSS_STATS), ("convergence_progress", np.float64),
                      ("valid_measurements", np.uint32), ("total_measurements", np.uint32)])


_ref = None
_emul = None


def _ref_lib():
    global _ref
    if _ref is None:
        _ref = native.restatement("chain_ref/progress_ref.c")
        _ref.ref_micp_progress.restype = C.c_double
        _ref.ref_micp_progress.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]
    return _ref


def _emul_lib():
    global _emul
    if _emul is None:
        _emul = native.emulator()
        _emul.emul_micp_progress.restype = C.c_double
        _emul.emul_micp_progress.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]
        _emul.emul_adaptive_max_dist.restype = C.c_float
        _emul.emul_adaptive_max_dist.argtypes = [C.c_float, C.c_float, C.c_double]
    return _emul


def _tf(a):
    a = np.ascontiguousarray(np.asarray(a).reshape(()))
    assert a.dtype.itemsize == 32, a.dtype
    return a


def oracle_progress(po, Tom, T_onew_oold, n_meas, valid, adaptive=True):
    """C restatement of :988-1007 on T_onew_map = Tom * T_onew_oold from the oracle's Transform product"""
    T = _tf(po.transform_mul(_tf(Tom), _tf(T_onew_oold)))
    return float(_ref_lib().ref_micp_progress(T.ctypes.data, int(n_meas), int(valid), int(bool(adaptive))))


def product_progress(Tom, T_onew_oold, n_meas, valid, adaptive=True):
    """the product's micp_progress (icp_loop.cuh) on the CPU"""
    a, b = _tf(Tom), _tf(T_onew_oold)
    return float(_emul_lib().emul_micp_progress(a.ctypes.data, b.ctypes.data, int(n_meas), int(valid), int(bool(adaptive))))


def product_gate(max_dist, max_dist_min, cp):
    """the product's icp_adaptive_max_dist (icp_loop.cuh) on the CPU"""
    return float(_emul_lib().emul_adaptive_max_dist(max_dist, max_dist_min, cp))


def progress_np(po, Tom, T_onew_oold, n_meas, valid, adaptive=True):
    """numpy restatement of micp_localization.cpp:988-1007: float64 where the reference computes in double, rounded to float32 where it
    declares a float (trans_force, trans_progress, qscalar, rot_progress, the product of the two, adaption_rate).  T_onew_map = Tom * T_onew_oold
    (:972) is the oracle's float32 Transform product; R.dot(Identity) is w for finite quaternions."""
    if n_meas == 0 or not adaptive:
        return 0.0
    T = po.transform_mul(_tf(Tom), _tf(T_onew_oold))
    x, y, z = (np.float32(v) for v in T["t"])
    trans_force = np.sqrt(np.float32(np.float32(x * x + y * y) + z * z))
    with np.errstate(over="ignore"):                       # exp(10 |t|) = inf for |t| > 71 m: trans_progress 0, as in C
        trans_progress = np.float32(1.0 / np.exp(10.0 * np.float64(trans_force)))
    w = np.float32(T["R"][3])
    rot_progress = np.float32(w * w)
    match_ratio = np.float64(n_meas) / np.float64(valid)
    return float(np.float32(np.float64(np.float32(trans_progress * rot_progress)) * match_ratio))


def valid_measurements(sensors):
    """stats.valid_measurements (:866-871): the mask ones of all datasets, counted as unpackMessage counts them (mask > 0)"""
    return int(sum(int((np.asarray(sd["dataset_mask"]) > 0).sum()) for sd in sensors))


def oracle_chain(po, osc, sensors, Tom, n_corrections=3, iterations=5, convergence_progress=0.0, adaptive_max_dist=True, f64_accum=True):
    """correct() generalised to n_corrections (:847-854): each oracle correctOnce (orc_micp_correct_once_multi, sensors as for
    Scene.micp_correct_once_multi) at the Tom the previous one left and with the progress it computed (oracle_progress).
    -> (Tom, progress, steps) with steps a MICP_STEP record array, like rmcl_b200.micp_correct."""
    valid = valid_measurements(sensors)
    total = int(sum(len(np.asarray(sd["dataset_mask"]).reshape(-1)) for sd in sensors))
    steps = np.zeros(int(n_corrections), MICP_STEP)
    T, cp = np.array(_tf(Tom), copy=True), float(convergence_progress)
    for s in range(int(n_corrections)):
        Tn, Td, Cm = osc.micp_correct_once_multi(sensors, T, iterations, cp, f64_accum=f64_accum)
        cp = oracle_progress(po, T, Td, int(Cm["n_meas"]), valid, adaptive_max_dist)
        T = np.array(Tn, copy=True)                                                   # Tn is Tom when n_meas == 0 (:974-984)
        steps[s]["Tom_new"], steps[s]["T_onew_oold"], steps[s]["Cmerged_o"] = Tn, Td, Cm
        steps[s]["convergence_progress"], steps[s]["valid_measurements"], steps[s]["total_measurements"] = cp, valid, total
    return T, cp, steps
