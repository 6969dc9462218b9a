"""TEST INFRASTRUCTURE ONLY: references for the global search (b2_pf_global_search, PCDSensorUpdaterB200.globalSearch).

* poses / peaks / records: the C restatement of the definition (pf_search_ref/pf_search_ref.c).
* Product*: the product's functions (rmcl_b200/csrc/kernels.cuh) compiled for the CPU (pf_search_ref/search_emul.cu, the emulator library
  plus the search's functions): candidates with and without the surface rule, the peak rule, the ranking and the separation pass.
* host_result: the restatement applied to a score array -> what the call must return for it.
Both libraries are built on first use, with native.py's recipes."""
import ctypes as C
import os

import numpy as np

import native
from rmcl_b200.synth import TRANSFORM_DTYPE

_ref = None
_emul = None


def _ref_lib():
    global _ref
    if _ref is None:
        _ref = native.restatement("pf_search_ref/pf_search_ref.c")
        _ref.ref_search_poses.restype = None
        _ref.ref_search_peaks.restype = C.c_uint64
        _ref.ref_search_records.restype = C.c_uint32
    return _ref


def _emul_lib():
    global _emul
    if _emul is None:
        _emul = C.CDLL(native._build("search_emul", native._NVCC, native._NVCC_FLAGS +
                                     ["-Xcompiler", "-fPIC,-fopenmp,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared"],
                                     [os.path.join(native.TESTS, "pf_search_ref", "search_emul.cu"),
                                      os.path.join(native.ROOT, "rmcl_b200", "csrc", "bvh_build.cpp")], ["-lgomp"], ".so"))
        _emul.emul_scene_create.restype = C.c_void_p
        _emul.emul_search_candidates.restype = None
        _emul.emul_search_peaks.restype = None
        _emul.emul_search_records.restype = C.c_uint32
    return _emul


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _grid(cfg):
    return float(cfg.x0), float(cfg.y0), float(cfg.z0), float(cfg.step), int(cfg.nx), int(cfg.ny), int(cfg.n_yaw)


def poses(cfg):
    """the restatement's candidate poses in c order (no surface rule)"""
    x0, y0, z0, step, nx, ny, K = _grid(cfg)
    out = np.zeros(nx * ny * K, TRANSFORM_DTYPE)
    _ref_lib().ref_search_poses(C.c_float(x0), C.c_float(y0), C.c_float(z0), C.c_float(step), C.c_uint32(nx), C.c_uint32(ny), C.c_uint32(K), _p(out))
    return out


def peaks(scores, nx, ny, K):
    """-> (peak flags, n_valid, n_peaks) of the restatement"""
    s = np.ascontiguousarray(scores, np.float32)
    flags, nv = np.zeros(len(s), np.uint8), C.c_uint64()
    n = _ref_lib().ref_search_peaks(_p(s), C.c_uint32(nx), C.c_uint32(ny), C.c_uint32(K), _p(flags), C.byref(nv))
    return flags, int(nv.value), int(n)


def _records(lib_fn, scores, list_, cfg):
    s = np.ascontiguousarray(scores, np.float32)
    lst = np.ascontiguousarray(list_, np.uint32).copy()
    kept = np.zeros(max(1, int(cfg.max_records)), np.uint32)
    n = lib_fn(_p(s), _p(lst), C.c_uint64(len(lst)), C.c_float(cfg.x0), C.c_float(cfg.y0), C.c_float(cfg.step), C.c_uint32(cfg.nx), C.c_uint32(cfg.ny),
               C.c_uint32(cfg.n_yaw), C.c_uint32(cfg.max_records), C.c_float(cfg.min_separation_xy), C.c_float(cfg.min_separation_yaw), _p(kept))
    return kept[:n]


def records(scores, peak_list, cfg):
    """the restatement's ranking and separation over the candidates peak_list -> the kept c, rank order"""
    return _records(_ref_lib().ref_search_records, scores, peak_list, cfg)


def host_result(scores, cfg):
    """the restatement applied to a whole score array -> (dict(n_candidates, n_valid, n_peaks, n_records), kept c in rank order)"""
    flags, nv, npk = peaks(scores, cfg.nx, cfg.ny, cfg.n_yaw)
    kept = records(scores, np.flatnonzero(flags), cfg)
    return dict(n_candidates=len(scores), n_valid=nv, n_peaks=npk, n_records=len(kept)), kept


class ProductScene:
    """the product's candidate functions on the CPU over its host-built BVH (in this library)"""

    def __init__(self, verts, faces):
        self.verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
        self.faces = np.ascontiguousarray(faces, np.uint32).reshape(-1, 3)
        err = C.c_char_p()
        h = _emul_lib().emul_scene_create(_p(self.verts), C.c_uint32(len(self.verts)), _p(self.faces), C.c_uint32(len(self.faces)), C.byref(err))
        if not h:
            raise RuntimeError("emul BVH build failed: " + err.value.decode())
        self._h = C.c_void_p(h)

    def __del__(self):
        if getattr(self, "_h", None):
            _emul_lib().emul_scene_destroy(self._h)

    def candidates(self, cfg, surface=None, mode=1):
        """mode 1: per-cell probe + placement (what the device runs); 2: pf_surface_pose on every candidate -> (poses, valid)"""
        x0, y0, z0, step, nx, ny, K = _grid(cfg)
        out, valid = np.zeros(nx * ny * K, TRANSFORM_DTYPE), np.zeros(nx * ny * K, np.uint8)
        _emul_lib().emul_search_candidates(self._h, C.c_float(x0), C.c_float(y0), C.c_float(z0), C.c_float(step), C.c_uint32(nx), C.c_uint32(ny),
                                           C.c_uint32(K), C.c_int(0 if surface is None else mode), None if surface is None else C.byref(surface),
                                           _p(out), _p(valid))
        return out, valid.astype(bool)


def product_poses(cfg):
    """the product's search_pose over the grid (no map needed)"""
    x0, y0, z0, step, nx, ny, K = _grid(cfg)
    out, valid = np.zeros(nx * ny * K, TRANSFORM_DTYPE), np.zeros(nx * ny * K, np.uint8)
    _emul_lib().emul_search_candidates(None, C.c_float(x0), C.c_float(y0), C.c_float(z0), C.c_float(step), C.c_uint32(nx), C.c_uint32(ny), C.c_uint32(K),
                                       C.c_int(0), None, _p(out), _p(valid))
    return out


def product_peaks(scores, nx, ny, K):
    s = np.ascontiguousarray(scores, np.float32)
    flags = np.zeros(len(s), np.uint8)
    _emul_lib().emul_search_peaks(_p(s), C.c_uint32(nx), C.c_uint32(ny), C.c_uint32(K), _p(flags))
    return flags


def product_records(scores, peak_list, cfg):
    return _records(_emul_lib().emul_search_records, scores, peak_list, cfg)
