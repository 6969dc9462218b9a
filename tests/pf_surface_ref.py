"""TEST INFRASTRUCTURE ONLY: references for the surface constraint (b2_pf_project_to_surface, PCDSensorUpdaterB200.projectToSurface).

* RefScene.project: the C restatement of the rule (pf_surface_ref/pf_surface_ref.c) over the oracle's closest hit, brute force or BVH.
* ProductScene.project: the product's pf_surface_one (rmcl_b200/csrc/kernels.cuh) compiled for the CPU over the product's host-built BVH
  (pf_surface_ref/surface_emul.cu).
* quat_rotate64 / quat_mul64: float64 quaternion helpers for the geometric checks.
Both libraries are built on first use into the per-user temporary directory of chain_ref."""
import ctypes as C
import os

import numpy as np

from chain_ref import _build
from rmcl_b200.api import SurfaceConfig

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_CSRC = os.path.join(_ROOT, "rmcl_b200", "csrc")
_ref = None
_emul = None


def _ref_lib():
    global _ref
    if _ref is None:
        src = os.path.join(_HERE, "pf_surface_ref", "pf_surface_ref.c")
        cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
        deps = [src, os.path.join(_ROOT, "oracle", "oracle.c"), os.path.join(_ROOT, "oracle", "oracle.h")]
        _ref = _build("pf_surface_ref", deps, [cc, "-O2", "-fopenmp", "-ffp-contract=off", "-mavx2", "-mfma", "-fPIC", "-std=gnu11", "-shared", src, "-lm"])
        _ref.orc_scene_create.restype = C.c_void_p
        _ref.orc_scene_destroy.argtypes = [C.c_void_p]
        _ref.orc_pf_surface.restype = None
    return _ref


def _emul_lib():
    global _emul
    if _emul is None:
        src = os.path.join(_HERE, "pf_surface_ref", "surface_emul.cu")
        deps = [src] + [os.path.join(_CSRC, f) for f in ("kernels.cuh", "icp_loop.cuh", "trace.cuh", "b2_math.cuh", "bvh8.h", "bvh_build.cpp")] + \
               [os.path.join(_ROOT, "include", "rmcl_b200.h")]
        nvcc = os.environ.get("NVCC", "nvcc")
        _emul = _build("pf_surface_emul", deps, [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-fmad=false",
                                                 "-Xcompiler", "-fPIC,-fopenmp,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared", src,
                                                 os.path.join(_CSRC, "bvh_build.cpp"), "-lgomp"])
        _emul.emul_surface_scene.restype = C.c_void_p
        _emul.emul_surface_scene_free.argtypes = [C.c_void_p]
        _emul.emul_pf_surface.restype = None
    return _emul


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _mesh(V, F):
    V = np.ascontiguousarray(V, np.float32).reshape(-1, 3)
    F = np.ascontiguousarray(F, np.uint32).reshape(-1, 3)
    return V, F


class RefScene:
    """the C restatement over the oracle's scene"""

    def __init__(self, V, F):
        self.V, self.F = _mesh(V, F)
        self._s = _ref_lib().orc_scene_create(_p(self.V), C.c_uint32(len(self.V)), _p(self.F), C.c_uint32(len(self.F)))
        assert self._s

    def __del__(self):
        if getattr(self, "_s", None):
            _ref_lib().orc_scene_destroy(self._s)

    def project(self, P, A, cfg=None, brute=0):
        """-> (poses, attrs) after the rule; the inputs are not changed"""
        P, A = np.array(P, copy=True), np.array(A, copy=True)
        _ref_lib().orc_pf_surface(C.c_void_p(self._s), C.c_uint32(len(P)), _p(P), _p(A), C.byref(cfg or SurfaceConfig.defaults()), C.c_int(int(brute)))
        return P, A


class ProductScene:
    """the product's pf_surface_one on the CPU"""

    def __init__(self, V, F):
        self.V, self.F = _mesh(V, F)
        self._s = _emul_lib().emul_surface_scene(_p(self.V), C.c_uint32(len(self.V)), _p(self.F), C.c_uint32(len(self.F)))
        assert self._s

    def __del__(self):
        if getattr(self, "_s", None):
            _emul_lib().emul_surface_scene_free(self._s)

    def project(self, P, A, cfg=None):
        P, A = np.array(P, copy=True), np.array(A, copy=True)
        _emul_lib().emul_pf_surface(C.c_void_p(self._s), _p(P), _p(A), C.c_uint32(len(P)), C.byref(cfg or SurfaceConfig.defaults()))
        return P, A


def quat_rotate64(q, v):
    """rotate v (n, 3) by unit quaternions q (n, 4, x y z w) in float64"""
    q = np.asarray(q, np.float64)
    v = np.asarray(v, np.float64)
    u, w = q[..., :3], q[..., 3:4]
    return v + 2.0 * np.cross(u, np.cross(u, v) + w * v)


def quat_mul64(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    ax, ay, az, aw = np.moveaxis(a, -1, 0)
    bx, by, bz, bw = np.moveaxis(b, -1, 0)
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], -1)
