"""TEST INFRASTRUCTURE ONLY: references for b2_rcc_set_cloud_spherical (PointCloud2 -> spherical scan + dataset).

* convert: the C restatement of Pc2ToScanNode::convert + fillEmpty + the spherical unpackMessage (pc2_scan_ref/pc2_scan_ref.c, which
  compiles the oracle's source in for the Transform product), with the elevation rule and the atan2 precision as test-only arguments.
* product: the product's own per-point and per-cell functions (rmcl_b200/csrc/kernels.cuh) compiled for the CPU (pc2_scan_ref/scan_emul.cu),
  the points visited in any order.
Both libraries are built on first use into the per-user temporary directory of chain_ref."""
import ctypes as C
import os

import numpy as np

from chain_ref import _build
from rmcl_b200.api import _SphericalModel
from rmcl_b200.synth import TRANSFORM_DTYPE, make_transform

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_CSRC = os.path.join(_ROOT, "rmcl_b200", "csrc")
_ref = None
_emul = None

ELEV_3D = 1         # the reference's elevation rule phi = atan2(z, |p|) (SURVEY D21)
ATAN2F = 2          # float atan2f instead of FP64 atan2 rounded to float


def _ref_lib():
    global _ref
    if _ref is None:
        src = os.path.join(_HERE, "pc2_scan_ref", "pc2_scan_ref.c")
        cc = "/usr/bin/gcc" if os.access("/usr/bin/gcc", os.X_OK) else "gcc"
        deps = [src, os.path.join(_ROOT, "oracle", "oracle.c"), os.path.join(_ROOT, "oracle", "oracle.h")]
        _ref = _build("pc2_scan_ref", deps, [cc, "-O2", "-fopenmp", "-ffp-contract=off", "-mavx2", "-mfma", "-fPIC", "-std=gnu11", "-shared", src, "-lm"])
        _ref.ref_pc2_to_scan.restype = None
        _ref.ref_spherical_dirs.restype = None
    return _ref


def _emul_lib():
    global _emul
    if _emul is None:
        src = os.path.join(_HERE, "pc2_scan_ref", "scan_emul.cu")
        deps = [src] + [os.path.join(_CSRC, f) for f in ("kernels.cuh", "icp_loop.cuh", "trace.cuh", "b2_math.cuh", "bvh8.h")] + \
               [os.path.join(_ROOT, "include", "rmcl_b200.h")]
        nvcc = os.environ.get("NVCC", "nvcc")
        _emul = _build("scan_emul", deps, [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-fmad=false",
                                           "-Xcompiler", "-fPIC,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared", src])
        _emul.emul_scan_from_cloud.restype = None
    return _emul


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _model(m):
    return _SphericalModel(m.phi_min, m.phi_inc, m.phi_size, m.theta_min, m.theta_inc, m.theta_size, m.range_min, m.range_max)


def _cloud_args(cloud):
    f = {p.name: p for p in cloud.fields}
    buf = np.ascontiguousarray(np.asarray(cloud.data, np.uint8).reshape(-1))
    if buf.size == 0:
        buf = np.zeros(1, np.uint8)
    off = np.array([f[c].offset for c in "xyz"], np.uint32)
    return buf, off, int(f["x"].datatype == 8)


def _tf(T):
    T = np.ascontiguousarray(make_transform() if T is None else T).reshape(())
    assert T.dtype == TRANSFORM_DTYPE
    return T


def dirs(model):
    """(n, 3) float32 direction table of a spherical model, as set_model_spherical evaluates it"""
    sm = _model(model)
    d = np.zeros((model.phi_size * model.theta_size, 3), np.float32)
    _ref_lib().ref_spherical_dirs(C.byref(sm), _p(d))
    return d


def convert(cloud, model, T=None, flags=0):
    """-> dict(ranges (n,), points (n,3), mask (n,), cell / theta / phi per point (cell -1: skipped, outside the model or out of range))"""
    buf, off, f64 = _cloud_args(cloud)
    sm, T = _model(model), _tf(T)
    n, npts = model.phi_size * model.theta_size, int(cloud.width) * int(cloud.height)
    out = dict(ranges=np.zeros(n, np.float32), points=np.zeros((n, 3), np.float32), mask=np.zeros(n, np.uint8),
               cell=np.zeros(max(npts, 1), np.int64), theta=np.zeros(max(npts, 1), np.float32), phi=np.zeros(max(npts, 1), np.float32))
    _ref_lib().ref_pc2_to_scan(_p(buf), C.c_uint32(cloud.width), C.c_uint32(cloud.height), C.c_uint32(cloud.point_step), C.c_uint64(cloud.row_step),
                               _p(off), C.c_int(f64), _p(T), C.byref(sm), C.c_int(flags), _p(out["ranges"]), _p(out["points"]), _p(out["mask"]),
                               _p(out["cell"]), _p(out["theta"]), _p(out["phi"]))
    for k in ("cell", "theta", "phi"):
        out[k] = out[k][:npts]
    return out


def product(cloud, model, T=None, order=None):
    """the product's scan_cloud_key / scan_cell_entry on the CPU, points visited in `order` (default: index order) -> dict(ranges, points, mask)"""
    buf, off, f64 = _cloud_args(cloud)
    sm, T = _model(model), _tf(T)
    n = model.phi_size * model.theta_size
    d = dirs(model)
    out = dict(ranges=np.zeros(n, np.float32), points=np.zeros((n, 3), np.float32), mask=np.zeros(n, np.uint8))
    order = None if order is None else np.ascontiguousarray(order, np.uint32)
    _emul_lib().emul_scan_from_cloud(_p(buf), C.c_uint32(cloud.width), C.c_uint32(cloud.height), C.c_uint64(cloud.row_step), C.c_uint32(cloud.point_step),
                                     _p(off), C.c_uint32(f64), _p(T), C.byref(sm), None if order is None else _p(order), _p(d),
                                     _p(out["ranges"]), _p(out["points"]), _p(out["mask"]))
    return out


def same(a, b):
    """ranges, points and mask equal bit for bit (NaN payloads not pinned)"""
    from pc2_ref import same_bits
    return same_bits(a["ranges"], b["ranges"]) and same_bits(a["points"], b["points"]) and np.array_equal(a["mask"], b["mask"])
