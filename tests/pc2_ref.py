"""TEST INFRASTRUCTURE ONLY: references for b2_rcc_set_cloud_o1dn (PointCloud2 -> O1Dn model + dataset).

* convert_np: a numpy float32 restatement of the reference's loop in its operation order -- estimateModelAndData
  (rmcl_ros/src/util/conversions.cpp:869-1073) restricted to the points filter keeps (rmcl_ros/src/util/scan_operations.cpp:41-143), then the
  dataset of MICPO1DnSensorCUDA::unpackMessage (MICPO1DnSensorCUDA.cpp:171-230).  reference_mask=True also applies the reference's use of a
  field named `mask` as the range (conversions.cpp:1014-1017), which the product deliberately does not (SURVEY Appendix D).
* product_np: the product's own per-ray function (rmcl_b200/csrc/kernels.cuh) compiled for the CPU (pc2_ref/pc2_emul.cu), built on first
  use into the per-user temporary directory of chain_ref."""
import ctypes as C
import os

import numpy as np

from chain_ref import _build

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(_HERE), "rmcl_b200", "csrc")
_emul = None


def out_dims(cloud, flt):
    """(W_out, H_out) of the filter: (dim - skip_begin - skip_end) / increment (scan_operations.cpp:46-47)"""
    w = (cloud.width - flt.width_skip_begin - flt.width_skip_end) // flt.width_increment
    h = (cloud.height - flt.height_skip_begin - flt.height_skip_end) // flt.height_increment
    return w, h


def _fields(cloud):
    f = {p.name: p for p in cloud.fields}
    return f


def _gather(buf, base, off, size):
    """bytes [base + off, base + off + size) of every point, at any alignment -> (n, size) uint8"""
    return buf[base[:, None] + off + np.arange(size)[None, :]]


def convert_np(cloud, flt, reference_mask=False):
    """-> dict(dirs (n,3) f32, ranges (n,) f32, points (n,3) f32, mask (n,) u8, width, height) of the filtered cloud"""
    f = _fields(cloud)
    w, h = out_dims(cloud, flt)
    i, j = np.meshgrid(np.arange(h, dtype=np.int64), np.arange(w, dtype=np.int64), indexing="ij")
    src_i = i.reshape(-1) * flt.height_increment + flt.height_skip_begin
    src_j = j.reshape(-1) * flt.width_increment + flt.width_skip_begin
    base = src_i * cloud.row_step + src_j * cloud.point_step          # rows use row_step (conversions.cpp:968-973)
    buf = np.asarray(cloud.data, np.uint8).reshape(-1)
    f64 = f["x"].datatype == 8
    dt, sz = (np.dtype("<f8"), 8) if f64 else (np.dtype("<f4"), 4)
    with np.errstate(all="ignore"):                                   # double -> float may overflow to inf, as in the reference
        x, y, z = [np.ascontiguousarray(_gather(buf, base, f[c].offset, sz)).view(dt).reshape(-1).astype(np.float32) for c in "xyz"]
        finite = np.isfinite(x) & np.isfinite(y) & np.isfinite(z)
        rng = np.sqrt((x * x + y * y) + z * z)                          # rm::Vector::l2norm, each op rounded to float
        d = np.stack([x / rng, y / rng, z / rng], 1)                   # rm::Vector::operator/=
        d[~finite] = 0.0
        rng = np.where(finite, rng, np.float32(0.0)).astype(np.float32)
        if reference_mask and "mask" in f:
            rng = _gather(buf, base, f["mask"].offset, 1)[:, 0].astype(np.float32)
        pts = d * rng[:, None] + np.float32(0.0)                      # dir * range + orig, orig = 0 (MICPO1DnSensorCUDA.cpp:201-203)
        mask = (~((rng < np.float32(flt.range_min)) | (rng > np.float32(flt.range_max)))).astype(np.uint8)
    return dict(dirs=d.astype(np.float32), ranges=rng, points=pts.astype(np.float32), mask=mask, width=w, height=h)


def _emul_lib():
    global _emul
    if _emul is None:
        src = os.path.join(_HERE, "pc2_ref", "pc2_emul.cu")
        deps = [src] + [os.path.join(_CSRC, f) for f in ("kernels.cuh", "icp_loop.cuh", "trace.cuh", "b2_math.cuh", "bvh8.h")] + \
               [os.path.join(os.path.dirname(_HERE), "include", "rmcl_b200.h")]
        nvcc = os.environ.get("NVCC", "nvcc")
        _emul = _build("pc2_emul", deps, [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-fmad=false",
                                          "-Xcompiler", "-fPIC,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared", src])
        _emul.emul_o1dn_from_cloud.restype = None
    return _emul


def product_np(cloud, flt):
    """the product's o1dn_cloud_entry on the CPU, one call per output ray -> the dict of convert_np"""
    f = _fields(cloud)
    w, h = out_dims(cloud, flt)
    n = w * h
    buf = np.ascontiguousarray(np.asarray(cloud.data, np.uint8).reshape(-1))
    out = dict(dirs=np.zeros((n, 3), np.float32), ranges=np.zeros(n, np.float32), points=np.zeros((n, 3), np.float32), mask=np.zeros(n, np.uint8),
               width=w, height=h)
    off = np.array([f[c].offset for c in "xyz"], np.uint32)
    hs = np.array([flt.height_skip_begin, flt.height_increment], np.uint32)
    ws = np.array([flt.width_skip_begin, flt.width_increment], np.uint32)
    p = lambda a: C.c_void_p(a.ctypes.data)
    _emul_lib().emul_o1dn_from_cloud(p(buf), C.c_uint32(w), C.c_uint32(h), C.c_uint64(cloud.row_step), C.c_uint32(cloud.point_step), p(off),
                                     C.c_uint32(int(f["x"].datatype == 8)), p(hs), p(ws), C.c_float(flt.range_min), C.c_float(flt.range_max),
                                     p(out["dirs"]), p(out["ranges"]), p(out["points"]), p(out["mask"]))
    return out


def same_bits(a, b):
    """bit-for-bit equality of two float arrays, every NaN counted equal to every NaN (the payload of 0/0 is not pinned)"""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)))
