"""TEST INFRASTRUCTURE ONLY: references for b2_pf_sample_cloud (the particle filter's beams drawn from a PointCloud2).

* sample: the C restatement of PCDSensorUpdaterOptix::update's sampling loop with the library's keyed draws (pf_cloud_ref/pf_cloud_ref.c,
  which compiles the oracle's source in for Philox4x32-10).
* product_samples: the product's per-sample function (rmcl_b200/csrc/kernels.cuh: pf_sample_beam) compiled for the CPU
  (pf_cloud_ref/cloud_emul.cu), every sample's flag and beam; product = those under the give-up rule.
Both libraries are built on first use by native.py."""
import ctypes as C

import numpy as np

import native
from rmcl_b200.synth import RANGE_MEAS_DTYPE

_ref = None
_emul = None
MAX_INVALIDS = 10


def _ref_lib():
    global _ref
    if _ref is None:
        _ref = native.restatement("pf_cloud_ref/pf_cloud_ref.c")
        _ref.ref_pf_sample_cloud.restype = C.c_uint32
        _ref.ref_pf_sample_one.restype = C.c_int
    return _ref


def _emul_lib():
    global _emul
    if _emul is None:
        _emul = native.emulator()
        _emul.emul_pf_samples.restype = None
    return _emul


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _cloud_args(cloud):
    f = {p.name: p for p in cloud.fields}
    buf = np.ascontiguousarray(np.asarray(cloud.data, np.uint8).reshape(-1))
    if buf.size == 0:
        buf = np.zeros(1, np.uint8)
    off = np.array([f[c].offset for c in "xyz"], np.uint32)
    return buf, off, int(f["x"].datatype == 8)


def sample(cloud, n_samples, seed, step):
    """the restatement's beams (RANGE_MEAS_DTYPE, sample order)"""
    buf, off, f64 = _cloud_args(cloud)
    out = np.zeros(max(n_samples, 1), RANGE_MEAS_DTYPE)
    n = _ref_lib().ref_pf_sample_cloud(_p(buf), C.c_uint32(cloud.width), C.c_uint32(cloud.height), C.c_uint64(cloud.row_step), C.c_uint32(cloud.point_step),
                                       _p(off), C.c_int(f64), C.c_uint32(n_samples), C.c_uint64(seed), C.c_uint32(step), _p(out))
    return out[:n]


def product_samples(cloud, n_samples, seed, step):
    """the product's pf_sample_beam for samples 0 .. n_samples-1 -> (valid flags (n,), beams (n,) RANGE_MEAS_DTYPE)"""
    buf, off, f64 = _cloud_args(cloud)
    valid, out = np.zeros(max(n_samples, 1), np.uint32), np.zeros(max(n_samples, 1), RANGE_MEAS_DTYPE)
    _emul_lib().emul_pf_samples(_p(buf), C.c_uint32(cloud.width), C.c_uint32(cloud.height), C.c_uint64(cloud.row_step), C.c_uint32(cloud.point_step),
                                _p(off), C.c_uint32(f64), C.c_uint64(seed), C.c_uint32(step), C.c_uint32(n_samples), _p(valid), _p(out))
    return valid[:n_samples], out[:n_samples]


def give_up(valid, beams):
    """the valid samples before the MAX_INVALIDS-th invalid one, in order"""
    bad = np.flatnonzero(valid == 0)
    end = bad[MAX_INVALIDS - 1] if len(bad) >= MAX_INVALIDS else len(valid)
    return beams[:end][valid[:end] != 0]


def product(cloud, n_samples, seed, step):
    if int(cloud.width) * int(cloud.height) == 0:
        return np.zeros(0, RANGE_MEAS_DTYPE)
    return give_up(*product_samples(cloud, n_samples, seed, step))


def _points(n, nan_frac, rng, special=None):
    """n sensor-frame points at 0.5 .. 40 m; a fraction nan_frac of them with one NaN coordinate; special: 'inf' (an infinite coordinate
    on every fourth point), 'zero' (every fourth point (0,0,0))"""
    p = rng.normal(size=(n, 3)) * [1.0, 1.0, 0.3]
    p *= (rng.uniform(0.5, 40.0, n) / np.linalg.norm(p, axis=1))[:, None]
    k = rng.permutation(n)[: int(round(nan_frac * n))]
    p[k, rng.integers(0, 3, len(k))] = np.nan
    if special == "inf":
        p[::4, 1] = np.inf
        p[1::8, 0] = -np.inf
    elif special == "zero":
        p[::4] = 0.0
    return p


def clouds():
    """(name, PointCloud2) of every layout and content the sampling tests cover"""
    from rmcl_b200 import synth
    rng = np.random.default_rng(11)
    yield "1x1", synth.pointcloud2(np.array([[3.0, -4.0, 12.0]]), 1, 1)
    yield "1xN_unorganised", synth.pointcloud2(_points(5000, 0.0, rng), 5000, 1)
    for frac in (0.0, 0.5, 0.999):
        yield f"128x1024_nan{frac}", synth.pointcloud2(_points(128 * 1024, frac, rng), 1024, 128)
    p = _points(64 * 512, 0.5, rng)
    yield "f64_unaligned_padded", synth.pointcloud2(p, 512, 64, dtype=np.float64, point_step=40, offsets=(3, 13, 27), row_pad=7)
    yield "f32_ps48_extra_padded", synth.pointcloud2(p, 512, 64, point_step=48, offsets=(20, 4, 33), row_pad=5,
                                                     extra={"intensity": 8, "ring": 12, "mask": 0})
    yield "all_nan", synth.pointcloud2(np.full((300, 3), np.nan), 30, 10)
    yield "inf", synth.pointcloud2(_points(4096, 0.1, rng, "inf"), 64, 64)
    yield "zero", synth.pointcloud2(_points(4096, 0.1, rng, "zero"), 64, 64, dtype=np.float64, point_step=24, offsets=(0, 8, 16))


N_SAMPLES = (0, 1, 180, 4096)
