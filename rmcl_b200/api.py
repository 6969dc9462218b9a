"""Host-side mirror of the reference's interface for the ray-casting-correspondence path, over the C ABI (ctypes).

Class / method names follow the reference (file:line cited per method); all arithmetic happens in librmcl_b200.so on the GPU.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np

from .synth import (CLUSTER_RECORD_DTYPE, CLUSTER_RESULT_DTYPE, CROSS_STATS_DTYPE, KLD_RESULT_DTYPE, PARTICLE_ATTR_DTYPE, PARTICLE_STATS_DTYPE, RANGE_MEAS_DTYPE,
                    RECOVERY_RESULT_DTYPE, RECOVERY_STATE_DTYPE, RESIDUAL_RESULT_DTYPE, SEARCH_BNB_RESULT_DTYPE, SEARCH_RECORD_DTYPE, TRANSFORM_DTYPE)

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("B2_LIB_PATH") or os.path.join(_HERE, "lib", "librmcl_b200.so")     # B2_LIB_PATH: experiment builds (scripts/)
_lib = None

B2_BUILD_HOST_SAH = 0
B2_BUILD_DEVICE_LBVH = 1


class B2Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"rmcl_b200 error {code}: {msg}")
        self.code = code


def lib_path():
    return _LIB_PATH


class _SphericalModel(C.Structure):
    _fields_ = [("phi_min", C.c_float), ("phi_inc", C.c_float), ("phi_size", C.c_uint32), ("theta_min", C.c_float), ("theta_inc", C.c_float),
                ("theta_size", C.c_uint32), ("range_min", C.c_float), ("range_max", C.c_float)]


class _PinholeModel(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
                ("range_min", C.c_float), ("range_max", C.c_float)]


class PFParams(C.Structure):
    """PCDSensorUpdaterEmbree config (rmcl_ros/src/rmcl/PCDSensorUpdaterEmbree.cpp:122-134)."""
    _fields_ = [("dist_sigma", C.c_float), ("real_hit_sim_miss_error", C.c_float), ("real_miss_sim_hit_error", C.c_float),
                ("real_miss_sim_miss_error", C.c_float), ("range_min", C.c_float), ("range_max", C.c_float), ("ng_mode", C.c_int),
                ("correspondence_type", C.c_int)]       # 0: ray casting (evaluate_rcc), 1: closest point (evaluate_cpc, :88-95,219-222)

    @staticmethod
    def defaults(ng_mode=0, correspondence_type=0):
        return PFParams(2.0, 100.0, 100.0, 0.0, 0.05, 80.0, ng_mode, correspondence_type)


class GladiatorConfig(C.Structure):
    """GladiatorResamplerConfig (rmcl_ros/include/rmcl_ros/rmcl/GladiatorResamplerConfig.hpp:7-20)."""
    _fields_ = [("min_noise_tx", C.c_float), ("min_noise_ty", C.c_float), ("min_noise_tz", C.c_float), ("min_noise_roll", C.c_float),
                ("min_noise_pitch", C.c_float), ("min_noise_yaw", C.c_float), ("likelihood_forget_per_meter", C.c_float),
                ("likelihood_forget_per_radian", C.c_float)]

    @staticmethod
    def defaults():
        return GladiatorConfig(0.03, 0.03, 0.0, 0.0, 0.0, 0.01, 0.3, 0.2)


class SurfaceConfig(C.Structure):
    """b2_surface_config: the surface constraint of projectToSurface (m, rad; align 0 keeps the orientation, 1 tilts the body z-axis onto
    the ground normal).  defaults() are the suggested values."""
    _fields_ = [("probe_above", C.c_float), ("probe_below", C.c_float), ("base_height", C.c_float), ("max_slope", C.c_float), ("align", C.c_int32)]

    @staticmethod
    def defaults():
        return SurfaceConfig(0.5, 1.0, 0.0, 0.6, 1)


class KLDConfig(C.Structure):
    """b2_kld_config: the bins and the bound of KLD-sampling (resampleKLD): res_xy and res_z in m (res_z = 0 leaves z unbinned), res_yaw in
    rad, the least particle count n_min, the bound's error epsilon and its upper normal quantile z.  defaults() are the suggested values:
    AMCL's defaults, whose kld_z of 0.99 AMCL passes as the quantile itself."""
    _fields_ = [("res_xy", C.c_float), ("res_z", C.c_float), ("res_yaw", C.c_float), ("n_min", C.c_uint32), ("epsilon", C.c_double), ("z", C.c_double)]

    @staticmethod
    def defaults():
        return KLDConfig(0.5, 0.0, math.radians(10.0), 100, 0.01, 0.99)


class ClusterConfig(C.Structure):
    """b2_cluster_config: the bins of estimateClusters (res_xy and res_z in m, res_z = 0 leaves z unbinned, res_yaw in rad: KLDConfig's) and
    the number of clusters to record, heaviest first (1 .. 16).  defaults() are AMCL's bin sizes and 8 records."""
    _fields_ = [("res_xy", C.c_float), ("res_z", C.c_float), ("res_yaw", C.c_float), ("max_records", C.c_uint32)]

    @staticmethod
    def defaults():
        return ClusterConfig(0.5, 0.0, math.radians(10.0), 8)


class RecoveryConfig(C.Structure):
    """b2_recovery_config: the rates of the slow and the fast average of the recovery (recoveryObserve), 0 <= alpha_slow <= alpha_fast <= 1.
    defaults() are AMCL's recovery_alpha_slow and recovery_alpha_fast."""
    _fields_ = [("alpha_slow", C.c_double), ("alpha_fast", C.c_double)]

    @staticmethod
    def defaults():
        return RecoveryConfig(0.001, 0.1)


class SteinConfig(C.Structure):
    """b2_stein_config: the Stein variational steps of steinUpdate: iterations per call, the reference set's size n_ref (0: every particle),
    the RMSProp step sizes step_t (m) and step_r (rad), the kernel bandwidth's floors min_bandwidth_t (m) and min_bandwidth_r (rad), and
    the likelihood's uniform share w_rand in [0, 1).  defaults() are the suggested values (SURVEY appendix L says why)."""
    _fields_ = [("iterations", C.c_uint32), ("n_ref", C.c_uint32), ("step_t", C.c_float), ("step_r", C.c_float), ("min_bandwidth_t", C.c_float),
                ("min_bandwidth_r", C.c_float), ("w_rand", C.c_float), ("pad", C.c_float)]

    @staticmethod
    def defaults():
        return SteinConfig(10, 4096, 0.02, 0.01, 0.05, 0.02, 0.05, 0.0)


class SearchConfig(C.Structure):
    """b2_search_config: the grid of globalSearch, candidate (i, j, k) at (x0 + i * step, y0 + j * step, z0) with heading -pi + 2 pi k /
    n_yaw (i < nx, j < ny), the number of records to return (1 .. 64) and the least distance (m) and heading difference (rad) a record
    keeps from every better one unless it differs in the other.  defaults(bb_min, bb_max, z0) covers the (x, y) box from bb_min to bb_max
    with the suggested values: step 0.25 m, 72 headings, 8 records, separations 1 m and 30 deg; without a box the grid is left empty."""
    _fields_ = [("x0", C.c_float), ("y0", C.c_float), ("z0", C.c_float), ("step", C.c_float), ("nx", C.c_uint32), ("ny", C.c_uint32), ("n_yaw", C.c_uint32),
                ("max_records", C.c_uint32), ("min_separation_xy", C.c_float), ("min_separation_yaw", C.c_float)]

    @staticmethod
    def defaults(bb_min=None, bb_max=None, z0=0.0, step=0.25):
        cfg = SearchConfig(0.0, 0.0, float(z0), float(step), 0, 0, 72, 8, 1.0, math.radians(30.0))
        if bb_min is not None and bb_max is not None:
            cfg.x0, cfg.y0 = float(bb_min[0]), float(bb_min[1])
            cfg.nx = int(math.floor((float(bb_max[0]) - float(bb_min[0])) / step)) + 1
            cfg.ny = int(math.floor((float(bb_max[1]) - float(bb_min[1])) / step)) + 1
        return cfg


class _SearchResult(C.Structure):
    _fields_ = [("n_candidates", C.c_uint64), ("n_valid", C.c_uint64), ("n_peaks", C.c_uint64), ("n_records", C.c_uint64)]


class _SteinResult(C.Structure):
    _fields_ = [("bandwidth", C.c_float * 3), ("n_ref", C.c_uint32), ("n_blocked", C.c_uint32), ("rms_step_t", C.c_float), ("rms_step_r", C.c_float),
                ("pad", C.c_float)]


class _SteinSliceResult(C.Structure):
    _fields_ = [("bandwidth", C.c_float * 3), ("n_ref", C.c_uint32), ("n_blocked", C.c_uint32), ("n_steps", C.c_uint32), ("sum_step_t2", C.c_double),
                ("sum_step_r2", C.c_double)]


class _CloudLayout(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("point_step", C.c_uint32), ("row_step", C.c_uint32), ("offset_x", C.c_uint32),
                ("offset_y", C.c_uint32), ("offset_z", C.c_uint32), ("datatype", C.c_uint8), ("is_bigendian", C.c_uint8), ("pad", C.c_uint8 * 2)]


B2_CLOUD_NO_FIELD = 0xFFFFFFFF


class O1DnCloudFilter(C.Structure):
    """The parameters of pc2_to_o1dn (rmcl_ros/src/nodes/conversion/pc2_to_o1dn.cpp:48-77): skips and increment of both axes, and the range
    limits of the model.  defaults() are the node's declared defaults."""
    _fields_ = [("height_skip_begin", C.c_uint32), ("height_skip_end", C.c_uint32), ("height_increment", C.c_uint32),
                ("width_skip_begin", C.c_uint32), ("width_skip_end", C.c_uint32), ("width_increment", C.c_uint32),
                ("range_min", C.c_float), ("range_max", C.c_float)]

    @staticmethod
    def defaults(range_min=0.3, range_max=50.0):
        return O1DnCloudFilter(0, 0, 1, 0, 0, 1, range_min, range_max)


def cloud_layout(cloud):
    """b2_cloud_layout of a sensor_msgs/PointCloud2-shaped object (width, height, point_step, row_step, is_bigendian, fields with name / offset /
    datatype): x, y and z are looked up by name, a missing one is marked B2_CLOUD_NO_FIELD; the datatype is that of x."""
    off = {f.name: f for f in cloud.fields}
    L = _CloudLayout(int(cloud.width), int(cloud.height), int(cloud.point_step), int(cloud.row_step),
                     *[int(off[k].offset) if k in off else B2_CLOUD_NO_FIELD for k in ("x", "y", "z")],
                     int(off["x"].datatype) if "x" in off else 0, int(bool(cloud.is_bigendian)))
    return L


def _identity_tf():
    T = np.zeros((), TRANSFORM_DTYPE)
    T["R"][3] = 1.0
    return T


def _cloud_buffer(cloud):
    """(address, bytes, on device) of a PointCloud2-shaped object's data: a torch tensor, CUDA (read in place) or host, pinned or pageable
    (uploaded), or a numpy / bytes buffer (uploaded)"""
    data = cloud.data
    if hasattr(data, "data_ptr") and not data.is_contiguous():
        raise TypeError("setPointCloud: cloud.data must be contiguous")
    if getattr(data, "is_cuda", False):
        return (*_records(data, 1), 1)
    if isinstance(data, (bytes, bytearray, memoryview)):
        data = np.frombuffer(data, np.uint8)
    ptr, nbytes = _records(data, 1, lambda d: np.ascontiguousarray(d).view(np.uint8).reshape(-1))
    return ptr if nbytes else None, nbytes, 0


class _MeshInfo(C.Structure):
    _fields_ = [("n_faces", C.c_uint32), ("n_vertices", C.c_uint32), ("n_nodes", C.c_uint32), ("n_leaf_tris", C.c_uint32), ("max_depth", C.c_uint32),
                ("bvh_bytes", C.c_uint64), ("build_ms", C.c_float), ("device", C.c_int), ("build_mode", C.c_int), ("sah_cost", C.c_float)]


EXPORTS = [
    "b2_last_error", "b2_version", "b2_device_count", "b2_mesh_create", "b2_mesh_destroy", "b2_mesh_get_info", "b2_mesh_intersect",
    "b2_mesh_intersect_stats", "b2_rcc_create", "b2_rcc_destroy", "b2_rcc_set_stream", "b2_rcc_set_tsb", "b2_rcc_set_model_spherical",
    "b2_rcc_set_model_pinhole", "b2_rcc_set_model_o1dn", "b2_rcc_set_model_ondn", "b2_rcc_set_params", "b2_rcc_set_dataset", "b2_rcc_set_ranges",
    "b2_rcc_find", "b2_rcc_cross_statistics", "b2_rcc_model_view", "b2_rcc_dataset_view", "b2_rcc_download_model", "b2_rcc_download_dataset",
    "b2_rcc_correct_once", "b2_rcc_correct_once_ranges", "b2_rcc_correct_batch", "b2_umeyama_batch", "b2_pf_create", "b2_pf_destroy",
    "b2_pf_set_stream", "b2_pf_sensor_update", "b2_pf_sensor_update_host", "b2_kernel_launch_count", "b2_rcc_enable_timing", "b2_rcc_last_timing", "b2_pf_motion_update", "b2_pf_likelihood_stats",
    "b2_rcc_set_correspondence_type", "b2_pf_resample_gladiator", "b2_pf_gladiator_randoms", "b2_rcc_segment", "b2_mesh_create_from_file", "b2_mesh_file_load", "b2_mesh_file_free", "b2_peek_cuda_error", "b2_mesh_blob_size", "b2_mesh_export_blob", "b2_mesh_create_from_blob", "b2_mesh_refit",
    "b2_rcc_correct_once_async", "b2_rcc_correct_once_wait", "b2_micp_correct_once", "b2_rcc_set_exec_mode", "b2_debug_read_bandwidth", "b2_rcc_set_sim_options", "b2_rcc_bind_dataset", "b2_rcc_bind_model_buffers", "b2_rcc_benchmark_batch", "b2_pf_p2p_init", "b2_pf_p2p_connect", "b2_pf_p2p_publish", "b2_pf_resample_gladiator_p2p", "b2_pf_p2p_connect_local", "b2_rcc_set_cpc_options", "b2_pf_set_mapping", "b2_pf_get_mapping",
    "b2_micp_correct", "b2_pf_init_uniform", "b2_pf_init_gaussian", "b2_pf_estimate_stats", "b2_rcc_set_cloud_o1dn",
    "b2_rcc_set_cloud_spherical", "b2_pf_sample_cloud", "b2_pf_resample_residual", "b2_pf_project_to_surface",
    "b2_pf_resample_kld", "b2_pf_cluster_stats", "b2_micp_pose_covariance", "b2_pf_recovery_reset", "b2_pf_recovery_observe",
    "b2_pf_recovery_inject", "b2_dfield_create", "b2_dfield_destroy", "b2_dfield_get_info", "b2_dfield_download", "b2_dfield_query",
    "b2_pf_sensor_update_field", "b2_pf_stein_update", "b2_pf_stein_slice_begin", "b2_pf_stein_slice_score", "b2_pf_stein_slice_move",
    "b2_pf_stein_slice_result", "b2_pf_global_search", "b2_pf_global_search_bnb",
]


def load_library():
    """Load librmcl_b200.so.  Fails loudly when it is missing: there is no CPU fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise B2Error(-2, f"CUDA library not built: {_LIB_PATH} (run `python -c 'import __graft_entry__ as g; g.build()'`)")
    lib = C.CDLL(_LIB_PATH)
    for name in EXPORTS:
        getattr(lib, name)            # AttributeError if the ABI is incomplete
    lib.b2_last_error.restype = C.c_char_p
    lib.b2_kernel_launch_count.restype = C.c_uint64
    for name in EXPORTS:
        if name not in ("b2_last_error", "b2_kernel_launch_count", "b2_mesh_file_free", "b2_peek_cuda_error"):
            getattr(lib, name).restype = C.c_int
    lib.b2_mesh_file_free.restype = None
    lib.b2_peek_cuda_error.restype = C.c_char_p
    _lib = lib
    return lib


def _chk(rc):
    if rc != 0:
        raise B2Error(rc, load_library().b2_last_error().decode("utf-8", "replace"))


def read_bandwidth(nbytes, iters=20, device=0):
    """GB/s of the library's read micro-benchmark over a working set of `nbytes` (L2 below its capacity, HBM far above)."""
    out = C.c_double()
    _chk(load_library().b2_debug_read_bandwidth(C.c_int(device), C.c_uint64(int(nbytes)), C.c_int(int(iters)), C.byref(out)))
    return out.value


def kernel_launch_count():
    return int(load_library().b2_kernel_launch_count())


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def _u8(a):
    return np.ascontiguousarray(a, np.uint8)


def _tf(a):
    a = np.ascontiguousarray(a)
    if a.dtype.itemsize != 32:
        raise TypeError("expected 32-byte Transform records (synth.TRANSFORM_DTYPE)")
    return a


def _devptr(x):
    """Device address of a torch CUDA tensor (or a raw int)."""
    if x is None:
        return None
    if isinstance(x, int):
        return C.c_void_p(x)
    if hasattr(x, "data_ptr"):
        if not x.is_cuda or not x.is_contiguous():
            raise TypeError("expected a contiguous CUDA tensor")
        return C.c_void_p(x.data_ptr())
    raise TypeError(type(x))


def _records(x, size, host=None):
    """(address, count) of an array of `size`-byte records.  host None: a contiguous CUDA tensor, read in place.  Otherwise a host array,
    made a contiguous numpy array by the conversion `host`; the address keeps that array alive.  A wrong kind of array, or a byte size that
    is not a whole number of records, raises TypeError."""
    if host is None:
        if not hasattr(x, "data_ptr") or not x.is_cuda or not x.is_contiguous():
            raise TypeError("expected a contiguous CUDA tensor")
        addr, nbytes = C.c_void_p(x.data_ptr()), x.numel() * x.element_size()
    else:
        a = host(x)
        addr, nbytes = a.ctypes.data_as(C.c_void_p), a.nbytes
    if nbytes % size:
        raise TypeError(f"expected {size}-byte records, got {nbytes} bytes")
    return addr, nbytes // size


def _agree(what, **arrays):
    """The C ABI takes one count for all arrays of a call, so the binding checks their lengths: each keyword is (array, record size[, host
    conversion]) as _records takes it, None passes as a null address.  -> (address of each array in keyword order..., the first array's
    count).  A count that differs from the first raises ValueError."""
    out, n, first = [], None, None
    for name, (x, *spec) in arrays.items():
        if x is None:
            out.append(None)
            continue
        addr, k = _records(x, *spec)
        if n is None:
            n, first = k, name
        elif k != n:
            raise ValueError(f"{what}: {n} {first} but {k} {name}")
        out.append(addr)
    return (*out, n)


def read_mesh_file(path):
    """Import step of Map.from_file alone (host only): -> (vertices (nv,3) float32, faces (nf,3) uint32)."""
    lib = load_library()
    v, f, nv, nf = C.POINTER(C.c_float)(), C.POINTER(C.c_uint32)(), C.c_uint32(), C.c_uint32()
    _chk(lib.b2_mesh_file_load(os.fsencode(path), C.byref(v), C.byref(nv), C.byref(f), C.byref(nf)))
    try:
        V = np.ctypeslib.as_array(v, (nv.value, 3)).copy()
        F = np.ctypeslib.as_array(f, (nf.value, 3)).copy()
    finally:
        lib.b2_mesh_file_free(v, f)
    return V, F


class Map:
    """Triangle mesh + in-HBM BVH; stands in for rm::EmbreeMap / rm::OptixMap (rm::import_embree_map, micp_localization.cpp:188)."""

    def __init__(self, verts, faces, device=0, build_mode=None):
        lib = load_library()
        if build_mode is None:
            build_mode = int(os.environ.get("B2_BUILD_MODE", B2_BUILD_DEVICE_LBVH))     # device build: faster to build AND to trace (DESIGN.md section 3)
        verts = _f32(verts).reshape(-1, 3)
        faces = np.ascontiguousarray(faces, np.uint32).reshape(-1, 3)
        h = C.c_void_p()
        _chk(lib.b2_mesh_create(_p(verts), C.c_uint32(len(verts)), _p(faces), C.c_uint32(len(faces)), C.c_int(device), C.c_int(build_mode), C.byref(h)))
        self._h = h
        self.device = device

    @classmethod
    def from_file(cls, path, device=0, build_mode=None):
        """rm::import_embree_map(file) twin: .ply (ascii / binary little endian) or .obj."""
        lib = load_library()
        if build_mode is None:
            build_mode = int(os.environ.get("B2_BUILD_MODE", B2_BUILD_DEVICE_LBVH))
        self = cls.__new__(cls)
        h = C.c_void_p()
        _chk(lib.b2_mesh_create_from_file(os.fsencode(path), C.c_int(device), C.c_int(build_mode), C.byref(h)))
        self._h, self.device = h, device
        return self

    def refit(self, verts):
        """Vertices moved, same faces: refit the resident BVH (SURVEY 8f1).  Device-built maps only."""
        verts = _f32(verts).reshape(-1, 3)
        _chk(load_library().b2_mesh_refit(self._h, _p(verts), C.c_uint32(len(verts)), C.c_int(0)))

    def export_blob(self):
        """The built BVH as bytes (numpy uint8): build once, broadcast / cache, `Map.from_blob` on the receiving side."""
        n = C.c_uint64()
        _chk(load_library().b2_mesh_blob_size(self._h, C.byref(n)))
        buf = np.empty(n.value, np.uint8)
        _chk(load_library().b2_mesh_export_blob(self._h, _p(buf), C.c_uint64(n.value)))
        return buf

    @classmethod
    def from_blob(cls, blob, device=0):
        blob = np.ascontiguousarray(blob, np.uint8)
        self = cls.__new__(cls)
        h = C.c_void_p()
        _chk(load_library().b2_mesh_create_from_blob(_p(blob), C.c_uint64(blob.size), C.c_int(device), C.byref(h)))
        self._h, self.device = h, device
        return self

    def close(self):
        if getattr(self, "_h", None):
            load_library().b2_mesh_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def info(self):
        inf = _MeshInfo()
        _chk(load_library().b2_mesh_get_info(self._h, C.byref(inf)))
        return {k: getattr(inf, k) for k, _ in _MeshInfo._fields_}

    def intersect(self, origs, dirs, tfar=np.inf):
        """Closest hit for arbitrary rays (replaces rtcIntersect1, PCDSensorUpdaterEmbree.cpp:30-47)."""
        o, d, n = _agree("intersect", origs=(origs, 12, _f32), dirs=(dirs, 12, _f32))
        t, f, ng, h = np.empty(n, np.float32), np.empty(n, np.uint32), np.empty((n, 3), np.float32), np.empty(n, np.uint8)
        _chk(load_library().b2_mesh_intersect(self._h, o, d, C.c_uint32(n), C.c_float(tfar), _p(t), _p(f), _p(ng), _p(h)))
        return t, f, ng, h

    def traversal_stats(self, origs, dirs, tfar=np.inf):
        o, d, n = _agree("traversal_stats", origs=(origs, 12, _f32), dirs=(dirs, 12, _f32))
        a, b = C.c_double(), C.c_double()
        _chk(load_library().b2_mesh_intersect_stats(self._h, o, d, C.c_uint32(n), C.c_float(tfar), C.byref(a), C.byref(b)))
        return a.value, b.value


class RCCB200:
    """Ray-casting correspondences on the GPU: the Correspondences_<VRAM_CUDA> interface
    (rmcl/include/rmcl/registration/Correspondences.hpp:16-88) + the fused drivers."""

    def __init__(self, map_: Map):
        self.map = map_
        h = C.c_void_p()
        _chk(load_library().b2_rcc_create(map_._h, C.byref(h)))
        self._h = h
        self.n = 0
        self.outdated = True                       # Correspondences.hpp:31
        self.max_dist = 1.0                        # params.max_dist, :22
        self.adaptive_max_dist_min = 0.15          # :23

    def close(self):
        if getattr(self, "_h", None):
            load_library().b2_rcc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def setStream(self, cuda_stream):
        _chk(load_library().b2_rcc_set_stream(self._h, C.c_void_p(int(cuda_stream))))

    def enableTiming(self, on=True):
        _chk(load_library().b2_rcc_enable_timing(self._h, C.c_int(int(on))))

    def lastTiming(self):
        """(find_ms, reduce_ms) of the most recent correctOnce, from CUDA events recorded on the handle's stream."""
        a, b = C.c_float(), C.c_float()
        _chk(load_library().b2_rcc_last_timing(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def setTsb(self, Tsb):                         # Correspondences.hpp:33-36
        _chk(load_library().b2_rcc_set_tsb(self._h, _p(_tf(Tsb))))

    def setParams(self, max_dist, adaptive_max_dist_min):
        self.max_dist, self.adaptive_max_dist_min = float(max_dist), float(adaptive_max_dist_min)
        _chk(load_library().b2_rcc_set_params(self._h, C.c_float(max_dist), C.c_float(adaptive_max_dist_min)))

    def setModel(self, m):                         # ModelSetter<ModelT>::setModel (RCCEmbree.cpp:21-24 ...)
        lib = load_library()
        name = type(m).__name__
        if name == "SphericalModel":
            sm = _SphericalModel(m.phi_min, m.phi_inc, m.phi_size, m.theta_min, m.theta_inc, m.theta_size, m.range_min, m.range_max)
            _chk(lib.b2_rcc_set_model_spherical(self._h, C.byref(sm)))
        elif name == "PinholeModel":
            pm = _PinholeModel(m.width, m.height, m.fx, m.fy, m.cx, m.cy, m.range_min, m.range_max)
            _chk(lib.b2_rcc_set_model_pinhole(self._h, C.byref(pm)))
        elif name == "O1DnModel":
            o, d = _f32(m.orig).reshape(3), _f32(m.dirs).reshape(-1, 3)
            _chk(lib.b2_rcc_set_model_o1dn(self._h, C.c_uint32(m.width), C.c_uint32(m.height), _p(o), _p(d), C.c_float(m.range_min), C.c_float(m.range_max)))
        elif name == "OnDnModel":
            o, d = _f32(m.origs).reshape(-1, 3), _f32(m.dirs).reshape(-1, 3)
            _chk(lib.b2_rcc_set_model_ondn(self._h, C.c_uint32(m.width), C.c_uint32(m.height), _p(o), _p(d), C.c_float(m.range_min), C.c_float(m.range_max)))
        else:
            raise TypeError(name)
        self.model = m
        self.n = m.size

    def setDataset(self, points, mask=None):       # public field `dataset`, Correspondences.hpp:24
        dev = hasattr(points, "data_ptr")
        p, m, n = _agree("setDataset", points=(points, 12, None if dev else _f32), mask=(mask, 1, None if dev else _u8))
        _chk(load_library().b2_rcc_set_dataset(self._h, p, m, C.c_uint32(n), C.c_int(int(dev))))
        self.outdated = True

    def setRanges(self, ranges):                   # MICP..Sensor..::unpackMessage / v1 setInputData
        if hasattr(ranges, "data_ptr"):
            _chk(load_library().b2_rcc_set_ranges(self._h, _devptr(ranges), C.c_uint32(ranges.numel()), C.c_int(1)))
        else:
            ranges = _f32(ranges).reshape(-1)
            _chk(load_library().b2_rcc_set_ranges(self._h, _p(ranges), C.c_uint32(len(ranges)), C.c_int(0)))
        self.outdated = True

    setInputData = setRanges

    def find(self, Tbm_est):                       # RCCEmbree.cpp:26-36
        _chk(load_library().b2_rcc_find(self._h, _p(_tf(Tbm_est))))
        self.outdated = False

    def computeCrossStatistics(self, T_snew_sold, convergence_progress=0.0):   # CorrespondencesCPU.cpp:10-39
        out = np.zeros((), CROSS_STATS_DTYPE)
        _chk(load_library().b2_rcc_cross_statistics(self._h, _p(_tf(T_snew_sold)), C.c_double(convergence_progress), _p(out)))
        return out

    def modelView(self):                           # Correspondences.hpp:47-54 (host copies)
        nn = C.c_uint32()
        _chk(load_library().b2_rcc_model_view(self._h, None, None, None, None, None, C.byref(nn)))
        n = nn.value
        out = dict(points=np.empty((n, 3), np.float32), normals=np.empty((n, 3), np.float32), hits=np.empty(n, np.uint8),
                   face_ids=np.empty(n, np.uint32), ranges=np.empty(n, np.float32))
        _chk(load_library().b2_rcc_download_model(self._h, _p(out["points"]), _p(out["normals"]), _p(out["hits"]), _p(out["face_ids"]), _p(out["ranges"])))
        return out

    def datasetView(self):                         # Correspondences.hpp:56-62 (host copies)
        p, m, n = C.c_void_p(), C.c_void_p(), C.c_uint32()
        _chk(load_library().b2_rcc_dataset_view(self._h, C.byref(p), C.byref(m), C.byref(n)))
        out = dict(points=np.empty((n.value, 3), np.float32), mask=np.empty(n.value, np.uint8))
        _chk(load_library().b2_rcc_download_dataset(self._h, _p(out["points"]), _p(out["mask"])))
        return out

    def segment(self, min_dist_outlier_scan=0.15, min_dist_outlier_map=0.15):
        """ScanMapSegmentationEmbreeNode::scanCB classification (scan_map_segmentation_embree.cpp:110-187) after setRanges(real scan) and
        find(pose): -> (outlier_scan (k,3), outlier_map (m,3), labels (n,))."""
        nn = C.c_uint32()
        _chk(load_library().b2_rcc_model_view(self._h, None, None, None, None, None, C.byref(nn)))
        n = nn.value
        a, b, lab = np.zeros((max(n, 1), 3), np.float32), np.zeros((max(n, 1), 3), np.float32), np.zeros(max(n, 1), np.uint8)
        na, nb = C.c_uint32(), C.c_uint32()
        _chk(load_library().b2_rcc_segment(self._h, C.c_float(min_dist_outlier_scan), C.c_float(min_dist_outlier_map), _p(a), C.c_uint32(n), C.byref(na),
                                           _p(b), C.c_uint32(n), C.byref(nb), _p(lab)))
        return a[: na.value].copy(), b[: nb.value].copy(), lab[:n].copy()

    _CO_OUT = np.dtype([("Tn", TRANSFORM_DTYPE), ("Td", TRANSFORM_DTYPE), ("Cm", CROSS_STATS_DTYPE)])

    def _co_scratch(self):
        """Persistent argument block of correctOnce: at ~10 kHz call rates the per-call numpy/ctypes object churn of the generic path
        (~12 us) would be a tenth of the step; here the arguments go into one preallocated 192-byte block and the addresses are plain ints."""
        sc = getattr(self, "_co", None)
        if sc is None:
            buf = (C.c_char * 192)()                  # Tom 0:32 | Tbo 32:64 | Tom_new 64:96 | T_onew_oold 96:128 | Cmerged_o 128:192
            base = C.addressof(buf)
            lib = load_library()
            lib.b2_rcc_correct_once.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
            lib.b2_rcc_correct_once_ranges.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
            lib.b2_rcc_correct_once_async.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_double]
            lib.b2_rcc_correct_once_wait.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
            self._co_async, self._co_wait = lib.b2_rcc_correct_once_async, lib.b2_rcc_correct_once_wait
            sc = self._co = (buf, memoryview(buf).cast("B"), base, lib.b2_rcc_correct_once, lib.b2_rcc_correct_once_ranges)
        return sc

    def correctOnce(self, Tom, Tbo, iterations=5, convergence_progress=0.0, ranges=None):
        """MICPLocalizationNode::correctOnce for this sensor (micp_localization.cpp:899-984), fully on the device.
        With `ranges` (host array) the scan upload is part of the call (end-to-end entry point)."""
        buf, mv, base, f_once, f_ranges = self._co_scratch()
        a, b = np.asarray(Tom).tobytes(), np.asarray(Tbo).tobytes()
        if len(a) != 32 or len(b) != 32:
            raise TypeError("expected 32-byte Transform records (synth.TRANSFORM_DTYPE)")
        mv[0:32] = a
        mv[32:64] = b
        if ranges is None:
            rc = f_once(self._h, base, base + 32, iterations, convergence_progress, base + 64, base + 96, base + 128)
        else:
            if hasattr(ranges, "data_ptr"):       # pinned / pageable HOST torch tensor
                rp, rn = ranges.data_ptr(), ranges.numel()
            else:
                ranges = _f32(ranges).reshape(-1)
                rp, rn = ranges.ctypes.data, len(ranges)
            rc = f_ranges(self._h, rp, rn, base, base + 32, iterations, convergence_progress, base + 64, base + 96, base + 128)
        if rc != 0:
            _chk(rc)
        self.outdated = False
        out = np.frombuffer(bytearray(mv[64:192]), self._CO_OUT)
        return out["Tn"][0], out["Td"][0], out["Cm"][0]

    def bindDataset(self, points, mask):
        """use caller-owned CUDA tensors as the dataset (no copy): the reference's public `dataset` member in VRAM (Correspondences.hpp:24)"""
        p, m, n = _agree("bindDataset", points=(points, 12), mask=(mask, 1))
        _chk(load_library().b2_rcc_bind_dataset(self._h, p, m, C.c_uint32(n)))
        self._bound = (points, mask)
        self.outdated = True

    def bindModelBuffers(self, points, normals, hits):
        """find() writes into these caller-owned CUDA tensors: the reference's protected `model_buffers_` (Correspondences.hpp:81-85); None unbinds"""
        if points is None:
            _chk(load_library().b2_rcc_bind_model_buffers(self._h, None, None, None, C.c_uint32(0)))
            self._bound_model = None
            return
        h, p, nr, n = _agree("bindModelBuffers", hits=(hits, 1), points=(points, 12), normals=(normals, 12))
        _chk(load_library().b2_rcc_bind_model_buffers(self._h, p, nr, h, C.c_uint32(n)))
        self._bound_model = (points, normals, hits)

    def setSimOptions(self, tfar_mode=0, min_mode=0, miss_fill=0):
        """the open rmagine simulate() semantics of SURVEY.md A.3: tfar = +inf, closest hit below range.min = miss, misses filled with zeros"""
        _chk(load_library().b2_rcc_set_sim_options(self._h, C.c_int(tfar_mode), C.c_int(min_mode), C.c_int(miss_fill)))

    def setExecMode(self, mode):
        """2 (default): one kernel, block sums exchanged by 64-bit atomics, programmatic launch; 1: cooperative launch, FP64 exchange behind a grid sync; 0: one reduction launch per inner iteration."""
        _chk(load_library().b2_rcc_set_exec_mode(self._h, C.c_int(int(mode))))

    def correctOnceAsync(self, Tom, Tbo, iterations=5, convergence_progress=0.0):
        """Enqueue one correctOnce on the handle's stream and return; collect with correctOnceWait()."""
        buf, mv, base, _, _ = self._co_scratch()
        mv[0:32] = np.asarray(Tom).tobytes()
        mv[32:64] = np.asarray(Tbo).tobytes()
        rc = self._co_async(self._h, base, base + 32, iterations, convergence_progress)
        if rc != 0:
            _chk(rc)

    def correctOnceWait(self):
        buf, mv, base, _, _ = self._co_scratch()
        rc = self._co_wait(self._h, base + 64, base + 96, base + 128)
        if rc != 0:
            _chk(rc)
        self.outdated = False
        out = np.frombuffer(bytearray(mv[64:192]), self._CO_OUT)
        return out["Tn"][0], out["Td"][0], out["Cm"][0]

    def benchmark(self, Tbm, n_runs=10):
        """v1 corrector.benchmark(T, Nruns) -> dict(sim, red, svd) seconds (lidar_corrector_optix_benchmark.cpp:143-155): stages run unfused"""
        Tbm = _tf(Tbm).reshape(-1)
        a, b, c = C.c_double(), C.c_double(), C.c_double()
        _chk(load_library().b2_rcc_benchmark_batch(self._h, _p(Tbm), C.c_uint32(len(Tbm)), C.c_uint32(n_runs), C.byref(a), C.byref(b), C.byref(c)))
        return dict(sim=a.value, red=b.value, svd=c.value)

    def correct(self, Tbm):
        """v1 {Sphere,Pinhole,O1Dn}Corrector::correct(Tbm[N]) -> (Tdelta[N], Ncorr[N], stats_b[N])
        (rmcl_ros/src/benchmarks/lidar_corrector_embree_benchmark.cpp:127-133)."""
        lib = load_library()
        if hasattr(Tbm, "data_ptr"):
            import torch
            pT, n = _records(Tbm, 32)
            Td = torch.empty((n, 8), dtype=torch.float32, device=Tbm.device)
            nc = torch.empty((n,), dtype=torch.int32, device=Tbm.device)
            st = torch.empty((n, 16), dtype=torch.float32, device=Tbm.device)
            _chk(lib.b2_rcc_correct_batch(self._h, pT, C.c_uint32(n), C.c_int(1), _devptr(Td), _devptr(nc), _devptr(st), C.c_int(1)))
            return Td, nc, st
        pT, n = _records(Tbm, 32, _tf)
        Td, nc, st = np.zeros(n, TRANSFORM_DTYPE), np.zeros(n, np.uint32), np.zeros(n, CROSS_STATS_DTYPE)
        _chk(lib.b2_rcc_correct_batch(self._h, pT, C.c_uint32(n), C.c_int(0), _p(Td), _p(nc), _p(st), C.c_int(0)))
        return Td, nc, st


class RCCB200Spherical(RCCB200):
    """rmcl::RCCEmbreeSpherical / RCCOptixSpherical twin (rmcl/include/rmcl/registration/RCCEmbree.hpp:18-33)."""

    def setPointCloud(self, cloud, T_sensor_cloud=None):
        """A sensor_msgs/PointCloud2 binned into the spherical model of the last setModel as this sensor's scan (b2_rcc_set_cloud_spherical):
        pc2_to_scan's conversion, fillEmpty and the dataset, in two kernels; the model and find's tile schedule stay.  `cloud` is
        PointCloud2-shaped (synth.pointcloud2 or the ROS message); its `data` is a numpy / bytes buffer or host tensor (uploaded, the call
        synchronises) or a CUDA uint8 tensor (read in place).  `T_sensor_cloud`: the cloud frame in the sensor frame (TRANSFORM_DTYPE),
        None = identity."""
        T = _tf(_identity_tf() if T_sensor_cloud is None else T_sensor_cloud)
        L = cloud_layout(cloud)
        ptr, nbytes, dev = _cloud_buffer(cloud)
        _chk(load_library().b2_rcc_set_cloud_spherical(self._h, ptr, C.c_uint64(nbytes), C.byref(L), _p(T), C.c_int(dev)))
        self.outdated = True


class RCCB200Pinhole(RCCB200):
    """rmcl::RCCEmbreePinhole twin (RCCEmbree.hpp:35-49)."""


class RCCB200O1Dn(RCCB200):
    """rmcl::RCCEmbreeO1Dn twin (RCCEmbree.hpp:51-66)."""

    def setPointCloud(self, cloud, filter=None):
        """An organised sensor_msgs/PointCloud2 as this sensor's scan (b2_rcc_set_cloud_o1dn): pc2_to_o1dn's conversion and filter, the O1Dn
        model and the dataset, in one kernel.  `cloud` is PointCloud2-shaped (synth.pointcloud2 or the ROS message); its `data` is a numpy /
        bytes buffer or host tensor (uploaded, the call synchronises) or a CUDA uint8 tensor (read in place).  `filter`: O1DnCloudFilter, default defaults()."""
        flt = filter if filter is not None else O1DnCloudFilter.defaults()
        L = cloud_layout(cloud)
        ptr, nbytes, dev = _cloud_buffer(cloud)
        _chk(load_library().b2_rcc_set_cloud_o1dn(self._h, ptr, C.c_uint64(nbytes), C.byref(L), C.byref(flt), C.c_int(dev)))
        w = (int(cloud.width) - flt.width_skip_begin - flt.width_skip_end) // flt.width_increment
        hgt = (int(cloud.height) - flt.height_skip_begin - flt.height_skip_end) // flt.height_increment
        self.model, self.n = None, w * hgt
        self.outdated = True


class RCCB200OnDn(RCCB200):
    """rmcl::RCCEmbreeOnDn twin (RCCEmbree.hpp:68-83)."""


class CPCB200(RCCB200):
    """rmcl::CPCEmbree twin (rmcl/include/rmcl/registration/CPCEmbree.hpp:20-54): closest-point correspondences.  find() runs one
    closest-point query per dataset point on the same map BVH (CPCEmbree.cpp:17-43); no sensor model.  computeCrossStatistics /
    correctOnce are the shared Correspondences_ code."""

    def __init__(self, map_: Map):
        super().__init__(map_)
        _chk(load_library().b2_rcc_set_correspondence_type(self._h, C.c_int(1)))

    def setModel(self, m):
        raise B2Error(-1, "CPCB200 has no sensor model (closest-point correspondences use the dataset points)")

    def setOptions(self, skip_masked=False):
        """skip_masked: do not query dataset points whose mask is 0 (the reference queries them and never uses the result)"""
        _chk(load_library().b2_rcc_set_cpc_options(self._h, C.c_int(int(skip_masked))))


# v1 names used by the legacy benchmarks (lidar_corrector_{embree,optix}_benchmark.cpp:86)
SphereCorrectorB200 = RCCB200Spherical
PinholeCorrectorB200 = RCCB200Pinhole
O1DnCorrectorB200 = RCCB200O1Dn
OnDnCorrectorB200 = RCCB200OnDn


def _sensor_args(sensors, Tbo, merge_weights):
    """-> (n, handle array, Tbo records, merge weights or None) of a multi-sensor call"""
    n = len(sensors)
    hs = (C.c_void_p * n)(*[s._h for s in sensors])
    Tb = np.ascontiguousarray(np.asarray(Tbo, TRANSFORM_DTYPE).reshape(n))
    w = None if merge_weights is None else np.ascontiguousarray(merge_weights, np.float64).reshape(n)
    return n, hs, Tb, w


def micp_correct_once(sensors, Tbo, Tom, iterations=5, convergence_progress=0.0, merge_weights=None, ranges=None):
    """MICPLocalizationNode::correctOnce over all sensors (micp_localization.cpp:899-984): `sensors` RCCB200 / CPCB200 handles on one device,
    `Tbo` one Transform per sensor, `merge_weights` the sensors' merge_weight_multiplier (MICPSensor.hpp:103), `ranges` optional per-sensor
    host scans (None entries keep the resident dataset).  -> (Tom_new, T_onew_oold, Cmerged_o)."""
    n, hs, Tb, w = _sensor_args(sensors, Tbo, merge_weights)
    keep, rp = [], None
    if ranges is not None:
        rp = (C.c_void_p * n)()
        for k, r in enumerate(ranges):
            if r is None:
                rp[k] = None
            elif hasattr(r, "data_ptr"):
                rp[k] = r.data_ptr()
            else:
                r = _f32(r).reshape(-1)
                keep.append(r)
                rp[k] = r.ctypes.data
    Tn, Td, Cm = np.zeros((), TRANSFORM_DTYPE), np.zeros((), TRANSFORM_DTYPE), np.zeros((), CROSS_STATS_DTYPE)
    _chk(load_library().b2_micp_correct_once(hs, _p(Tb), _p(w), rp, C.c_uint32(n), _p(_tf(Tom)), C.c_uint32(iterations), C.c_double(convergence_progress),
                                             _p(Tn), _p(Td), _p(Cm)))
    for s in sensors:
        s.outdated = False
    return Tn, Td, Cm


# b2_micp_step (rmcl_b200.h): one correction of a chain, what MICPSensorStats needs (micp_localization.cpp:1009-1015)
MICP_STEP_DTYPE = np.dtype([("Tom_new", TRANSFORM_DTYPE), ("T_onew_oold", TRANSFORM_DTYPE), ("Cmerged_o", CROSS_STATS_DTYPE),
                            ("convergence_progress", np.float64), ("valid_measurements", np.uint32), ("total_measurements", np.uint32)])
assert MICP_STEP_DTYPE.itemsize == 144


def micp_correct(sensors, Tbo, Tom, n_corrections=3, iterations=5, convergence_progress=0.0, merge_weights=None, adaptive_max_dist=True):
    """`n_corrections` x MICPLocalizationNode::correctOnce back to back on the device (micp_localization.cpp:856-1007; 3 is correct(), :847-854):
    each step traces at the pose the previous one produced and gates with the max_dist its convergence progress gives, without the host in
    between.  Runs on the sensors' resident datasets (setRanges / setDataset / bindDataset first).  -> (Tom, convergence_progress, steps) with
    `steps` a MICP_STEP_DTYPE record array, one per correction."""
    n, hs, Tb, w = _sensor_args(sensors, Tbo, merge_weights)
    T = np.array(_tf(Tom), copy=True)
    cp = C.c_double(float(convergence_progress))
    steps = np.zeros(int(n_corrections), MICP_STEP_DTYPE)
    _chk(load_library().b2_micp_correct(hs, _p(Tb), _p(w), C.c_uint32(n), _p(T), C.byref(cp), C.c_int(int(bool(adaptive_max_dist))),
                                        C.c_uint32(int(n_corrections)), C.c_uint32(int(iterations)), _p(steps) if len(steps) else None))
    for s in sensors:
        s.outdated = False
    return T, cp.value, steps


# b2_micp_covariance (rmcl_b200.h): the pose covariance of a correction and the information it comes from
MICP_COVARIANCE_DTYPE = np.dtype([("information", np.float64, 36), ("covariance", np.float64, 36), ("eigenvalues", np.float64, 6),
                                  ("eigenvectors", np.float64, 36), ("sigma2", np.float64), ("residual_sq_sum", np.float64), ("weight_sum", np.float64),
                                  ("length_scale", np.float64), ("n_pairs", np.uint64, 4), ("n_degenerate", np.uint32), ("degenerate_mask", np.uint32)])
assert MICP_COVARIANCE_DTYPE.itemsize == 984


class _MicpCovConfig(C.Structure):
    _fields_ = [("tau", C.c_double), ("degenerate_variance", C.c_double)]


def micp_pose_covariance(sensors, Tbo, T_onew_oold, convergence_progress=0.0, merge_weights=None, Tbo_ref=None, tau=1e-3, degenerate_variance=1e2):
    """The covariance of the correction that just ran on `sensors` (b2_micp_pose_covariance, SURVEY appendix I): from the point-to-plane
    information of the final correspondences, about Tom_new * Tbo_ref (default Tbo[0]) in its body frame, x y z roll pitch yaw.  Pass the
    correction's T_onew_oold and the progress it gated with (after micp_correct: steps[-1]["T_onew_oold"] and the input progress for one step,
    else steps[-2]["convergence_progress"]).  -> a MICP_COVARIANCE_DTYPE record."""
    n, hs, Tb, w = _sensor_args(sensors, Tbo, merge_weights)
    ref = None if Tbo_ref is None else _tf(np.asarray(Tbo_ref, TRANSFORM_DTYPE).reshape(()))
    cfg = _MicpCovConfig(float(tau), float(degenerate_variance))
    out = np.zeros((), MICP_COVARIANCE_DTYPE)
    _chk(load_library().b2_micp_pose_covariance(hs, _p(Tb), _p(w), C.c_uint32(n), _p(_tf(np.asarray(T_onew_oold, TRANSFORM_DTYPE).reshape(()))),
                                                C.c_double(float(convergence_progress)), _p(ref), C.byref(cfg), _p(out)))
    return out


def umeyama_transform(stats, device=0):
    """rm::umeyama_transform for an array of CrossStatistics (micp_localization.cpp:952-953)."""
    ps, n = _records(stats, 64, np.ascontiguousarray)
    out = np.zeros(n, TRANSFORM_DTYPE)
    _chk(load_library().b2_umeyama_batch(ps, C.c_uint32(n), _p(out), C.c_int(0), C.c_int(device), None))
    return out


class _DfieldParams(C.Structure):
    _fields_ = [("resolution", C.c_float), ("truncation", C.c_float), ("bb_min", C.c_void_p), ("bb_max", C.c_void_p)]


class _DfieldInfo(C.Structure):
    _fields_ = [("dims", C.c_uint32 * 3), ("brick_dims", C.c_uint32 * 3), ("origin", C.c_float * 3), ("resolution", C.c_float), ("inv_resolution", C.c_float),
                ("truncation", C.c_float), ("bricks_total", C.c_uint64), ("bricks_allocated", C.c_uint64), ("bytes", C.c_uint64), ("build_ms", C.c_float),
                ("device", C.c_int)]


class DistanceField:
    """Truncated distance field of a map (b2_dfield_*; AMCL's likelihood field): nodes every `resolution` m over [bb_min, bb_max] (default:
    the map's box grown by `truncation`) holding min(distance to the surface, truncation), stored as sparse 8^3-cell bricks.  Lookups are
    trilinear, within (sqrt(3)/2) * resolution of the clamped distance.  A snapshot of the map: rebuild it after Map.refit."""

    def __init__(self, map_: Map, resolution, truncation, bb_min=None, bb_max=None):
        self.map = map_                 # the library keeps its own reference too
        lo = None if bb_min is None else _f32(bb_min).reshape(3)
        hi = None if bb_max is None else _f32(bb_max).reshape(3)
        prm = _DfieldParams(float(resolution), float(truncation), None if lo is None else lo.ctypes.data, None if hi is None else hi.ctypes.data)
        h = C.c_void_p()
        _chk(load_library().b2_dfield_create(map_._h, C.byref(prm), C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            load_library().b2_dfield_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def info(self):
        inf = _DfieldInfo()
        _chk(load_library().b2_dfield_get_info(self._h, C.byref(inf)))
        out = {k: getattr(inf, k) for k, _ in _DfieldInfo._fields_}
        for k in ("dims", "brick_dims", "origin"):
            out[k] = tuple(out[k])
        return out

    def download(self):
        """-> (index uint32 (bz, by, bx): brick slot or 0xFFFFFFFF, bricks float32 (n_allocated, 9, 9, 9) indexed [z, y, x])"""
        inf = self.info()
        bx, by, bz = inf["brick_dims"]
        index = np.empty((bz, by, bx), np.uint32)
        bricks = np.empty((inf["bricks_allocated"], 9, 9, 9), np.float32)
        _chk(load_library().b2_dfield_download(self._h, _p(index), _p(bricks) if bricks.size else None))
        return index, bricks

    def query(self, points):
        """Lookups of (n, 3) points: numpy in, numpy out; a float32 CUDA tensor in, a CUDA tensor out (read in place)."""
        lib = load_library()
        if hasattr(points, "data_ptr"):
            import torch
            pts = points.reshape(-1, 3)
            out = torch.empty(pts.shape[0], dtype=torch.float32, device=pts.device)
            if pts.dtype != torch.float32:
                raise TypeError("expected a float32 tensor")
            _chk(lib.b2_dfield_query(self._h, _devptr(pts), C.c_uint32(pts.shape[0]), _devptr(out), C.c_int(1)))
            return out
        pts = _f32(points).reshape(-1, 3)
        out = np.empty(len(pts), np.float32)
        _chk(lib.b2_dfield_query(self._h, _p(pts), C.c_uint32(len(pts)), _p(out), C.c_int(0)))
        return out


class PCDSensorUpdaterB200:
    """Particle-filter sensor update: ParticleUpdater<MemT>::update (rmcl_ros/include/rmcl_ros/rmcl/ParticleUpdater.hpp:39-43) with the
    hot loop of PCDSensorUpdaterEmbree::update (PCDSensorUpdaterEmbree.cpp:290-342).  Its beams are drawn from the cloud of setInput
    (`samples` of them, keyed by `seed` and `step`; quirk D5) or passed to update()."""

    def __init__(self, map_: Map):
        self.map = map_
        h = C.c_void_p()
        _chk(load_library().b2_pf_create(map_._h, C.byref(h)))
        self._h = h
        self.config = PFParams.defaults()
        self.samples = 100              # PCDSensorUpdaterEmbree.cpp:124
        self.seed = 0                   # the same on every rank of a sharded particle set
        self.step = 0                   # advanced by every update() that samples the input
        self._input = None
        self._field = None
        self._stream = 0                # the handle's stream, as setStream last set it

    def close(self):
        if getattr(self, "_h", None):
            load_library().b2_pf_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def setStream(self, cuda_stream):
        _chk(load_library().b2_pf_set_stream(self._h, C.c_void_p(int(cuda_stream))))
        self._stream = int(cuda_stream)

    def setMapping(self, mode):
        """0 lanes = beams of one particle, 1 lanes = particles, 2 lanes = particles sorted by pose, 3 (default) auto by timing; results identical."""
        _chk(load_library().b2_pf_set_mapping(self._h, C.c_int(mode)))

    def mapping(self):
        mode, cur = C.c_int(0), C.c_int(0)
        _chk(load_library().b2_pf_get_mapping(self._h, C.byref(mode), C.byref(cur)))
        return mode.value, cur.value

    def sampleBeams(self, cloud, n_samples=None, seed=None, step=None):
        """PCDSensorUpdaterOptix::update's beam sampling (PCDSensorUpdaterOptix.cpp:227-311, b2_pf_sample_cloud): up to `n_samples` (default
        self.samples) beams drawn from the finite points of a PointCloud2-shaped `cloud`, keyed by (seed, step) (default self.seed / self.step),
        as a RANGE_MEAS_DTYPE array in merge order.  A CUDA uint8 tensor as cloud.data is read in place by a kernel; host data is read on the
        host where the draws land."""
        n = self.samples if n_samples is None else int(n_samples)
        L = cloud_layout(cloud)
        ptr, nbytes, dev = _cloud_buffer(cloud)
        out = np.zeros(n, RANGE_MEAS_DTYPE)
        got = C.c_uint32()
        _chk(load_library().b2_pf_sample_cloud(self._h, ptr, C.c_uint64(nbytes), C.byref(L), C.c_int(dev), C.c_uint32(n),
                                               C.c_uint64(self.seed if seed is None else int(seed)), C.c_uint32(self.step if step is None else int(step)),
                                               _p(out) if n else None, C.byref(got)))
        return out[: got.value]

    def setInput(self, cloud):
        """Input<PointCloud2::ConstSharedPtr>::setInput (rmcl_localization.cpp:512-530): the cloud the next update() samples its beams from.
        The reference is kept; the data is read when update() runs."""
        self._input = cloud

    def setDistanceField(self, field):
        """While a DistanceField is set, update() on CUDA tensors evaluates each beam from it (b2_pf_sensor_update_field) instead of tracing
        the map; update() on numpy arrays raises B2Error.  None returns to the map."""
        if field is not None and not isinstance(field, DistanceField):
            raise TypeError("expected a DistanceField or None")
        self._field = field

    def update(self, particle_poses, particle_attrs, Tsb, beams=None, params: PFParams | None = None, inplace=False):
        """RAM variant: numpy arrays in, updated attrs array out (inplace=True: the caller's attrs array is updated itself, as the reference's
        update(MemoryView) does -- no staging copy; pin the arrays and the transfers overlap the kernel).  VRAM variant: torch CUDA tensors, attrs
        updated in place.  beams=None: `samples` beams are drawn from the setInput cloud with (seed, step), then step advances by one."""
        prm = params or self.config
        dev = hasattr(particle_poses, "data_ptr")
        if self._field is not None and not dev:
            raise B2Error(-1, "update: a distance field is set; the field update takes CUDA tensors only")
        if inplace and not dev:
            assert isinstance(particle_attrs, np.ndarray) and particle_attrs.flags.c_contiguous and particle_attrs.flags.writeable
        attrs = particle_attrs if dev or inplace else np.ascontiguousarray(particle_attrs).copy()
        p, a, n = _agree("update", poses=(particle_poses, 32, None if dev else _tf), attrs=(attrs, 36, None if dev else np.ascontiguousarray))
        if beams is None:
            if self._input is None:
                raise B2Error(-1, "update: no beams and no input cloud (setInput first)")
            beams = self.sampleBeams(self._input)
            self.step += 1
        pb, nb = _records(beams, 64, np.ascontiguousarray)
        Tsb = _tf(Tsb)
        lib = load_library()
        if not dev:
            _chk(lib.b2_pf_sensor_update_host(self._h, p, a, C.c_uint32(n), _p(Tsb), pb, C.c_uint32(nb), C.byref(prm)))
        elif self._field is not None:
            _chk(lib.b2_pf_sensor_update_field(self._h, self._field._h, p, a, C.c_uint32(n), _p(Tsb), pb, C.c_uint32(nb), C.byref(prm)))
        else:
            _chk(lib.b2_pf_sensor_update(self._h, p, a, C.c_uint32(n), _p(Tsb), pb, C.c_uint32(nb), C.byref(prm)))
        return attrs

    def steinUpdate(self, particle_poses, Tsb, beams, config=None, params: PFParams | None = None, seed=None, step=0):
        """Stein variational steps toward the beams' likelihood over the distance field of setDistanceField (b2_pf_stein_update; SURVEY
        appendix L): in place on the (n, 8) float32 CUDA tensor of poses, on the handle's stream.  Each of config.iterations steps moves every
        particle in x, y and yaw along the kernel-weighted score of a reference set plus the kernel's repulsion; a step the map's walls block
        is not taken.  z, roll, pitch and the attributes stay: the next update() scores the moved particles.  `config`: a SteinConfig
        (default defaults()); `params`: the sensor model's dist_sigma (default self.config); `seed` (default self.seed) and `step` key the
        reference draws.  -> dict(bandwidth, n_ref, n_blocked, rms_step_t, rms_step_r), read back with a synchronise."""
        if self._field is None:
            raise B2Error(-1, "steinUpdate: no distance field (setDistanceField first)")
        cfg = config or SteinConfig.defaults()
        prm = params or self.config
        pb, nb = _records(beams, 64, np.ascontiguousarray)
        p, n = _records(particle_poses, 32)
        out = _SteinResult()
        _chk(load_library().b2_pf_stein_update(self._h, self._field._h, p, C.c_uint32(n), _p(_tf(Tsb)), pb if nb else None, C.c_uint32(nb), C.byref(prm),
                                               C.byref(cfg), C.c_uint64(self.seed if seed is None else int(seed)), C.c_uint32(int(step)), C.byref(out)))
        return {"bandwidth": tuple(out.bandwidth), "n_ref": out.n_ref, "n_blocked": out.n_blocked, "rms_step_t": out.rms_step_t,
                "rms_step_r": out.rms_step_r}

    def steinBegin(self, n_all, first, n_local, j_first, j_count, Tsb, beams, config=None, params: PFParams | None = None, seed=None, step=0):
        """Open a session of Stein steps on a slice of a set sharded over GPUs (b2_pf_stein_slice_begin; SURVEY L14): this rank moves the
        particles [first, first + n_local) of n_all and scores J's references [j_first, j_first + j_count).  Arguments as steinUpdate's.
        Uploads the beams (a synchronise); steinScore and steinMove then only launch kernels on the handle's stream."""
        if self._field is None:
            raise B2Error(-1, "steinBegin: no distance field (setDistanceField first)")
        cfg = config or SteinConfig.defaults()
        prm = params or self.config
        pb, nb = _records(beams, 64, np.ascontiguousarray)
        _chk(load_library().b2_pf_stein_slice_begin(self._h, self._field._h, C.c_uint32(n_all), C.c_uint32(first), C.c_uint32(n_local), C.c_uint32(j_first),
                                                    C.c_uint32(j_count), _p(_tf(Tsb)), pb if nb else None, C.c_uint32(nb),
                                                    C.byref(prm), C.byref(cfg), C.c_uint64(self.seed if seed is None else int(seed)), C.c_uint32(int(step))))

    def steinScore(self, poses_all, iteration, snap):
        """Iteration `iteration`'s score of the session's J range (b2_pf_stein_slice_score): poses_all the (n_all, 8) float32 CUDA tensor of
        the whole set, snap a float32 CUDA tensor whose first j_count rows of 6 (x, y, psi, gx, gy, gpsi) are written."""
        _chk(load_library().b2_pf_stein_slice_score(self._h, _devptr(poses_all), C.c_uint32(int(iteration)), _devptr(snap)))

    def steinMove(self, poses_all, snap_all, iteration, poses_out):
        """Iteration `iteration`'s bandwidth over poses_all and move of the session's slice against J's whole snapshot snap_all (m rows of 6)
        into poses_out (n_local rows of 8; may be poses_all[first:first + n_local]) (b2_pf_stein_slice_move)."""
        _chk(load_library().b2_pf_stein_slice_move(self._h, _devptr(poses_all), _devptr(snap_all), C.c_uint32(int(iteration)), _devptr(poses_out)))

    def steinResult(self):
        """The session's record (b2_pf_stein_slice_result, a synchronise): -> dict(bandwidth, n_ref, n_blocked, n_steps, sum_step_t2,
        sum_step_r2); n_blocked counts this slice over all iterations, the step count and sums cover its last iteration."""
        r = _SteinSliceResult()
        _chk(load_library().b2_pf_stein_slice_result(self._h, C.byref(r)))
        return {"bandwidth": tuple(r.bandwidth), "n_ref": r.n_ref, "n_blocked": r.n_blocked, "n_steps": r.n_steps, "sum_step_t2": r.sum_step_t2,
                "sum_step_r2": r.sum_step_r2}

    def steinUpdateSharded(self, poses_local, Tsb, beams, dist, config=None, params: PFParams | None = None, seed=None, step=0):
        """steinUpdate on a particle set sharded over ranks in equal contiguous slices (rank order = global order): poses_local, this rank's
        (n, 8) float32 CUDA tensor, moves in place.  Per iteration the poses (32 B per particle) and J's snapshot (24 B per reference) are
        all-gathered over `dist` (torch.distributed, nccl); the slices then equal steinUpdate of the whole set byte for byte.  `seed`
        (default self.seed) must be the same on every rank.  For the call the handle runs on torch's current stream, where the collectives
        run, so the iterations need no host synchronise; the handle's stream is restored afterwards.  -> steinUpdate's dict for the whole
        set: bandwidth and n_ref, n_blocked summed over ranks, the RMS steps from the summed squares."""
        import torch
        from .shard import stein_update_sharded
        cfg = config or SteinConfig.defaults()
        prev = self._stream
        self.setStream(torch.cuda.current_stream(poses_local.device).cuda_stream)
        try:
            return stein_update_sharded(
                lambda n_all, first, n_local, j_first, j_count: self.steinBegin(n_all, first, n_local, j_first, j_count, Tsb, beams, cfg, params, seed, step),
                self.steinScore, self.steinMove, self.steinResult, poses_local, dist, cfg.iterations, cfg.n_ref)
        finally:
            self.setStream(prev)

    def globalSearch(self, field, Tsb, beams, config=None, surface=None, params: PFParams | None = None, scores=None):
        """Where on the map does this scan fit best (b2_pf_global_search; SURVEY appendix M): every pose of `config`'s (x, y, yaw) grid (a
        SearchConfig; default: SearchConfig.defaults() over the DistanceField `field`'s (x, y) box at z0 = 0) is scored as update() from the
        field would score a particle there from {0, 0, 0}, the score array's local maxima are ranked, and those at least the config's
        separations from a better one are kept.  `surface` (a SurfaceConfig) puts each candidate where projectToSurface would; one off the
        surface scores -1.  `params`: the sensor model (default self.config).  `scores`: a float32 CUDA tensor of n_candidates elements that
        receives every score in candidate order (x fastest, yaw slowest), the likelihood map.  Synchronises.  -> (result, records): a dict
        (n_candidates, n_valid, n_peaks, n_records) and the kept peaks as a synth.SEARCH_RECORD_DTYPE array, records[0] the best."""
        if not isinstance(field, DistanceField):
            raise TypeError("expected a DistanceField")
        cfg = config
        if cfg is None:
            inf = field.info()
            hi = [inf["origin"][a] + (inf["dims"][a] - 1) * inf["resolution"] for a in range(2)]
            cfg = SearchConfig.defaults(inf["origin"][:2], hi)
        prm = params or self.config
        pb, nb = _records(beams, 64, np.ascontiguousarray)
        sp = None
        if scores is not None:
            sp, ns = _records(scores, 4)
            want = int(cfg.nx) * int(cfg.ny) * int(cfg.n_yaw)
            if ns != want:
                raise ValueError(f"globalSearch: {want} candidates but {ns} scores")
        recs = np.zeros(max(1, min(int(cfg.max_records), 64)), SEARCH_RECORD_DTYPE)
        out = _SearchResult()
        _chk(load_library().b2_pf_global_search(self._h, field._h, _p(_tf(Tsb)), pb if nb else None, C.c_uint32(nb), C.byref(prm), C.byref(cfg),
                                                 None if surface is None else C.byref(surface), _p(recs), sp, C.byref(out)))
        res = {k: int(getattr(out, k)) for k, _ in _SearchResult._fields_}
        return res, recs[:res["n_records"]]

    def globalSearchBnB(self, field, Tsb, beams, config=None, surface=None, params: PFParams | None = None, min_ratio=0.0):
        """globalSearch's records on grids too large or too fine to score exhaustively (b2_pf_global_search_bnb; SURVEY appendix N): an exact
        branch and bound over a quadtree per heading, bounded from a min-pooled pyramid of the field.  `field`, `Tsb`, `beams`, `config`,
        `surface` and `params` as for globalSearch; the grid may hold more than 2^30 candidates (nx, ny up to 2^24).  The records are
        globalSearch's records whose score is >= tau = min_ratio * s* (s* the best score of the grid), in the same order, byte for byte:
        min_ratio 0 gives all of them, 1 those that share the best score.  Synchronises.  -> (result, records): a dict (n_candidates,
        n_bounded, n_leaves, n_peaks, n_records, n_bounded_pass (one per pass), n_level (per tree level, 0 = leaves scored), best_score,
        threshold, n_passes, depth; the fields of synth.SEARCH_BNB_RESULT_DTYPE, n_bounded_pass cut to n_passes) and the records as a
        synth.SEARCH_RECORD_DTYPE array, records[0] the best."""
        if not isinstance(field, DistanceField):
            raise TypeError("expected a DistanceField")
        cfg = config
        if cfg is None:
            inf = field.info()
            hi = [inf["origin"][a] + (inf["dims"][a] - 1) * inf["resolution"] for a in range(2)]
            cfg = SearchConfig.defaults(inf["origin"][:2], hi)
        prm = params or self.config
        pb, nb = _records(beams, 64, np.ascontiguousarray)
        recs = np.zeros(max(1, min(int(cfg.max_records), 64)), SEARCH_RECORD_DTYPE)
        out = np.zeros((), SEARCH_BNB_RESULT_DTYPE)
        _chk(load_library().b2_pf_global_search_bnb(self._h, field._h, _p(_tf(Tsb)), pb if nb else None, C.c_uint32(nb), C.byref(prm), C.byref(cfg),
                                                     None if surface is None else C.byref(surface), C.c_float(min_ratio), _p(recs), _p(out)))
        res = {k: out[k].tolist() for k in SEARCH_BNB_RESULT_DTYPE.names}
        res["n_bounded_pass"] = res["n_bounded_pass"][:res["n_passes"]]
        return res, recs[:res["n_records"]]

    def motionUpdate(self, particle_poses, particle_attrs, T_bnew_bold, forget_rate, check_collision=False):
        """TFMotionUpdaterGPU (rmcl_ros/src/rmcl/particle_motion.cu:11-46): in place on torch CUDA tensors.  check_collision adds the CPU
        updater's wall check (TFMotionUpdaterCPU.cpp:17-50,205-216)."""
        p, a, n = _agree("motionUpdate", poses=(particle_poses, 32), attrs=(particle_attrs, 36))
        _chk(load_library().b2_pf_motion_update(self._h, p, a, C.c_uint32(n), _p(_tf(T_bnew_bold)), C.c_double(forget_rate), C.c_int(int(check_collision))))

    def projectToSurface(self, particle_poses, particle_attrs, config=None):
        """Keep the particles on the map's walkable surface (b2_pf_project_to_surface; the surface-constrained motion update of
        rmcl/docs/RMCL.md:72): in place on torch CUDA tensors, on the handle's stream.  Each particle is put on the first surface under it
        within `config`'s probe window whose slope is at most max_slope (and tilted onto it with align 1); one found no such surface keeps
        its pose and gets the likelihood {0, 0, 10000}, so the next resampling replaces it.  `config`: a SurfaceConfig (default: defaults())."""
        cfg = config or SurfaceConfig.defaults()
        p, a, n = _agree("projectToSurface", poses=(particle_poses, 32), attrs=(particle_attrs, 36))
        _chk(load_library().b2_pf_project_to_surface(self._h, p, a, C.c_uint32(n), C.byref(cfg)))

    def likelihoodStats(self, particle_attrs, dist=None):
        """compute_stats (rmcl_ros/src/rmcl/resampling.cu:41-92) of the local particles; with `dist` (torch.distributed, particles sharded
        across ranks) the 8 bytes are all-reduced (SUM / MAX) -- the only exchange step of the particle-filter cycle."""
        a, n = _records(particle_attrs, 36)
        s, m = C.c_float(), C.c_float()
        _chk(load_library().b2_pf_likelihood_stats(self._h, a, C.c_uint32(n), C.byref(s), C.byref(m)))
        s, m = s.value, m.value
        if dist is not None and dist.is_initialized() and dist.get_world_size() > 1:
            import torch
            dev = particle_attrs.device if dist.get_backend() == "nccl" else "cpu"
            ts = torch.tensor([s], dtype=torch.float64, device=dev)
            tm = torch.tensor([m], dtype=torch.float64, device=dev)
            dist.all_reduce(ts, op=dist.ReduceOp.SUM)
            dist.all_reduce(tm, op=dist.ReduceOp.MAX)
            s, m = float(ts[0]), float(tm[0])
        return s, m

    def initSamplesUniform(self, particle_poses, particle_attrs, bb_min, bb_max, seed, first=0):
        """RmclNode::initSamplesUniform (rmcl_ros/src/nodes/rmcl_localization.cpp:277-342) on the device: fills the caller's (n, 8) / (n, 9)
        float32 CUDA tensors in place with particles first .. first+n-1 of a set drawn uniformly from the box (x, y, z, roll, pitch, yaw)."""
        lo, hi = np.ascontiguousarray(bb_min, np.float64).reshape(6), np.ascontiguousarray(bb_max, np.float64).reshape(6)
        p, a, n = _agree("initSamplesUniform", poses=(particle_poses, 32), attrs=(particle_attrs, 36))
        _chk(load_library().b2_pf_init_uniform(self._h, p, a, C.c_uint32(first), C.c_uint32(n), _p(lo), _p(hi), C.c_uint64(seed)))
        return particle_poses, particle_attrs

    def initSamples(self, particle_poses, particle_attrs, pose, cov, seed, first=0):
        """RmclNode::initSamples(PoseWithCovarianceStamped) (rmcl_localization.cpp:165-275) on the device: `pose` is the message pose (a
        Transform record), `cov` its 36 covariance entries (row-major); the noise acts in the pose frame.  Fills the tensors in place."""
        T = _tf(pose).reshape(())
        c = np.ascontiguousarray(cov, np.float64).reshape(36)
        p, a, n = _agree("initSamples", poses=(particle_poses, 32), attrs=(particle_attrs, 36))
        _chk(load_library().b2_pf_init_gaussian(self._h, p, a, C.c_uint32(first), C.c_uint32(n), _p(T), _p(c), C.c_uint64(seed)))
        return particle_poses, particle_attrs

    def estimateStats(self, particle_poses, particle_attrs, max_induction_particles=50000):
        """RmclNode::estimateStats (rmcl_ros/src/nodes/rmcl_localization.cpp:642-731) on the device: the statistics of the first
        min(n, max_induction_particles) particles of the (n, 8) / (n, 9) float32 CUDA tensors, as a synth.PARTICLE_STATS_DTYPE record (the
        fields of rmcl_msgs/ParticleStats): likelihood statistics, translation bounds, the weighted Markley mean pose and its 6x6 covariance."""
        p, a, n = _agree("estimateStats", poses=(particle_poses, 32), attrs=(particle_attrs, 36))
        k = max(0, min(n, int(max_induction_particles)))
        out = np.zeros((), PARTICLE_STATS_DTYPE)
        _chk(load_library().b2_pf_estimate_stats(self._h, p, a, C.c_uint32(k), _p(out)))
        return out

    def estimateClusters(self, particle_poses, particle_attrs, config=None, labels=None):
        """The filter's pose hypotheses (b2_pf_cluster_stats; AMCL's cluster statistics) of the (n, 8) / (n, 9) float32 CUDA tensors: the
        particles of likelihood > 0 are binned as resampleKLD bins them, touching bins are joined, and the clusters are ranked by weight.
        `config` is a ClusterConfig; `labels`, if given, is an n-element int32 / uint32 CUDA tensor that receives every particle's rank
        (0xFFFFFFFF: in no cluster).  -> (result, records): a synth.CLUSTER_RESULT_DTYPE record (n_clusters, n_records, bins, n_clustered,
        weight_total, rounds, weight_sum, weight_max) and the n_records heaviest clusters as synth.CLUSTER_RECORD_DTYPE, records[0] the
        best hypothesis: its share `weight` of the set, and in `stats` what estimateStats gives of its members alone."""
        cfg = config or ClusterConfig.defaults()
        p, a, lab, n = _agree("estimateClusters", poses=(particle_poses, 32), attrs=(particle_attrs, 36), labels=(labels, 4))
        out = np.zeros((), CLUSTER_RESULT_DTYPE)
        recs = np.zeros(max(1, min(int(cfg.max_records), 16)), CLUSTER_RECORD_DTYPE)
        _chk(load_library().b2_pf_cluster_stats(self._h, p, a, C.c_uint32(n), C.byref(cfg), _p(recs), lab, _p(out)))
        return out, recs[:int(out["n_records"])]

    def recoveryReset(self):
        """Zero the recovery's record {w_slow, w_fast, p_inject} (b2_pf_recovery_reset), on the handle's stream.  Call it after
        (re)initialising the set: initSamples and initSamplesUniform leave the record as it is."""
        _chk(load_library().b2_pf_recovery_reset(self._h))

    def recoveryObserve(self, particle_attrs, cfg=None, want_state=False):
        """Augmented MCL's averages (b2_pf_recovery_observe): call once after each update(), on the whole (n, 9) float32 CUDA tensor of
        attributes (a sharded set passes the all-gathered set).  The slow and the fast average of the set's mean likelihood follow it at
        `cfg`'s rates (a RecoveryConfig, default defaults()), and p_inject = max(0, 1 - w_fast / w_slow) is kept on the device for
        recoveryInject.  want_state: -> a synth.RECOVERY_STATE_DTYPE record (w_avg, w_slow, w_fast, p_inject), read back with a
        synchronise; otherwise the call only enqueues and returns None."""
        c = cfg or RecoveryConfig.defaults()
        a, n = _records(particle_attrs, 36)
        out = np.zeros((), RECOVERY_STATE_DTYPE) if want_state else None
        _chk(load_library().b2_pf_recovery_observe(self._h, a, C.c_uint32(n), C.byref(c), _p(out)))
        return out

    def recoveryInject(self, particle_poses, particle_attrs, bb_min, bb_max, surface=None, max_tries=16, seed=1234, step=0, first=0, want_result=False):
        """Augmented MCL's injection (b2_pf_recovery_inject): call after resampling.  In place on the (n, 8) / (n, 9) float32 CUDA tensors,
        particles first .. first+n-1 of the set: each is replaced with the probability p_inject of the last recoveryObserve by a pose drawn
        uniformly from the box (x, y, z, roll, pitch, yaw) as initSamplesUniform draws it; with `surface` (a SurfaceConfig) a candidate is
        taken only where projectToSurface finds ground, as it moves it, and up to max_tries candidates are drawn.  A replaced particle has
        the likelihood {0, 0, 0}: no weight until the next update() evaluates it.  After an injection the averages restart from 0.
        want_result: -> a synth.RECOVERY_RESULT_DTYPE record (p_inject, n_replaced, n_failed), read back with a synchronise; otherwise the
        call only enqueues and returns None."""
        lo, hi = np.ascontiguousarray(bb_min, np.float64).reshape(6), np.ascontiguousarray(bb_max, np.float64).reshape(6)
        p, a, n = _agree("recoveryInject", poses=(particle_poses, 32), attrs=(particle_attrs, 36))
        out = np.zeros((), RECOVERY_RESULT_DTYPE) if want_result else None
        _chk(load_library().b2_pf_recovery_inject(self._h, p, a, C.c_uint32(first), C.c_uint32(n), _p(lo), _p(hi), None if surface is None else C.byref(surface),
                                                  C.c_uint32(max_tries), C.c_uint64(seed), C.c_uint32(step), _p(out)))
        return out

    def gladiatorRandoms(self, seed, step, first, n, device=None):
        """The draws resample() uses for champions first..first+n-1 (raw u32 opponent word + 6 normals each), as torch CUDA tensors."""
        import torch
        dev = device if device is not None else torch.device("cuda", self.map.device)
        raw = torch.empty(n, dtype=torch.int32, device=dev)
        nrm = torch.empty((n, 6), dtype=torch.float32, device=dev)
        _chk(load_library().b2_pf_gladiator_randoms(self._h, C.c_uint64(seed), C.c_uint32(step), C.c_uint32(first), C.c_uint32(n), _devptr(raw), _devptr(nrm)))
        return raw, nrm

    def resample(self, particle_poses, particle_attrs, particle_poses_new, particle_attrs_new, config=None, seed=1234, step=0, first=0, raw=None, normals=None):
        """GladiatorResamplerGPU::resample (rmcl_ros/src/rmcl/resampling.cu:108-221) on torch CUDA tensors.  `particle_poses/attrs` hold all
        particles opponents are drawn from; the outputs receive champions first .. first+len(out)-1 (single GPU: first = 0, same length)."""
        cfg = config or GladiatorConfig.defaults()
        p, a, n_all = _agree("resample", poses=(particle_poses, 32), attrs=(particle_attrs, 36))
        pn, an, r, nrm, n_local = _agree("resample", poses_new=(particle_poses_new, 32), attrs_new=(particle_attrs_new, 36), raw=(raw, 4), normals=(normals, 24))
        _chk(load_library().b2_pf_resample_gladiator(self._h, p, a, C.c_uint32(n_all), C.c_uint32(first), C.c_uint32(n_local), pn, an, C.byref(cfg),
                                                     C.c_uint64(seed), C.c_uint32(step), r, nrm))
        return particle_poses_new, particle_attrs_new

    def resampleResidual(self, particle_poses, particle_attrs, particle_poses_new, particle_attrs_new, config=None, seed=1234, step=0, first=0, n_new=None):
        """ResidualResamplerCPU::update (rmcl_ros/src/rmcl/ResidualResamplerCPU.cpp:55-202) on torch CUDA tensors (b2_pf_resample_residual).
        Resamples all particles of `particle_poses/attrs` into an output set of n_new slots (default: the length of the outputs); the outputs
        receive slots first .. first+len(out)-1, and entries at or beyond the result's n_particles are left untouched.  `config` is a
        GladiatorConfig (the same fields and defaults).  -> a synth.RESIDUAL_RESULT_DTYPE record: n_particles, draws, weight_sum, weight_max."""
        cfg = config or GladiatorConfig.defaults()
        p, a, n = _agree("resampleResidual", poses=(particle_poses, 32), attrs=(particle_attrs, 36))
        pn, an, n_local = _agree("resampleResidual", poses_new=(particle_poses_new, 32), attrs_new=(particle_attrs_new, 36))
        n_new = first + n_local if n_new is None else int(n_new)
        out = np.zeros((), RESIDUAL_RESULT_DTYPE)
        _chk(load_library().b2_pf_resample_residual(self._h, p, a, C.c_uint32(n), C.c_uint32(n_new), C.c_uint32(first), C.c_uint32(n_local), pn, an,
                                                    C.byref(cfg), C.c_uint64(seed), C.c_uint32(step), _p(out)))
        return out

    def resampleKLD(self, particle_poses, particle_attrs, particle_poses_new, particle_attrs_new, kld=None, config=None, seed=1234, step=0, first=0, n_max=None):
        """KLD-sampling (Fox 2003; b2_pf_resample_kld) on torch CUDA tensors: all particles of `particle_poses/attrs` are resampled into an
        output set of at most n_max slots (default: the length of the outputs), as many as the bins the drawn set occupies call for; the
        outputs receive slots first .. first+len(out)-1, and entries at or beyond the result's n_particles are left untouched.  `kld` is a
        KLDConfig, `config` a GladiatorConfig (the copies' noise and forget factors).  -> a synth.KLD_RESULT_DTYPE record: n_particles, bins,
        weight_sum, weight_max."""
        kcfg = kld or KLDConfig.defaults()
        cfg = config or GladiatorConfig.defaults()
        p, a, n = _agree("resampleKLD", poses=(particle_poses, 32), attrs=(particle_attrs, 36))
        pn, an, n_local = _agree("resampleKLD", poses_new=(particle_poses_new, 32), attrs_new=(particle_attrs_new, 36))
        n_max = first + n_local if n_max is None else int(n_max)
        out = np.zeros((), KLD_RESULT_DTYPE)
        _chk(load_library().b2_pf_resample_kld(self._h, p, a, C.c_uint32(n), C.c_uint32(n_max), C.c_uint32(first), C.c_uint32(n_local), pn, an,
                                               C.byref(cfg), C.byref(kcfg), C.c_uint64(seed), C.c_uint32(step), _p(out)))
        return out

    def p2pConnect(self, dist, n_per_rank):
        """Map the other ranks' particle exchange buffers over NVLink (CUDA IPC): once per particle-set size.  Raises B2Error if the GPUs have no
        peer access or CUDA IPC is unavailable (the caller then stays with resampleSharded's all-gather)."""
        import torch
        ws, rank = dist.get_world_size(), dist.get_rank()
        mine = np.zeros(128, np.uint8)
        _chk(load_library().b2_pf_p2p_init(self._h, C.c_uint32(n_per_rank), _p(mine)))
        dev = torch.device("cuda", self.map.device) if dist.get_backend() == "nccl" else "cpu"
        allh = [torch.zeros(128, dtype=torch.uint8, device=dev) for _ in range(ws)]
        dist.all_gather(allh, torch.from_numpy(mine).to(dev))
        table = np.ascontiguousarray(torch.stack(allh).cpu().numpy())
        _chk(load_library().b2_pf_p2p_connect(self._h, _p(table), C.c_uint32(ws), C.c_uint32(rank), C.c_uint32(n_per_rank)))
        self._p2p = (ws, rank, n_per_rank)

    def resampleShardedP2P(self, poses_local, attrs_local, dist, config=None, seed=1234, step=0, want_traffic=False):
        """Gladiator resampling over peer memory (b2_pf_resample_gladiator_p2p): publish the shard, barrier, one kernel that reads opponents'
        likelihoods (4 B) and winners' records (68 B) from the owners' HBM, barrier.  -> (poses_new, attrs_new[, remote bytes read])"""
        import torch
        cfg = config or GladiatorConfig.defaults()
        n = poses_local.shape[0]
        if getattr(self, "_p2p", None) is None or self._p2p[2] != n:
            raise B2Error(-1, "resampleShardedP2P: call p2pConnect(dist, n_per_rank) first")
        _chk(load_library().b2_pf_p2p_publish(self._h, _devptr(poses_local), _devptr(attrs_local), C.c_uint32(n)))
        dist.barrier()
        P_new, A_new = torch.empty_like(poses_local), torch.empty_like(attrs_local)
        t = C.c_uint64()
        _chk(load_library().b2_pf_resample_gladiator_p2p(self._h, _devptr(P_new), _devptr(A_new), C.byref(cfg), C.c_uint64(seed), C.c_uint32(step),
                                                         C.byref(t) if want_traffic else None))
        torch.cuda.synchronize(poses_local.device)
        dist.barrier()                      # nobody overwrites a published shard while a peer may still read it
        return (P_new, A_new, int(t.value)) if want_traffic else (P_new, A_new)

    def resampleP2PLocalWorld(self, poses_all, attrs_all, world, rank, config=None, seed=1234, step=0):
        """test hook: `world` equal shards on ONE device; this handle plays `rank`.  -> (poses_new, attrs_new, bytes read from "remote" shards)"""
        import torch
        cfg = config or GladiatorConfig.defaults()
        n_all = poses_all.shape[0]
        n = n_all // world
        _chk(load_library().b2_pf_p2p_connect_local(self._h, _devptr(poses_all), _devptr(attrs_all), C.c_uint32(world), C.c_uint32(rank), C.c_uint32(n)))
        P_new = torch.empty((n, 8), dtype=torch.float32, device=poses_all.device)
        A_new = torch.empty((n, 9), dtype=torch.float32, device=poses_all.device)
        t = C.c_uint64()
        _chk(load_library().b2_pf_resample_gladiator_p2p(self._h, _devptr(P_new), _devptr(A_new), C.byref(cfg), C.c_uint64(seed), C.c_uint32(step), C.byref(t)))
        return P_new, A_new, int(t.value)

    def resampleSharded(self, poses_local, attrs_local, dist, config=None, seed=1234, step=0):
        """Particles sharded over ranks (equal contiguous slices in rank order): all-gather the particle set (the exchange step of this
        stage: 68 B per particle over NVLink), then every rank resamples its own champions against GLOBAL opponents.  Draws are keyed by the
        global particle index, so the result equals the single-GPU resample of the concatenated set.  (n, 8) / (n, 9) float32 CUDA tensors."""
        import torch
        from .shard import gladiator_resample_sharded

        def run(P_all, A_all, first, n_local):
            P_new, A_new = torch.empty_like(poses_local), torch.empty_like(attrs_local)
            return self.resample(P_all, A_all, P_new, A_new, config, seed, step, first=first)

        return gladiator_resample_sharded(run, poses_local, attrs_local, dist, sync=lambda: torch.cuda.synchronize(poses_local.device))
