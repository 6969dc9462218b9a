"""GPU tests of b2_rcc_set_cloud_spherical / RCCB200Spherical.setPointCloud: the device conversion of a PointCloud2 into the spherical model
equals the C restatement of tests/pc2_scan_ref bit for bit; corrections and segmentation after it equal those after set_ranges fed with the
restated ranges; the find's tile schedule survives a cloud; the key buffer resets itself; refusals change nothing; the C++ adapter matches
the Python path."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import pc2_scan_ref as ref
import rmcl_b200
from pc2_ref import same_bits
from conftest import gpu_map
from rmcl_b200 import synth
from rmcl_b200.api import B2_CLOUD_NO_FIELD, cloud_layout

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAP = "cube29"
TGT = synth.make_transform((0.7, -0.4, 0.3), (0.02, -0.03, 0.4))
T_SC = synth.make_transform((0.05, -0.02, 0.1), (0.0, 0.02, -0.6))          # a cloud frame rotated and offset against the sensor


def _lib():
    return rmcl_b200.load_library()


def _scan_points(W, H, seed=0):
    """sensor-frame points of a W x H spherical scan of the cube map at TGT (C2's elevations; misses NaN), a few (0,0,0) and inf points"""
    c2 = synth.c2_sensor()
    m = synth.SphericalModel(c2.phi_min, c2.phi_inc * (c2.phi_size - 1) / max(H - 1, 1), H, -math.pi, 2 * math.pi / W, W, 0.5, 12.0)
    h = rmcl_b200.RCCB200Spherical(gpu_map(MAP))
    h.setModel(m)
    h.find(TGT)
    p = h.modelView()["points"].astype(np.float64)
    rng = np.random.default_rng(seed)
    k = rng.permutation(len(p))
    p[k[: max(1, len(p) // 500)]] = 0.0
    p[k[len(p) // 500: len(p) // 250], 1] = np.inf
    return p


def _c2(range_max=12.0):
    m = synth.c2_sensor()
    m.range_max = range_max
    return m


def _ranges(h):
    n = C.c_uint32()
    assert _lib().b2_rcc_debug_model_tables(h._h, None, None, C.byref(n)) == 0
    r = np.zeros(n.value, np.float32)
    assert _lib().b2_rcc_debug_model_tables(h._h, None, C.c_void_p(r.ctypes.data), C.byref(n)) == 0
    return r


def _perm(h):
    n = C.c_uint32()
    assert _lib().b2_rcc_debug_tile_perm(h._h, None, 0, C.byref(n)) == 0
    out = np.zeros(max(n.value, 1), np.uint16)
    assert _lib().b2_rcc_debug_tile_perm(h._h, C.c_void_p(out.ctypes.data), C.c_uint32(len(out)), C.byref(n)) == 0
    return out[: n.value]


def _got(h):
    ds = h.datasetView()
    return dict(ranges=_ranges(h), points=ds["points"], mask=ds["mask"])


def _handle(m, cls=rmcl_b200.RCCB200Spherical):
    h = cls(gpu_map(MAP))
    h.setModel(m)
    return h


def _feed(h, c, T, src):
    import torch
    host = c.data
    if src == "pinned":
        c.data = torch.from_numpy(host).pin_memory()
    elif src == "device":
        c.data = torch.from_numpy(host).cuda()
    try:
        h.setPointCloud(c, T)
    finally:
        c.data = host


def _cases():
    rng = np.random.default_rng(3)
    c2 = _c2()
    p2048 = _scan_points(2048, 128, 1)                                      # two points per C2 cell
    yield "c2_128x2048", c2, synth.pointcloud2(p2048, 2048, 128), None
    q = p2048[rng.permutation(len(p2048))]
    yield "unorganised_shuffled", c2, synth.pointcloud2(q, len(q), 1, point_step=32, offsets=(16, 4, 24)), None
    yield "one_cell", synth.SphericalModel(0.0, 0.0, 1, 0.0, 0.0, 1, 0.5, 12.0), synth.pointcloud2(p2048[:50000], 50000, 1), None
    for n in (0, 1, 255, 256, 257):
        yield f"n{n}", c2, synth.pointcloud2(p2048[rng.permutation(len(p2048))[:n]], n, 1), None
    p = _scan_points(1024, 64, 2)
    yield "f64_unaligned_padded_T", c2, synth.pointcloud2(p, 1024, 64, dtype=np.float64, point_step=48, offsets=(1, 13, 27), row_pad=5,
                                                          extra={"intensity": 41}), T_SC
    yield "f32_unaligned_padded", c2, synth.pointcloud2(p, 1024, 64, point_step=23, offsets=(9, 2, 17), row_pad=3), None


def test_cloud_matches_restatement():
    for name, m, c, T in _cases():
        want = ref.convert(c, m, T)
        h = _handle(m)
        for src in ("pageable", "pinned", "device"):
            _feed(h, c, T, src)
            assert ref.same(_got(h), want), (name, src)
        if name == "c2_128x2048":
            assert int(want["mask"].sum()) > 50000


def _pair(m, c, T=None, cls=rmcl_b200.RCCB200Spherical):
    want = ref.convert(c, m, T)
    a, b = _handle(m, cls), _handle(m, cls)
    a.setPointCloud(c, T)
    b.setRanges(want["ranges"])
    return a, b, want


def _bits(*xs):
    return b"".join(np.asarray(x).tobytes() for x in xs)


def test_corrections_and_segmentation_equal_the_ranges_path():
    m = _c2()
    c = synth.pointcloud2(_scan_points(1024, 128, 4), 1024, 128, dtype=np.float64, point_step=32, offsets=(0, 8, 16))
    a, b, want = _pair(m, c)
    assert ref.same(_got(a), _got(b))
    Tguess = synth.compose(TGT, synth.make_transform((0.1, -0.05, 0.02), (0.0, 0.01, -0.03)))
    I = synth.make_transform()
    for cp in (0.0, 0.4):
        ra, rb = a.correctOnce(Tguess, I, 5, cp), b.correctOnce(Tguess, I, 5, cp)
        assert _bits(*ra) == _bits(*rb) and ra[2]["n_meas"] > 1000
    a.find(TGT)
    b.find(TGT)
    assert _bits(*a.segment(0.15, 0.15)) == _bits(*b.segment(0.15, 0.15))
    # two sensors: the cloud-fed spherical sensor with an O1Dn one fed from its own cloud
    o = rmcl_b200.RCCB200O1Dn(gpu_map(MAP))
    o.setPointCloud(synth.pointcloud2(_scan_points(256, 16, 5), 256, 16), rmcl_b200.O1DnCloudFilter.defaults(0.3, 12.0))
    Tbo = np.stack([synth.make_transform(), synth.make_transform((0.1, 0.0, 0.05))])
    for w in (None, [1.0, 0.5]):
        ra = rmcl_b200.micp_correct_once([a, o], Tbo, Tguess, 5, 0.0, merge_weights=w)
        rb = rmcl_b200.micp_correct_once([b, o], Tbo, Tguess, 5, 0.0, merge_weights=w)
        assert _bits(*ra) == _bits(*rb)
    for sa_, sb_ in (([a], [b]), ([a, o], [b, o])):
        Tb = Tbo[: len(sa_)]
        ta, cpa, sa = rmcl_b200.micp_correct(sa_, Tb, Tguess, n_corrections=3)
        tb, cpb, sb = rmcl_b200.micp_correct(sb_, Tb, Tguess, n_corrections=3)
        assert _bits(ta, sa) == _bits(tb, sb) and cpa == cpb
    assert sa["valid_measurements"][0] == int(want["mask"].sum()) + int(o.datasetView()["mask"].sum())


def test_closest_point_handle_with_a_spherical_model():
    """a handle switched to closest-point correspondences (B2_CORR_CPC) keeps its spherical model, and the cloud fills its dataset the same way"""
    m = _c2()
    c = synth.pointcloud2(_scan_points(1024, 32, 6), 1024, 32)
    a, b, want = _pair(m, c, T_SC)
    for x in (a, b):
        assert _lib().b2_rcc_set_correspondence_type(x._h, C.c_int(1)) == 0
    a.setPointCloud(c, T_SC)
    assert ref.same(_got(a), want)
    Tguess = synth.compose(TGT, synth.make_transform((0.05, 0.02, 0.0), (0.0, 0.0, 0.02)))
    I = synth.make_transform()
    assert _bits(*a.correctOnce(Tguess, I, 5, 0.0)) == _bits(*b.correctOnce(Tguess, I, 5, 0.0))


def test_tile_schedule_survives_a_cloud_and_keys_reset_themselves():
    m = _c2()
    c1 = synth.pointcloud2(_scan_points(2048, 128, 7), 2048, 128)
    p2 = _scan_points(1024, 128, 8)
    c2 = synth.pointcloud2(p2[: 1024 * 40], 1024, 40, point_step=48, offsets=(8, 16, 24))     # fewer points: stale keys would show
    I = synth.make_transform()
    Tguess = synth.compose(TGT, synth.make_transform((0.05, 0.05, 0.0), (0.0, 0.0, 0.02)))
    h = _handle(m)
    h.setPointCloud(c1)
    h.correctOnce(Tguess, I, 5, 0.0)
    P1 = _perm(h)
    assert len(P1) == 128 * 1024 // 32 and not np.array_equal(P1, np.arange(len(P1)))
    h.setPointCloud(c2)
    assert np.array_equal(_perm(h), P1)                                     # the model did not change, neither did its schedule
    assert ref.same(_got(h), ref.convert(c2, m))                             # back to back = the second cloud alone
    fresh = _handle(m)
    fresh.setPointCloud(c2)
    assert ref.same(_got(h), _got(fresh))
    h.setPointCloud(c2)
    h.setPointCloud(c2)
    assert ref.same(_got(h), _got(fresh))
    h.setModel(m)                                                           # a later set_model_* still resets it
    assert len(_perm(h)) == 0


def _refuse(h, c, L=None, nbytes=None, T=None, data=True):
    T = synth.make_transform() if T is None else T
    L = cloud_layout(c) if L is None else L
    ptr = C.c_void_p(c.data.ctypes.data) if data else None
    return _lib().b2_rcc_set_cloud_spherical(h._h, ptr, C.c_uint64(c.data.size if nbytes is None else nbytes), C.byref(L),
                                             C.c_void_p(T.ctypes.data), C.c_int(0))


def test_refusals_change_nothing():
    m = _c2()
    c = synth.pointcloud2(_scan_points(1024, 32, 9), 1024, 32, dtype=np.float64, point_step=32, offsets=(0, 8, 16))
    h = _handle(m)
    h.setPointCloud(c)
    h.correctOnce(TGT, synth.make_transform(), 5, 0.0)
    g0, perm0 = _got(h), _perm(h)
    assert len(perm0) > 0
    n0 = rmcl_b200.kernel_launch_count()
    cases = []
    for k in "xyz":
        L = cloud_layout(c)
        setattr(L, "offset_" + k, B2_CLOUD_NO_FIELD)
        cases.append(dict(L=L))
    for dt, big in ((2, 0), (9, 0), (8, 1)):
        L = cloud_layout(c)
        L.datatype, L.is_bigendian = dt, big
        cases.append(dict(L=L))
    L = cloud_layout(c)
    L.offset_z = 25
    cases.append(dict(L=L))
    cases.append(dict(nbytes=(c.height - 1) * c.row_step + (c.width - 1) * c.point_step + 24 - 1))
    L = cloud_layout(c)
    L.width, L.height = 0x10000, 0x10000
    cases.append(dict(L=L))
    T = synth.make_transform()
    T["t"][2] = np.nan
    cases.append(dict(T=T))
    cases.append(dict(data=False))
    for kw in cases:
        assert _refuse(h, c, **kw) == -1, kw
    assert rmcl_b200.kernel_launch_count() == n0
    assert ref.same(_got(h), g0) and np.array_equal(_perm(h), perm0)
    # handles whose current model is not spherical, or a spherical model the cloud cannot be binned into
    others = [rmcl_b200.RCCB200Spherical(gpu_map(MAP)), _handle(synth.c4_sensor(), rmcl_b200.RCCB200Pinhole)]
    o = rmcl_b200.RCCB200O1Dn(gpu_map(MAP))
    o.setPointCloud(synth.pointcloud2(_scan_points(64, 8, 1), 64, 8))
    others.append(o)
    s = _handle(m)
    s.setModel(synth.O1DnModel(4, 2, np.zeros(3, np.float32), np.tile([1.0, 0.0, 0.0], (8, 1)).astype(np.float32), 0.3, 12.0))
    others.append(s)
    for bad in (synth.SphericalModel(0.0, 0.0, 2, 0.0, 0.1, 8, 0.5, 12.0), synth.SphericalModel(0.0, 0.1, 2, 0.0, 0.0, 8, 0.5, 12.0),
                synth.SphericalModel(0.0, 0.1, 2, 0.0, 0.1, 8, 0.5, np.inf), synth.SphericalModel(np.nan, 0.1, 2, 0.0, 0.1, 8, 0.5, 12.0)):
        others.append(_handle(bad))
    before = [x.datasetView() for x in others]
    n1 = rmcl_b200.kernel_launch_count()
    for k, x in enumerate(others):
        assert _refuse(x, c) == -1
        msg = _lib().b2_last_error().decode()
        assert ("not spherical" in msg) if k < 4 else ("increment 0" in msg or "non-finite" in msg), (k, msg)
    assert rmcl_b200.kernel_launch_count() == n1
    for x, b in zip(others, before):
        a = x.datasetView()
        assert same_bits(a["points"], b["points"]) and np.array_equal(a["mask"], b["mask"])
    assert _lib().b2_peek_cuda_error().decode() == ""


def test_cpp_adapter_matches_python(tmp_path):
    """tests/pointcloud_scan_cpp: unpackPointCloud into an RCCB200Spherical over PointCloud2-shaped structs, then correctOnce -- byte for
    byte the Python path"""
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "pointcloud_scan_cpp")
    lib_dir = os.path.dirname(rmcl_b200.lib_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "pointcloud_scan_cpp", "pointcloud_scan_cpp.cpp"), "-L" + lib_dir, "-lrmcl_b200",
                           "-L" + os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + lib_dir])
    from conftest import mesh
    V, F = mesh(MAP)
    with open(tmp_path / "map.bin", "wb") as f:
        np.array([len(V), len(F)], np.uint32).tofile(f)
        V.astype(np.float32).tofile(f)
        F.astype(np.uint32).tofile(f)
    m = _c2()
    c = synth.pointcloud2(_scan_points(1024, 64, 3), 1024, 64, dtype=np.float64, point_step=48, offsets=(3, 17, 29), row_pad=6, extra={"intensity": 44})
    with open(tmp_path / "cloud.bin", "wb") as f:
        np.array([c.width, c.height, c.point_step, c.row_step, 0, len(c.fields)], np.uint32).tofile(f)
        for fl in c.fields:
            f.write(fl.name.encode().ljust(16, b"\0"))
            np.array([fl.offset, fl.datatype], np.uint32).tofile(f)
        np.array([m.phi_min, m.phi_inc], np.float32).tofile(f)
        np.array([m.phi_size], np.uint32).tofile(f)
        np.array([m.theta_min, m.theta_inc], np.float32).tofile(f)
        np.array([m.theta_size], np.uint32).tofile(f)
        np.array([m.range_min, m.range_max], np.float32).tofile(f)
        np.asarray(T_SC).tofile(f)
        np.asarray(TGT).tofile(f)
        c.data.tofile(f)
    out = subprocess.run([exe, str(tmp_path / "map.bin"), str(tmp_path / "cloud.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "REFUSED setPointCloud" in out.stdout and "no x, y or z field" in out.stdout
    h = _handle(m)
    h.setPointCloud(c, T_SC)
    ds = h.datasetView()
    I = synth.make_transform()
    Tn, _, _ = h.correctOnce(TGT, I, 5, 0.0)
    assert (tmp_path / "out.bin").read_bytes() == _bits(ds["points"], ds["mask"], Tn)
    assert ref.same(_got(h), ref.convert(c, m, T_SC))
