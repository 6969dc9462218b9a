"""GPU tests of b2_rcc_set_cloud_o1dn / RCCB200O1Dn.setPointCloud: the device conversion of an organised PointCloud2 equals the restatement of
tests/pc2_ref bit for bit; corrections after it equal those after set_model_o1dn + set_ranges fed with the restated tables; the find's tile
schedule is kept across clouds of one layout and reset otherwise; refusals change nothing; the C++ adapter matches the Python path."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import native
import pc2_ref as ref
import rmcl_b200
from conftest import gpu_map
from rmcl_b200 import O1DnCloudFilter, synth

pytestmark = pytest.mark.gpu
MAP = "cube29"
TGT = synth.make_transform((0.7, -0.4, 0.3), (0.02, -0.03, 0.4))


def _scan_points(W, H, seed=0):
    """sensor-frame points of a spherical W x H scan of the cube map at TGT (misses beyond 12 m are NaN), with a few (0,0,0) and inf points"""
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / max(H - 1, 1), H, -np.pi, 2 * np.pi / W, W, 0.5, 12.0)
    h = rmcl_b200.RCCB200Spherical(gpu_map(MAP))
    h.setModel(m)
    h.find(TGT)
    p = h.modelView()["points"].astype(np.float64)
    rng = np.random.default_rng(seed)
    k = rng.permutation(len(p))
    p[k[: max(1, len(p) // 500)]] = 0.0
    p[k[len(p) // 500: len(p) // 250], 1] = np.inf
    return p


def _lib():
    return rmcl_b200.load_library()


def _tables(h):
    n = C.c_uint32()
    assert _lib().b2_rcc_debug_model_tables(h._h, None, None, C.byref(n)) == 0
    d, r = np.zeros((n.value, 3), np.float32), np.zeros(n.value, np.float32)
    assert _lib().b2_rcc_debug_model_tables(h._h, C.c_void_p(d.ctypes.data), C.c_void_p(r.ctypes.data), C.byref(n)) == 0
    return d, r


def _perm(h):
    n = C.c_uint32()
    assert _lib().b2_rcc_debug_tile_perm(h._h, None, 0, C.byref(n)) == 0
    out = np.zeros(max(n.value, 1), np.uint16)
    assert _lib().b2_rcc_debug_tile_perm(h._h, C.c_void_p(out.ctypes.data), C.c_uint32(len(out)), C.byref(n)) == 0
    return out[: n.value]


def _assert_same(h, want):
    d, r = _tables(h)
    ds = h.datasetView()
    assert ref.same_bits(d, want["dirs"]) and ref.same_bits(r, want["ranges"])
    assert ref.same_bits(ds["points"], want["points"]) and np.array_equal(ds["mask"], want["mask"])


FORMATS = [dict(dtype=np.float32, point_step=16, offsets=(0, 4, 8)),
           dict(dtype=np.float64, point_step=48, offsets=(1, 13, 27), row_pad=5, extra={"mask": 40, "intensity": 41}),
           dict(dtype=np.float32, point_step=32, offsets=(20, 9, 2), row_pad=3, extra={"mask": 0})]


@pytest.mark.parametrize("W,H", [(1, 1), (255, 1), (256, 1), (257, 1), (1024, 128), (2048, 65)])
def test_cloud_matches_restatement(W, H):
    import torch
    p = _scan_points(W, H, seed=W + H)
    h = rmcl_b200.RCCB200O1Dn(gpu_map(MAP))
    for fi, fmt in enumerate(FORMATS):
        c = synth.pointcloud2(p, W, H, seed=fi, **fmt)
        for flt in (O1DnCloudFilter.defaults(0.3, 12.0), O1DnCloudFilter(H // 3, H // 4, 2 if H > 2 else 1, 1 if W > 2 else 0, W // 5, 3 if W > 3 else 1, 0.0, 10.0)):
            want = ref.convert_np(c, flt)
            host = c.data
            for src in ("pageable", "pinned", "device"):
                if src == "pinned":
                    c.data = torch.from_numpy(host).pin_memory()
                elif src == "device":
                    c.data = torch.from_numpy(host).cuda()
                h.setPointCloud(c, flt)
                c.data = host
                if want["width"] * want["height"] == 0:
                    assert h.datasetView()["points"].shape == (0, 3)
                    continue
                _assert_same(h, want)


def _cloud_case(W=256, H=32, seed=1):
    c = synth.pointcloud2(_scan_points(W, H, seed), W, H, dtype=np.float64, point_step=48, offsets=(0, 8, 16), row_pad=8)
    flt = O1DnCloudFilter(0, 0, 1, 0, 0, 1, 0.3, 12.0)
    return c, flt, ref.convert_np(c, flt)


def _pair(c, flt, want):
    a = rmcl_b200.RCCB200O1Dn(gpu_map(MAP))
    a.setPointCloud(c, flt)
    b = rmcl_b200.RCCB200O1Dn(gpu_map(MAP))
    b.setModel(synth.O1DnModel(want["width"], want["height"], np.zeros(3, np.float32), want["dirs"], flt.range_min, flt.range_max))
    b.setRanges(want["ranges"])
    return a, b


def _bits(*xs):
    return b"".join(np.asarray(x).tobytes() for x in xs)


def test_corrections_equal_the_table_path():
    c, flt, want = _cloud_case()
    assert np.isnan(want["dirs"]).any()                                     # (0,0,0) points: NaN rays are traced like the table path's
    a, b = _pair(c, flt, want)
    Tguess = synth.compose(TGT, synth.make_transform((0.1, -0.05, 0.02), (0.0, 0.01, -0.03)))
    I = synth.make_transform()
    for cp in (0.0, 0.4):
        ra, rb = a.correctOnce(Tguess, I, 5, cp), b.correctOnce(Tguess, I, 5, cp)
        assert _bits(*ra) == _bits(*rb) and ra[2]["n_meas"] > 1000
    # two sensors: the cloud-fed O1Dn sensor with a spherical one
    m = synth.c1_sensor()
    s = rmcl_b200.RCCB200Spherical(gpu_map(MAP))
    s.setModel(m)
    s.find(TGT)
    s.setRanges(synth.noisy_ranges(s.modelView()["ranges"], m.range_max, seed=4))
    Tbo = np.stack([synth.make_transform(), synth.make_transform()])
    for w in (None, [1.0, 0.5]):
        ra = rmcl_b200.micp_correct_once([a, s], Tbo, Tguess, 5, 0.0, merge_weights=w)
        rb = rmcl_b200.micp_correct_once([b, s], Tbo, Tguess, 5, 0.0, merge_weights=w)
        assert _bits(*ra) == _bits(*rb)
    for sensors in (([a], [b]), ([a, s], [b, s])):
        Tb = Tbo[: len(sensors[0])]
        ta, cpa, sa = rmcl_b200.micp_correct(sensors[0], Tb, Tguess, n_corrections=3)
        tb, cpb, sb = rmcl_b200.micp_correct(sensors[1], Tb, Tguess, n_corrections=3)
        assert _bits(ta, sa) == _bits(tb, sb) and cpa == cpb
    assert sa["valid_measurements"][0] == int(want["mask"].sum()) + int((s.datasetView()["mask"] > 0).sum())


def test_tile_schedule_kept_across_clouds_of_one_layout():
    W, H = 1024, 128
    flt = O1DnCloudFilter.defaults(0.3, 12.0)
    p1, p2 = _scan_points(W, H, 5), _scan_points(W, H, 6)
    c1, c2 = synth.pointcloud2(p1, W, H), synth.pointcloud2(p2, W, H, point_step=48, offsets=(8, 16, 24))
    I = synth.make_transform()
    Tguess = synth.compose(TGT, synth.make_transform((0.05, 0.05, 0.0), (0.0, 0.0, 0.02)))
    h = rmcl_b200.RCCB200O1Dn(gpu_map(MAP))
    h.setPointCloud(c1, flt)
    h.correctOnce(Tguess, I, 5, 0.0)
    P1 = _perm(h)
    assert len(P1) == W * H // 32 and np.array_equal(np.sort(P1), np.arange(len(P1))) and not np.array_equal(P1, np.arange(len(P1)))
    h.setPointCloud(c2, flt)
    assert np.array_equal(_perm(h), P1)                                     # the previous loop's schedule carries over
    fresh = rmcl_b200.RCCB200O1Dn(gpu_map(MAP))
    fresh.setPointCloud(c2, flt)
    assert _bits(*h.correctOnce(Tguess, I, 5, 0.0)) == _bits(*fresh.correctOnce(Tguess, I, 5, 0.0))
    # a layout change resets it: another filter, the same ray count in another raster, or a model from set_model_o1dn
    for other in (synth.pointcloud2(p2.reshape(H, W, 3)[:, ::2].reshape(-1, 3), W // 2, H), synth.pointcloud2(p2, 2 * W, H // 2)):
        h.setPointCloud(c1, flt)
        h.correctOnce(Tguess, I, 5, 0.0)
        assert len(_perm(h)) > 0
        h.setPointCloud(other, flt)
        assert len(_perm(h)) == 0
    h.setPointCloud(c1, flt)
    h.correctOnce(Tguess, I, 5, 0.0)
    want = ref.convert_np(c1, flt)
    h.setModel(synth.O1DnModel(W, H, np.zeros(3, np.float32), want["dirs"], 0.3, 12.0))
    assert len(_perm(h)) == 0
    # and a cloud after set_model_o1dn starts from the identity schedule, like a fresh handle
    h.setPointCloud(c1, flt)
    assert len(_perm(h)) == 0


def test_refusals_change_nothing():
    from rmcl_b200.api import B2_CLOUD_NO_FIELD, cloud_layout
    c, flt, want = _cloud_case(256, 16, seed=9)
    h = rmcl_b200.RCCB200O1Dn(gpu_map(MAP))
    h.setPointCloud(c, flt)
    h.correctOnce(TGT, synth.make_transform(), 5, 0.0)
    d0, r0 = _tables(h)
    ds0, perm0 = h.datasetView(), _perm(h)
    assert len(perm0) == 256 * 16 // 32
    n0 = rmcl_b200.kernel_launch_count()
    cases = []
    for k in "xyz":
        L = cloud_layout(c)
        setattr(L, "offset_" + k, B2_CLOUD_NO_FIELD)
        cases.append((L, flt, c.data.size))
    for dt, big in ((2, 0), (9, 0), (7, 1)):
        L = cloud_layout(c)
        L.datatype, L.is_bigendian = dt, big
        cases.append((L, flt, c.data.size))
    L = cloud_layout(c)
    L.offset_z = 41
    cases.append((L, flt, c.data.size))
    cases += [(cloud_layout(c), O1DnCloudFilter(0, 0, 0, 0, 0, 1, 0.3, 12.0), c.data.size),
              (cloud_layout(c), O1DnCloudFilter(10, 7, 1, 0, 0, 1, 0.3, 12.0), c.data.size),
              (cloud_layout(c), O1DnCloudFilter(0, 0, 1, 200, 57, 1, 0.3, 12.0), c.data.size),
              (cloud_layout(c), flt, (c.height - 1) * c.row_step + (c.width - 1) * c.point_step + 24 - 1)]
    L = cloud_layout(c)
    L.width, L.height = 0x10000, 0x10000
    cases.append((L, flt, c.data.size))
    for L, f, nbytes in cases:
        rc = _lib().b2_rcc_set_cloud_o1dn(h._h, C.c_void_p(c.data.ctypes.data), C.c_uint64(nbytes), C.byref(L), C.byref(f), C.c_int(0))
        assert rc == -1, _lib().b2_last_error().decode()
    assert _lib().b2_rcc_set_cloud_o1dn(h._h, None, C.c_uint64(c.data.size), C.byref(cloud_layout(c)), C.byref(flt), C.c_int(0)) == -1
    assert rmcl_b200.kernel_launch_count() == n0
    d1, r1 = _tables(h)
    ds1 = h.datasetView()
    assert ref.same_bits(d0, d1) and ref.same_bits(r0, r1) and ref.same_bits(ds0["points"], ds1["points"]) and np.array_equal(ds0["mask"], ds1["mask"])
    assert np.array_equal(_perm(h), perm0)
    assert _lib().b2_peek_cuda_error().decode() == ""


def test_cpp_adapter_matches_python(tmp_path):
    """tests/pointcloud_cpp: unpackPointCloud over PointCloud2-shaped structs, then correctOnce -- byte for byte the Python path"""
    exe = native.adapter("pointcloud_cpp")
    from conftest import mesh
    V, F = mesh(MAP)
    with open(tmp_path / "map.bin", "wb") as f:
        np.array([len(V), len(F)], np.uint32).tofile(f)
        V.astype(np.float32).tofile(f)
        F.astype(np.uint32).tofile(f)
    c = synth.pointcloud2(_scan_points(512, 24, 3), 512, 24, dtype=np.float64, point_step=48, offsets=(3, 17, 29), row_pad=6, extra={"mask": 47})
    flt = O1DnCloudFilter(1, 2, 1, 3, 1, 2, 0.3, 12.0)
    with open(tmp_path / "cloud.bin", "wb") as f:
        np.array([c.width, c.height, c.point_step, c.row_step, 0, len(c.fields)], np.uint32).tofile(f)
        for fl in c.fields:
            f.write(fl.name.encode().ljust(16, b"\0"))
            np.array([fl.offset, fl.datatype], np.uint32).tofile(f)
        np.array([flt.height_skip_begin, flt.height_skip_end, flt.height_increment, flt.width_skip_begin, flt.width_skip_end, flt.width_increment],
                 np.uint32).tofile(f)
        np.array([flt.range_min, flt.range_max], np.float32).tofile(f)
        c.data.tofile(f)
    out = subprocess.run([exe, str(tmp_path / "map.bin"), str(tmp_path / "cloud.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "REFUSED setPointCloud" in out.stdout and "no x, y or z field" in out.stdout
    h = rmcl_b200.RCCB200O1Dn(gpu_map(MAP))
    h.setPointCloud(c, flt)
    ds = h.datasetView()
    I = synth.make_transform()
    Tn, _, _ = h.correctOnce(I, I, 5, 0.0)
    got = (tmp_path / "out.bin").read_bytes()
    assert got == _bits(ds["points"], ds["mask"], Tn)
    want = ref.convert_np(c, flt)
    assert ref.same_bits(ds["points"], want["points"])
