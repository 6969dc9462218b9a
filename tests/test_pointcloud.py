"""CPU tests of the PointCloud2 -> O1Dn conversion (b2_rcc_set_cloud_o1dn, pc2_to_o1dn + MICPO1DnSensorCUDA::unpackMessage): the numpy
restatement of tests/pc2_ref on known answers, the product's per-ray function compiled for the CPU against it bit for bit, and every
refusal of the C entry point (its arguments are checked before the handle, so no device is needed)."""
import ctypes as C

import numpy as np
import pytest

import pc2_ref as ref
import rmcl_b200
from rmcl_b200 import O1DnCloudFilter, synth
from rmcl_b200.api import cloud_layout


def _flt(hb=0, he=0, hi=1, wb=0, we=0, wi=1, rmin=0.0, rmax=100.0):
    return O1DnCloudFilter(hb, he, hi, wb, we, wi, rmin, rmax)


def _u32(a):
    return np.asarray(a, np.float32).view(np.uint32)


def test_axis_points():
    p = np.array([[2, 0, 0], [0, -3, 0], [0, 0, 0.5], [3, 4, 0]], np.float32)
    r = ref.convert_np(synth.pointcloud2(p, 4, 1), _flt(rmin=1.0, rmax=4.0))
    assert np.array_equal(r["dirs"], np.float32([[1, 0, 0], [0, -1, 0], [0, 0, 1], [0.6, 0.8, 0]]))
    assert np.array_equal(r["ranges"], [2, 3, 0.5, 5])
    assert np.array_equal(r["points"], [[2, 0, 0], [0, -3, 0], [0, 0, 0.5], [3, 4, 0]])
    assert r["mask"].tolist() == [1, 1, 0, 0]


@pytest.mark.parametrize("rmin", [0.0, -1.0, 0.3])
def test_non_finite_points_become_range_zero(rmin):
    """D quirk (reproduced): NaN / +-inf in any coordinate -> dir 0, range 0; that range is valid when range_min <= 0"""
    p = np.array([[np.nan, 1, 1], [1, np.inf, 1], [1, 1, -np.inf], [np.nan] * 3], np.float32)
    r = ref.convert_np(synth.pointcloud2(p, 2, 2), _flt(rmin=rmin))
    assert np.array_equal(_u32(r["dirs"]), np.zeros((4, 3), np.uint32)) and np.array_equal(_u32(r["ranges"]), np.zeros(4, np.uint32))
    assert np.array_equal(_u32(r["points"]), np.zeros((4, 3), np.uint32))
    assert r["mask"].tolist() == [int(rmin <= 0)] * 4


@pytest.mark.parametrize("rmin", [0.0, 0.3])
def test_origin_point_gives_nan_directions(rmin):
    """D quirk (reproduced): a finite (0,0,0) -> range 0, dir 0/0 = NaN, point NaN; the mask tests the range only"""
    r = ref.convert_np(synth.pointcloud2(np.zeros((1, 3), np.float32), 1, 1), _flt(rmin=rmin))
    assert np.all(np.isnan(r["dirs"])) and r["ranges"][0] == 0.0 and np.all(np.isnan(r["points"]))
    assert r["mask"].tolist() == [int(rmin <= 0)]


def test_float64_input_is_rounded_to_float():
    p = np.array([[0.1, 0.2, 0.3], [1e300, 0, 0], [1 + 2.0 ** -40, 0, 0]], np.float64)
    c = synth.pointcloud2(p, 3, 1, dtype=np.float64, point_step=32, offsets=(0, 8, 16))
    r = ref.convert_np(c, _flt())
    with np.errstate(all="ignore"):
        q = p.astype(np.float32)
        n = np.sqrt((q[0, 0] * q[0, 0] + q[0, 1] * q[0, 1]) + q[0, 2] * q[0, 2])
    assert r["ranges"][0] == n and np.array_equal(r["dirs"][0], q[0] / n)
    assert r["ranges"][1] == 0.0 and np.array_equal(r["dirs"][1], [0, 0, 0])         # 1e300 -> inf in float: not finite
    assert r["ranges"][2] == 1.0 and np.array_equal(r["dirs"][2], [1, 0, 0])


def test_row_padding_and_field_layout_change_nothing():
    rng = np.random.default_rng(1)
    p = rng.normal(size=(6 * 5, 3)).astype(np.float32) * 5
    base = ref.convert_np(synth.pointcloud2(p, 6, 5), _flt())
    for kw in (dict(row_pad=3), dict(point_step=48, offsets=(40, 1, 23), row_pad=13), dict(point_step=32, offsets=(8, 4, 0), extra={"intensity": 12})):
        r = ref.convert_np(synth.pointcloud2(p, 6, 5, **kw), _flt())
        assert all(ref.same_bits(base[k], r[k]) for k in ("dirs", "ranges", "points")) and np.array_equal(base["mask"], r["mask"])


@pytest.mark.parametrize("W,H", [(1, 1), (7, 1), (1, 9), (10, 6), (13, 11)])
def test_every_skip_and_increment_edge(W, H):
    """the filter equals slicing the raster [skip_begin : dim - skip_end : increment] and keeping the first (dim - skips) // increment"""
    rng = np.random.default_rng(W * 100 + H)
    p = rng.normal(size=(H, W, 3)).astype(np.float32) * 4
    c = synth.pointcloud2(p.reshape(-1, 3), W, H, row_pad=2)
    full = ref.convert_np(c, _flt())

    def axis_cases(d):
        for b in range(d + 1):
            for e in range(d - b + 1):
                for inc in sorted({1, 2, 3, max(1, d - b - e), d - b - e + 1}):
                    yield b, e, inc
    n = 0
    for hb, he, hi in axis_cases(H):
        for wb, we, wi in list(axis_cases(W))[:: max(1, W // 3)]:
            r = ref.convert_np(c, _flt(hb, he, hi, wb, we, wi))
            h_out, w_out = (H - hb - he) // hi, (W - wb - we) // wi
            assert (r["width"], r["height"]) == (w_out, h_out)
            rows = np.arange(h_out) * hi + hb
            cols = np.arange(w_out) * wi + wb
            sel = (rows[:, None] * W + cols[None, :]).reshape(-1)
            for k in ("dirs", "ranges", "points", "mask"):
                assert np.array_equal(r[k], full[k][sel]), (hb, he, hi, wb, we, wi, k)
            n += 1
    assert n > 0


def test_mask_field_is_ignored_deliberately():
    """D quirk (deviation): the reference stores a field named `mask` as the range (0 or 1); the product ignores the field"""
    rng = np.random.default_rng(2)
    p = rng.normal(size=(40, 3)).astype(np.float32) * 3
    with_mask = synth.pointcloud2(p, 8, 5, point_step=16, extra={"mask": 12})
    plain = synth.pointcloud2(p, 8, 5)
    a, b = ref.convert_np(with_mask, _flt()), ref.convert_np(plain, _flt())
    assert all(ref.same_bits(a[k], b[k]) for k in ("dirs", "ranges", "points")) and np.array_equal(a["mask"], b["mask"])
    lit = ref.convert_np(with_mask, _flt(), reference_mask=True)
    assert set(np.unique(lit["ranges"])) <= {0.0, 1.0} and not np.array_equal(lit["ranges"], a["ranges"])
    e = ref.product_np(with_mask, _flt())
    assert all(ref.same_bits(a[k], e[k]) for k in ("dirs", "ranges", "points"))


def _special_points(n, rng):
    p = (rng.normal(size=(n, 3)) * rng.choice([1e-3, 1.0, 30.0, 1e4], size=(n, 1))).astype(np.float64)
    k = rng.random(n)
    p[k < 0.03, rng.integers(0, 3)] = np.nan
    p[(k >= 0.03) & (k < 0.05), 0] = np.inf
    p[(k >= 0.05) & (k < 0.06), 2] = -np.inf
    p[(k >= 0.06) & (k < 0.07)] = 0.0
    p[(k >= 0.07) & (k < 0.08), 1] = 1e39                                   # finite as double, inf as float
    p[(k >= 0.08) & (k < 0.09)] *= 1e-40                                    # subnormal-range coordinates
    return p


@pytest.mark.parametrize("dtype,point_step,offsets,row_pad,flt", [
    (np.float32, 16, (0, 4, 8), 0, (0, 0, 1, 0, 0, 1, 0.3, 50.0)),
    (np.float32, 48, (5, 18, 31), 9, (3, 2, 2, 7, 1, 3, 0.0, 30.0)),
    (np.float64, 32, (0, 8, 16), 0, (0, 1, 1, 2, 0, 1, -1.0, 80.0)),
    (np.float64, 48, (1, 13, 27), 5, (1, 0, 3, 0, 5, 2, 0.5, 1e4)),
])
def test_product_function_matches_restatement(dtype, point_step, offsets, row_pad, flt):
    """the product's per-ray function (kernels.cuh, compiled for the CPU) equals the restatement bit for bit, NaN-aware, on >= 100 000 points"""
    rng = np.random.default_rng(point_step + row_pad)
    W, H = 1024, 128
    c = synth.pointcloud2(_special_points(W * H, rng), W, H, dtype=dtype, point_step=point_step, offsets=offsets, row_pad=row_pad, seed=3)
    f = O1DnCloudFilter(*flt)
    a, b = ref.convert_np(c, f), ref.product_np(c, f)
    assert a["width"] * a["height"] >= 100_000 // (flt[2] * flt[5]) // 2
    for k in ("dirs", "ranges", "points"):
        assert ref.same_bits(a[k], b[k]), k
    assert np.array_equal(a["mask"], b["mask"])
    assert np.isnan(a["dirs"]).any() and (a["ranges"] == 0).any()


def test_product_function_on_120k_points_unfiltered():
    rng = np.random.default_rng(11)
    c = synth.pointcloud2(_special_points(300 * 400, rng), 400, 300, point_step=16)
    a, b = ref.convert_np(c, _flt(rmin=0.3, rmax=50.0)), ref.product_np(c, _flt(rmin=0.3, rmax=50.0))
    assert len(a["ranges"]) == 120_000
    assert all(ref.same_bits(a[k], b[k]) for k in ("dirs", "ranges", "points")) and np.array_equal(a["mask"], b["mask"])


def _call(cloud, flt, data=None, nbytes=None, layout=None):
    """b2_rcc_set_cloud_o1dn with no handle: argument refusals name their cause, valid arguments reach the handle check"""
    lib = rmcl_b200.load_library()
    buf = cloud.data if data is None else data
    L = cloud_layout(cloud) if layout is None else layout
    rc = lib.b2_rcc_set_cloud_o1dn(None, None if buf is None else C.c_void_p(buf.ctypes.data), C.c_uint64(buf.size if nbytes is None else nbytes),
                                   C.byref(L), C.byref(flt), C.c_int(0))
    return rc, lib.b2_last_error().decode()


def test_refusals():
    p = np.ones((4 * 3, 3), np.float32)
    c = synth.pointcloud2(p, 4, 3, point_step=16, row_pad=4)
    ok = _flt()
    rc, msg = _call(c, ok)
    assert rc == -1 and "null argument 'h'" in msg                           # everything else is acceptable
    cases = []
    for name in "xyz":
        L = cloud_layout(c)
        setattr(L, f"offset_{name}", rmcl_b200.api.B2_CLOUD_NO_FIELD)
        cases.append((dict(layout=L), ok, "no x, y or z field"))
    bare = synth.pointcloud2(p, 4, 3)
    bare.fields = [f for f in bare.fields if f.name != "y"]                # a cloud without a field named y
    cases.append((dict(layout=cloud_layout(bare)), ok, "no x, y or z field"))
    for dt in (0, 2, 6, 9):
        L = cloud_layout(c)
        L.datatype = dt
        cases.append((dict(layout=L), ok, "datatype"))
    L = cloud_layout(c)
    L.is_bigendian = 1
    cases.append((dict(layout=L), ok, "big-endian"))
    cases += [({}, _flt(hi=0), "increment 0"), ({}, _flt(wi=0), "increment 0"),
              ({}, _flt(hb=2, he=2), "skips"), ({}, _flt(wb=5), "skips"), ({}, _flt(we=3, wb=2), "skips"),
              ({}, _flt(hb=0xFFFFFFFF, he=4), "skips")]
    for k, off in enumerate((13, 14, 0xFFFFFFF0)):
        L = cloud_layout(c)
        setattr(L, "offset_" + "xyz"[k], off)
        cases.append((dict(layout=L), ok, "ends beyond point_step"))
    L = cloud_layout(c)
    L.datatype = 8                                                            # z at 8 + 8 bytes = 16: fits; y at 4 + 8 overlaps but fits
    rc, msg = _call(c, ok, layout=L)
    assert "null argument 'h'" in msg
    L.offset_z = 9
    cases.append((dict(layout=L), ok, "ends beyond point_step"))
    need = 2 * c.row_step + 3 * 16 + 12
    cases.append((dict(nbytes=need - 1), ok, "the last point read ends at byte %d" % need))
    cases.append((dict(nbytes=0), ok, "bytes given"))
    L = cloud_layout(c)
    L.row_step = 0xFFFFFFFF
    cases.append((dict(layout=L), ok, "bytes given"))
    L = cloud_layout(c)
    L.width, L.height = 0x10000, 0x10000
    cases.append((dict(layout=L), ok, "model too large"))
    for kw, flt, want in cases:
        rc, msg = _call(c, flt, **kw)
        assert rc == -1 and want in msg, (kw, want, msg)
    # exactly enough bytes is accepted, and so are filters whose output is empty
    assert "null argument 'h'" in _call(c, ok, nbytes=need)[1]
    assert "null argument 'h'" in _call(c, _flt(hb=3))[1] and "null argument 'h'" in _call(c, _flt(wi=5))[1]
    # null pointers
    lib = rmcl_b200.load_library()
    L = cloud_layout(c)
    assert lib.b2_rcc_set_cloud_o1dn(None, None, C.c_uint64(c.data.size), C.byref(L), C.byref(ok), C.c_int(0)) == -1
    assert "data" in lib.b2_last_error().decode()
    assert lib.b2_rcc_set_cloud_o1dn(None, C.c_void_p(c.data.ctypes.data), C.c_uint64(c.data.size), None, C.byref(ok), C.c_int(0)) == -1
    assert lib.b2_rcc_set_cloud_o1dn(None, C.c_void_p(c.data.ctypes.data), C.c_uint64(c.data.size), C.byref(L), None, C.c_int(0)) == -1


def test_layout_record_sizes():
    assert C.sizeof(rmcl_b200.api._CloudLayout) == 32 and C.sizeof(O1DnCloudFilter) == 32
