"""CPU tests of the PointCloud2 -> spherical scan conversion (b2_rcc_set_cloud_spherical: pc2_to_scan + fillEmpty + the spherical
unpackMessage): the C restatement of tests/pc2_scan_ref on known answers under both elevation rules, the round trip through a model's own
direction table (and the reference rule's row shift, SURVEY D21), the product's per-point and per-cell functions compiled for the CPU
against the restatement bit for bit, and every refusal of the C entry point (its arguments are checked before the handle)."""
import ctypes as C
import math

import numpy as np
import pytest

import pc2_scan_ref as ref
import rmcl_b200
from rmcl_b200 import synth
from rmcl_b200.api import B2_CLOUD_NO_FIELD, cloud_layout

RULES = [0, ref.ELEV_3D]
F32 = np.float32


def _model(phi=(-0.1, 0.1, 3), theta=(-1.0, 0.25, 8), rng=(0.5, 10.0)):
    return synth.SphericalModel(F32(phi[0]), F32(phi[1]), phi[2], F32(theta[0]), F32(theta[1]), theta[2], F32(rng[0]), F32(rng[1]))


def _planar(angles, ranges):
    a, r = np.asarray(angles, np.float64), np.asarray(ranges, np.float64)
    return np.stack([np.cos(a) * r, np.sin(a) * r, np.zeros_like(a)], 1)


def _cloud(p, **kw):
    p = np.asarray(p, np.float64).reshape(-1, 3)
    return synth.pointcloud2(p, len(p), 1, **kw)


FILL = F32(F32(10.0) + F32(1.0))


@pytest.mark.parametrize("rule", RULES)
def test_last_writer_wins(rule):
    """points 0..4 all fall into column 4 (theta 0) of row 1 (phi 0): the last in-range one wins; a later out-of-range point (r = 50)
    and non-finite points change nothing"""
    m = _model()
    p = np.array([[2, 0, 0], [3, 0, 0], [50, 0, 0], [np.nan, 0, 0], [1, np.inf, 0], [0, 0, -np.inf], [0, 0.25, 0]], np.float64)
    p[6] = _planar([0.5], [7.0])[0]                                         # column 6 (theta 0.5)
    r = ref.convert(_cloud(p), m, flags=rule)
    want = np.full(24, FILL, F32)
    want[8 + 4] = 3.0
    want[8 + 6] = F32(np.sqrt(F32(F32(p[6, 0]) * F32(p[6, 0])) + F32(F32(p[6, 1]) * F32(p[6, 1]))))
    assert np.array_equal(r["ranges"], want)
    assert r["cell"].tolist() == [12, 12, -1, -1, -1, -1, 14]
    assert r["mask"].sum() == 2 and r["mask"][12] == 1 and r["mask"][14] == 1
    # the fill value is fillEmpty's range_max + 1: outside the range, so masked, its point dir * (range_max + 1)
    d = ref.dirs(m)
    assert np.array_equal(r["points"][0], d[0] * FILL + F32(0.0))


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("rmin", [0.0, 0.5])
def test_origin_point(rule, rmin):
    """a finite (0,0,0): range 0, atan2(0, 0) = 0 for both angles -> column 4, row 1; written when range_min <= 0, as in the reference"""
    m = _model(rng=(rmin, 10.0))
    r = ref.convert(_cloud(np.zeros((1, 3))), m, flags=rule)
    assert r["cell"].tolist() == ([12] if rmin <= 0 else [-1])
    assert (r["ranges"][12] == 0.0) == (rmin <= 0) and r["mask"].sum() == int(rmin <= 0)


@pytest.mark.parametrize("rule", RULES)
def test_range_test_is_inclusive(rule):
    lo, hi = F32(0.5), F32(10.0)
    rs = [lo, hi, np.nextafter(lo, F32(0)), np.nextafter(hi, F32(20))]
    for k, rr in enumerate(rs):
        r = ref.convert(_cloud([[float(rr), 0.0, 0.0]]), _model(rng=(lo, hi)), flags=rule)
        assert (r["cell"][0] == 12) == (k < 2), (k, rr)


@pytest.mark.parametrize("rule", RULES)
def test_bin_edges_truncate_toward_zero_and_do_not_wrap(rule):
    """D23 (reproduced): bin coordinate q = (theta - min) / inc; int(q + 0.5) sends (-1.5, -0.5] to column 0, drops q <= -1.5, and drops
    q >= n - 0.5 instead of wrapping it to column 0"""
    m = _model()                                                            # theta from -1.0 in 0.25 steps, 8 columns
    qs = [-1.6, -1.4, -1.0, -0.6, -0.4, 0.0, 3.0, 6.6, 7.4, 7.6, 8.2]
    want = [-1, 0, 0, 0, 0, 0, 3, 7, 7, -1, -1]
    p = _planar([-1.0 + q * 0.25 for q in qs], [5.0] * len(qs))
    r = ref.convert(_cloud(p), m, flags=rule)
    assert [(-1 if c < 0 else c - 8) for c in r["cell"]] == want
    assert np.array_equal(ref.product(_cloud(p), m)["ranges"], ref.convert(_cloud(p), m)["ranges"])


def test_increment_zero_with_one_bin_takes_every_point():
    """D24 (deviation): phi_inc = 0, phi_n = 1 (a 2-D scanner) puts every point into row 0 whatever its elevation; the reference divides
    0 by 0 there.  theta_inc = 0, theta_n = 1 likewise puts every point into column 0."""
    rng = np.random.default_rng(4)
    p = rng.normal(size=(200, 3)) * [5, 5, 2]
    m = _model(phi=(0.0, 0.0, 1), theta=(-math.pi, 2 * math.pi / 16, 16), rng=(0.0, 100.0))
    for rule in RULES:
        r = ref.convert(_cloud(p), m, flags=rule)
        th = np.trunc(((r["theta"] - F32(m.theta_min)) / F32(m.theta_inc)).astype(np.float64) + 0.5).astype(np.int64)
        th[(th < 0) | (th >= 16)] = -1                                      # D23: just below +pi is dropped
        assert np.array_equal(r["cell"], th) and (th >= 0).sum() > 180
    m1 = _model(phi=(-0.5, 0.25, 5), theta=(0.3, 0.0, 1), rng=(0.0, 100.0))
    r = ref.convert(_cloud(p), m1)
    rows = np.trunc(((r["phi"] - F32(m1.phi_min)) / F32(m1.phi_inc)).astype(np.float64) + 0.5)
    inside = (rows >= 0) & (rows < 5) & np.isfinite(p).all(1)
    assert inside.sum() > 50 and np.array_equal(r["cell"][inside], rows[inside].astype(np.int64))
    assert ref.same(ref.product(_cloud(p), m), ref.convert(_cloud(p), m)) and ref.same(ref.product(_cloud(p), m1), ref.convert(_cloud(p), m1))


def test_planar_cloud_both_rules_agree():
    rng = np.random.default_rng(5)
    p = rng.normal(size=(20000, 3)) * 20
    p[:, 2] = 0.0
    m = synth.c2_sensor()
    m.phi_min = -64 * m.phi_inc                                             # a row at phi = 0
    a, b = ref.convert(_cloud(p), m), ref.convert(_cloud(p), m, flags=ref.ELEV_3D)
    assert np.array_equal(a["cell"], b["cell"]) and ref.same(a, b) and (a["cell"] >= 0).sum() > 10000


def _round_trip_cloud(m, seed):
    d = ref.dirs(m).astype(np.float64)
    r = np.random.default_rng(seed).uniform(1.0, 100.0, len(d)).astype(F32)
    return synth.pointcloud2((d.astype(F32) * r[:, None]).astype(F32), m.theta_size, m.phi_size), r


def test_round_trip_returns_every_cell():
    """points dir(cell) * r of a model's own direction table, converted back into that model, fill every cell with their own range (to
    float rounding); with C2 (theta from -pi) column 0 comes back at +pi, half an increment below theta_min + n * inc, and is dropped (D23)"""
    c2 = synth.c2_sensor()
    shifted = synth.SphericalModel(c2.phi_min, c2.phi_inc, c2.phi_size, -math.pi + c2.theta_inc / 2, c2.theta_inc, c2.theta_size, 0.5, 120.0)
    for m, lost in ((shifted, 0), (c2, c2.phi_size)):
        c, r = _round_trip_cloud(m, 1)
        out = ref.convert(c, m)
        n = m.phi_size * m.theta_size
        hit = out["cell"] >= 0
        assert n - hit.sum() == lost
        assert np.array_equal(out["cell"][hit], np.arange(n)[hit])
        if lost:
            grid = hit.reshape(m.phi_size, m.theta_size)
            assert grid[:, 1:].all() and not grid[:, 0].any()
        assert np.allclose(out["ranges"][hit], r[hit], rtol=2e-6, atol=0) and out["mask"].sum() == hit.sum()


def test_round_trip_with_the_reference_rule_shifts_rows():
    """D21: the reference bins elevation atan2(z, |p|) = atan(sin phi); a point of row k lands on row int((atan(sin phi_k) - phi_min) / inc + 0.5).
    For C2 that is 7 rows too high at -25 deg (6.6 rows) and 2 rows at +15 deg (1.6 rows)."""
    m = synth.c2_sensor()
    m.theta_min = -math.pi + m.theta_inc / 2
    c, _ = _round_trip_cloud(m, 2)
    out = ref.convert(c, m, flags=ref.ELEV_3D)
    phi = np.float64(F32(m.phi_min)) + np.arange(m.phi_size) * np.float64(F32(m.phi_inc))
    q = (np.arctan(np.sin(phi)) - np.float64(F32(m.phi_min))) / np.float64(F32(m.phi_inc))
    assert abs((q[0] - 0) - 6.6) < 0.05 and abs((m.phi_size - 1) - q[-1] - 1.6) < 0.05
    row_want = np.floor(q + 0.5).astype(np.int64)
    clear = np.abs(q + 0.5 - np.round(q + 0.5)) > 1e-3                      # rows whose prediction is not on a rounding edge
    got = out["cell"].reshape(m.phi_size, m.theta_size) // m.theta_size
    for k in np.nonzero(clear)[0]:
        assert (got[k] == row_want[k]).all(), k
    assert row_want[0] == 7 and row_want[-1] == m.phi_size - 1 - 2
    moved = row_want != np.arange(m.phi_size)
    assert moved.sum() >= m.phi_size // 2 and (np.abs(phi[moved]) > np.radians(4)).all()
    filled = out["mask"].reshape(m.phi_size, m.theta_size).any(1)          # rows no point lands on stay at the fill value
    assert not filled[:7].any() and not filled[-2:].any() and filled.sum() < m.phi_size


def _special_points(n, rng, scale=40.0):
    p = rng.normal(size=(n, 3)) * [1.0, 1.0, 0.3] * rng.uniform(0.1, scale, (n, 1))
    k = rng.random(n)
    p[k < 0.02, rng.integers(0, 3)] = np.nan
    p[(k >= 0.02) & (k < 0.03), 0] = np.inf
    p[(k >= 0.03) & (k < 0.035)] = 0.0
    p[(k >= 0.035) & (k < 0.04), 1] = 1e39                                 # finite as double, inf as float
    p[(k >= 0.04) & (k < 0.05), 2] = 0.0                                   # exactly planar
    return p


@pytest.mark.parametrize("case", ["c2_f32", "c2_f64_padded_T", "one_cell", "collisions"])
def test_product_functions_match_restatement(case):
    """the product's per-point and per-cell functions (kernels.cuh, compiled for the CPU) equal the restatement bit for bit on > 100 000
    points visited in a shuffled order, including cells many points contend for"""
    rng = np.random.default_rng(len(case))
    m, T, kw, W, H = synth.c2_sensor(), None, {}, 1024, 120
    if case == "c2_f64_padded_T":
        kw = dict(dtype=np.float64, point_step=40, offsets=(3, 13, 27), row_pad=7)
        T = synth.make_transform((0.3, -0.2, 0.15), (0.02, -0.05, 0.7))
    elif case == "one_cell":
        m = synth.SphericalModel(0.0, 0.0, 1, 0.0, 0.0, 1, 0.5, 40.0)
    elif case == "collisions":
        m = synth.SphericalModel(np.radians(-20.0), np.radians(5.0), 9, -math.pi, 2 * math.pi / 24, 24, 0.0, 30.0)
    c = synth.pointcloud2(_special_points(W * H, rng), W, H, seed=2, **kw)
    a = ref.convert(c, m, T)
    b = ref.product(c, m, T, order=rng.permutation(W * H))
    assert ref.same(a, b)
    assert (a["cell"] >= 0).sum() > 1000 and a["mask"].any()
    if case in ("one_cell", "collisions"):
        assert (a["cell"] >= 0).sum() > 20 * m.phi_size * m.theta_size


def test_fp64_angles_against_the_float_atan2f_path():
    """with atan2f (the reference's float path) instead of FP64 atan2 rounded to float, a point changes its cell only where its two float
    angles are at most one ulp apart and a bin boundary lies between them"""
    rng = np.random.default_rng(9)
    m = synth.c2_sensor()
    W, H = 1024, 128
    c = synth.pointcloud2(_special_points(W * H, rng), W, H)
    a, f = ref.convert(c, m), ref.convert(c, m, flags=ref.ATAN2F)
    assert (a["cell"] >= 0).sum() > 50000

    def col(th):
        return np.floor(((th - F32(m.theta_min)) / F32(m.theta_inc)).astype(np.float64) + 0.5)

    def row(ph):
        return np.floor(((ph - F32(m.phi_min)) / F32(m.phi_inc)).astype(np.float64) + 0.5)
    ulp = lambda x, y: np.abs(x.view(np.int32).astype(np.int64) - y.view(np.int32).astype(np.int64))
    for k in np.nonzero(a["cell"] != f["cell"])[0]:
        th_a, th_f, ph_a, ph_f = a["theta"][k:k + 1], f["theta"][k:k + 1], a["phi"][k:k + 1], f["phi"][k:k + 1]
        changed_col, changed_row = col(th_a) != col(th_f), row(ph_a) != row(ph_f)
        assert changed_col or changed_row, k
        assert not changed_col or ulp(th_a, th_f) <= 1, k
        assert not changed_row or ulp(ph_a, ph_f) <= 1, k


def _call(cloud, data=None, nbytes=None, layout=None, T=None):
    """b2_rcc_set_cloud_spherical with no handle: argument refusals name their cause, valid arguments reach the handle check"""
    lib = rmcl_b200.load_library()
    buf = cloud.data if data is None else data
    L = cloud_layout(cloud) if layout is None else layout
    T = synth.make_transform() if T is None else T
    rc = lib.b2_rcc_set_cloud_spherical(None, C.c_void_p(buf.ctypes.data), C.c_uint64(buf.size if nbytes is None else nbytes), C.byref(L),
                                        C.c_void_p(T.ctypes.data), C.c_int(0))
    return rc, lib.b2_last_error().decode()


def test_refusals():
    p = np.ones((4 * 3, 3), np.float32)
    c = synth.pointcloud2(p, 4, 3, point_step=16, row_pad=4)
    rc, msg = _call(c)
    assert rc == -1 and "null argument 'h'" in msg                           # everything else is acceptable
    cases = []
    for name in "xyz":
        L = cloud_layout(c)
        setattr(L, f"offset_{name}", B2_CLOUD_NO_FIELD)
        cases.append((dict(layout=L), "no x, y or z field"))
    bare = synth.pointcloud2(p, 4, 3)
    bare.fields = [f for f in bare.fields if f.name != "z"]
    cases.append((dict(layout=cloud_layout(bare)), "no x, y or z field"))
    for dt in (0, 2, 6, 9):
        L = cloud_layout(c)
        L.datatype = dt
        cases.append((dict(layout=L), "datatype %d" % dt))
    L = cloud_layout(c)
    L.is_bigendian = 1
    cases.append((dict(layout=L), "big-endian"))
    for k, off in enumerate((13, 14, 0xFFFFFFF0)):
        L = cloud_layout(c)
        setattr(L, "offset_" + "xyz"[k], off)
        cases.append((dict(layout=L), "ends beyond point_step"))
    L = cloud_layout(c)
    L.datatype = 8
    L.offset_z = 9
    cases.append((dict(layout=L), "field z at offset 9 ends beyond point_step 16"))
    need = 2 * c.row_step + 3 * 16 + 12
    cases.append((dict(nbytes=need - 1), "the last point read ends at byte %d" % need))
    cases.append((dict(nbytes=0), "bytes given"))
    L = cloud_layout(c)
    L.row_step = 0xFFFFFFFF
    cases.append((dict(layout=L), "bytes given"))
    L = cloud_layout(c)
    L.width, L.height = 0x10000, 0x10000
    cases.append((dict(layout=L), "at most 2^32 - 2"))
    for k, v in ((0, np.nan), (3, np.inf), (4, -np.inf)):
        T = synth.make_transform((0.1, 0.2, 0.3))
        if k < 4:
            T["R"][k] = v
        else:
            T["t"][0] = v
        cases.append((dict(T=T), "T_sensor_cloud is not finite"))
    for kw, want in cases:
        rc, msg = _call(c, **kw)
        assert rc == -1 and want in msg, (kw, want, msg)
    # exactly enough bytes, 2^32 - 2 points (refused only for the bytes), and a cloud of no points (no data needed) pass the argument checks
    assert "null argument 'h'" in _call(c, nbytes=need)[1]
    L = cloud_layout(c)
    L.width, L.height = 0xFFFFFFFE, 1
    assert "bytes given" in _call(c, layout=L)[1]
    lib = rmcl_b200.load_library()
    T = synth.make_transform()
    L = cloud_layout(c)
    L.width = 0
    assert lib.b2_rcc_set_cloud_spherical(None, None, C.c_uint64(0), C.byref(L), C.c_void_p(T.ctypes.data), C.c_int(0)) == -1
    assert "null argument 'h'" in lib.b2_last_error().decode()
    # null pointers
    L = cloud_layout(c)
    assert lib.b2_rcc_set_cloud_spherical(None, None, C.c_uint64(c.data.size), C.byref(L), C.c_void_p(T.ctypes.data), C.c_int(0)) == -1
    assert "null argument 'data'" in lib.b2_last_error().decode()
    assert lib.b2_rcc_set_cloud_spherical(None, C.c_void_p(c.data.ctypes.data), C.c_uint64(c.data.size), None, C.c_void_p(T.ctypes.data), C.c_int(0)) == -1
    assert "null argument 'L'" in lib.b2_last_error().decode()
    assert lib.b2_rcc_set_cloud_spherical(None, C.c_void_p(c.data.ctypes.data), C.c_uint64(c.data.size), C.byref(L), None, C.c_int(0)) == -1
    assert "null argument 'T'" in lib.b2_last_error().decode()
