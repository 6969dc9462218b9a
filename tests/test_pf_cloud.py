"""CPU tests of the particle filter's beam sampling from a PointCloud2 (b2_pf_sample_cloud): the C restatement of tests/pf_cloud_ref on
known answers, the product's per-sample function compiled for the CPU against the restatement bit for bit on every cloud layout and sample
count, the uniformity of the keyed draws, and every refusal of the C entry point (its arguments are checked before the handle)."""
import ctypes as C

import numpy as np
import pytest

import pf_cloud_ref as ref
import rmcl_b200
from rmcl_b200 import synth
from rmcl_b200.api import B2_CLOUD_NO_FIELD, cloud_layout

F32 = np.float32
CLOUDS = dict(ref.clouds())


def test_known_answers():
    """one point: every sample is that point; the draw of sample k, try 0 is point philox(k, 3, step, 0)[0] % n"""
    from oracle import pyoracle as po
    po.build()
    b = ref.sample(CLOUDS["1x1"], 5, 7, 3)
    assert len(b) == 5
    assert np.array_equal(b["range"], np.full(5, F32(13.0))) and np.array_equal(b["dir"], np.tile(np.array([3, -4, 12], F32) / F32(13), (5, 1)))
    assert not b["orig"].any() and np.array_equal(b["cov"][:, [0, 4, 8]], np.full((5, 3), F32(0.1))) and not b["cov"][:, [1, 2, 3, 5, 6, 7]].any()
    x = np.arange(1, 1001, dtype=np.float64)
    c = synth.pointcloud2(np.stack([x, np.zeros_like(x), np.zeros_like(x)], 1), 1000, 1)
    seed = 0x123456789ABCDEF
    for step in (0, 5, 0xFFFFFFFF):
        b = ref.sample(c, 40, seed, step)
        want = [po.philox4x32_10([k, 3, step, 0], [seed & 0xFFFFFFFF, seed >> 32])[0] % 1000 + 1 for k in range(40)]
        assert np.array_equal(b["range"], np.array(want, F32)), step


def test_give_up_rule_and_special_points():
    """all NaN: ten samples fail and nothing comes back; 99.9 % NaN: the 10th failed sample ends the update; (0,0,0) gives range 0 and
    0x7fffffff directions; an infinite coordinate passes with range inf"""
    assert len(ref.sample(CLOUDS["all_nan"], 4096, 1, 0)) == 0
    v, _ = ref.product_samples(CLOUDS["all_nan"], 20, 1, 0)
    assert not v.any()
    c = CLOUDS["128x1024_nan0.999"]                                        # a sample finds a point with probability 1 - 0.999^100 = 9.5 %
    lens = []
    for seed in range(20):
        v, beams = ref.product_samples(c, 4096, seed, 0)
        bad = np.flatnonzero(v == 0)
        got = ref.sample(c, 4096, seed, 0)
        assert len(bad) >= 10 and len(got) == bad[9] - 9 and got.tobytes() == beams[: bad[9]][v[: bad[9]] != 0].tobytes()
        lens.append(len(got))
    assert max(lens) > 0
    z = ref.sample(CLOUDS["zero"], 4096, 3, 1)
    zero = z["range"] == 0
    assert zero.sum() > 500 and (z["dir"][zero].view(np.uint32) == 0x7FFFFFFF).all()
    assert not np.isnan(z["dir"][~zero]).any()
    i = ref.sample(CLOUDS["inf"], 4096, 4, 1)
    inf = np.isinf(i["range"])
    assert inf.sum() > 500 and (i["range"][inf] > 0).all() and np.isfinite(i["range"][~inf]).all()
    d = i["dir"][inf]
    assert (np.isnan(d) == (d.view(np.uint32) == 0x7FFFFFFF)).all() and np.isnan(d).any()


@pytest.mark.parametrize("name", list(CLOUDS))
def test_product_function_matches_restatement(name):
    """the product's pf_sample_beam (kernels.cuh, compiled for the CPU) under the give-up rule equals the restatement byte for byte"""
    c = CLOUDS[name]
    for n in ref.N_SAMPLES:
        for seed, step in ((0, 0), (0xDEADBEEF12345678, 17)):
            a, b = ref.sample(c, n, seed, step), ref.product(c, n, seed, step)
            assert a.tobytes() == b.tobytes(), (name, n, seed, step)
            if n and name not in ("all_nan", "128x1024_nan0.999"):
                assert len(a) == n, (name, n)


def test_layouts_read_the_same_points():
    """the same points as FLOAT64 at unaligned offsets with padded rows and as FLOAT32 in 48-byte points with extra fields: identical beams
    (the FLOAT64 values are floats widened, so narrowing is exact)"""
    a = ref.sample(CLOUDS["f64_unaligned_padded"], 4096, 9, 2)
    b = ref.sample(CLOUDS["f32_ps48_extra_padded"], 4096, 9, 2)
    assert len(a) == 4096 and a.tobytes() == b.tobytes()


def test_draws_are_uniform():
    """drawn indices pass a chi-square test: on a 64-point cloud (first tries) and on the 64 finite points of a 128-point cloud whose even
    points are NaN (later tries and words)"""
    from scipy.stats import chisquare
    x = np.arange(1, 129, dtype=np.float64)
    p = np.stack([x, np.zeros_like(x), np.zeros_like(x)], 1)
    c64 = synth.pointcloud2(p[:64], 8, 8)
    p[::2, 2] = np.nan
    c128 = synth.pointcloud2(p, 128, 1, point_step=12)
    for c, want_bins in ((c64, np.arange(1, 65)), (c128, np.arange(2, 129, 2))):
        counts = np.zeros(129, np.int64)
        for step in range(40):
            v, b = ref.product_samples(c, 512, 2024, step)
            assert v.all()
            np.add.at(counts, b["range"].astype(np.int64), 1)
        assert counts.sum() == counts[want_bins].sum() == 40 * 512
        assert chisquare(counts[want_bins]).pvalue > 1e-3


def _call(cloud=None, data=None, nbytes=None, layout=None, n_samples=4, beams=True, n_beams=True):
    """b2_pf_sample_cloud with no handle -> (rc, message, *n_beams); argument refusals name their cause, valid arguments reach the handle check"""
    lib = rmcl_b200.load_library()
    buf = cloud.data if data is None else data
    L = cloud_layout(cloud) if layout is None else layout
    out = np.zeros(max(n_samples, 1), synth.RANGE_MEAS_DTYPE)
    nb = C.c_uint32(777)
    ptr = None if buf is False else C.c_void_p(buf.ctypes.data)
    nbytes = cloud.data.size if nbytes is None else nbytes
    rc = lib.b2_pf_sample_cloud(None, ptr, C.c_uint64(nbytes), None if L is False else C.byref(L),
                                C.c_int(0), C.c_uint32(n_samples), C.c_uint64(1), C.c_uint32(0), C.c_void_p(out.ctypes.data) if beams else None,
                                C.byref(nb) if n_beams else None)
    assert not out.view(np.uint8).any()
    return rc, lib.b2_last_error().decode(), nb.value


def test_refusals():
    p = np.ones((4 * 3, 3), np.float32)
    c = synth.pointcloud2(p, 4, 3, point_step=16, row_pad=4)
    rc, msg, nb = _call(c)
    assert rc == -1 and "null argument 'h'" in msg and nb == 777
    cases = []
    for name in "xyz":
        L = cloud_layout(c)
        setattr(L, f"offset_{name}", B2_CLOUD_NO_FIELD)
        cases.append((dict(layout=L), "pf_sample_cloud: the cloud has no x, y or z field"))
    bare = synth.pointcloud2(p, 4, 3)
    bare.fields = [f for f in bare.fields if f.name != "x"]
    cases.append((dict(layout=cloud_layout(bare)), "no x, y or z field"))
    for dt in (0, 2, 6, 9):
        L = cloud_layout(c)
        L.datatype = dt
        cases.append((dict(layout=L), "pf_sample_cloud: field x has datatype %d; FLOAT32 (7) and FLOAT64 (8) are read" % dt))
    L = cloud_layout(c)
    L.is_bigendian = 1
    cases.append((dict(layout=L), "pf_sample_cloud: big-endian clouds are not read"))
    for k, off in enumerate((13, 14, 0xFFFFFFF0)):
        L = cloud_layout(c)
        setattr(L, "offset_" + "xyz"[k], off)
        cases.append((dict(layout=L), "field %s at offset %d ends beyond point_step 16" % ("xyz"[k], off)))
    L = cloud_layout(c)
    L.datatype = 8
    L.offset_z = 9
    cases.append((dict(layout=L), "field z at offset 9 ends beyond point_step 16"))
    need = 2 * c.row_step + 3 * 16 + 12
    cases.append((dict(nbytes=need - 1), "pf_sample_cloud: %d bytes given, the last point read ends at byte %d" % (need - 1, need)))
    cases.append((dict(nbytes=0), "bytes given"))
    cases.append((dict(nbytes=0, n_samples=0), "bytes given"))                 # the layout is checked whatever the sample count
    L = cloud_layout(c)
    L.row_step = 0xFFFFFFFF
    cases.append((dict(layout=L), "bytes given"))
    L = cloud_layout(c)
    L.width, L.height = 0x10000, 0x10000
    cases.append((dict(layout=L), "pf_sample_cloud: 4294967296 points, at most 2^32 - 1 are read"))
    cases += [(dict(data=False), "null argument 'data'"), (dict(layout=False), "null argument 'L'"), (dict(beams=False), "null argument 'beams'"),
              (dict(n_beams=False), "null argument 'n_beams'")]
    for kw, want in cases:
        rc, msg, nb = _call(c, **kw)
        assert rc == -1 and want in msg and nb == 777, (kw, want, msg)
    # exactly enough bytes, 2^32 - 1 points (refused only for the bytes), no samples without a beams array, and a cloud of no points
    # without data pass the argument checks
    assert "null argument 'h'" in _call(c, nbytes=need)[1]
    L = cloud_layout(c)
    L.width, L.height = 0xFFFFFFFF, 1
    assert "bytes given" in _call(c, layout=L)[1]
    assert "null argument 'h'" in _call(c, n_samples=0, beams=False)[1]
    L = cloud_layout(c)
    L.height = 0
    assert "null argument 'h'" in _call(c, data=False, nbytes=0, layout=L)[1]
