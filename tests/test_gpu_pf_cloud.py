"""GPU tests of b2_pf_sample_cloud / PCDSensorUpdaterB200.sampleBeams, setInput and update(beams=None): beams drawn from a device, a pinned
and a pageable cloud are byte-identical to each other and to the C restatement of tests/pf_cloud_ref; an update fed from a cloud equals
b2_pf_sensor_update fed the restated beams bit for bit (both correspondence types, mappings 0 and 2, device and host particles) and agrees
with the oracle; sharded halves equal the whole; step advances per update; refusals change nothing and launch nothing; the C++ adapter
matches the Python path."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import native
import pf_cloud_ref as ref
import rmcl_b200
import test_gpu_pf_edges as E
from rmcl_b200 import synth
from rmcl_b200.api import B2_CLOUD_NO_FIELD, cloud_layout

pytestmark = pytest.mark.gpu
SEED = 0x5EED0123456789AB


def _lib():
    return rmcl_b200.load_library()


def _with_source(c, src):
    """the cloud with its bytes in pageable host memory (as is), pinned host memory or device memory"""
    import torch
    if src == "pinned":
        return synth.PointCloud2(c.width, c.height, c.fields, c.is_bigendian, c.point_step, c.row_step, torch.from_numpy(c.data).pin_memory())
    if src == "device":
        return synth.PointCloud2(c.width, c.height, c.fields, c.is_bigendian, c.point_step, c.row_step, torch.from_numpy(c.data).cuda())
    return c


def scan_cloud(seed=3, nan_frac=0.3, dtype=np.float32, **kw):
    """a 32 x 64 cloud of the PF edge scene seen from its scan pose (sensor frame), nan_frac of the points NaN"""
    B = E.beams(32 * 64, seed, penalties=False)
    p = B["dir"].astype(np.float64) * B["range"].astype(np.float64)[:, None]
    rng = np.random.default_rng(seed)
    p[rng.permutation(len(p))[: int(nan_frac * len(p))], rng.integers(0, 3)] = np.nan
    return synth.pointcloud2(p, 64, 32, dtype=dtype, **kw)


def test_sources_match_restatement():
    up = E.updater()
    for name, c in ref.clouds():
        for n in ref.N_SAMPLES:
            for seed, step in ((0, 0), (SEED, 41)):
                want = ref.sample(c, n, seed, step).tobytes()
                for src in ("pageable", "pinned", "device"):
                    got = up.sampleBeams(_with_source(c, src), n, seed, step)
                    assert got.tobytes() == want, (name, n, seed, step, src)
    assert _lib().b2_peek_cuda_error().decode() == ""


@pytest.mark.parametrize("corr", [0, 1])
def test_update_from_cloud_equals_explicit_beams(po, corr):
    prm = E.params(E.PRM, corr, 0)
    c = scan_cloud(4, point_step=32, offsets=(4, 12, 20), row_pad=8)
    step = 9
    B = ref.sample(c, 100, SEED, step)
    assert len(B) == 100
    P = E.admissible(E.scan_particles(3000, 5, 0.4, 0.3), B, 5, 0.4, 0.3, corr)
    A = E.attrs(len(P), n_meas=3, mean=0.7)
    want = E.oracle_pf(po).pf_update(P, A, E.tsb(), B, E.params(E.PRM, corr, 0, po))
    for mapping in (0, 2):
        for src in ("pageable", "device"):
            a, b = E.updater(mapping), E.updater(mapping)
            a.seed, a.step = SEED, step
            a.setInput(_with_source(c, src))
            Pd, Ad = E.to_dev(P, A)
            a.update(Pd, Ad, E.tsb(), params=prm)
            got = E.from_dev(Ad)
            assert a.step == step + 1
            exp = E.update_dev(b, P, A, B, prm)
            assert got.tobytes() == exp.tobytes(), (mapping, src)
            E.assert_oracle(got, want, f"corr {corr} map {mapping} {src}")
        # host particles (b2_pf_sensor_update_host)
        a, b = E.updater(mapping), E.updater(mapping)
        a.seed, a.step = SEED, step
        a.setInput(c)
        got = a.update(P, A, E.tsb(), params=prm)
        assert got.tobytes() == b.update(P, A, E.tsb(), B, prm).tobytes() and a.step == step + 1
        E.assert_oracle(got, want, f"corr {corr} map {mapping} host")


def test_sharded_halves_equal_the_whole():
    """every rank samples the same beams from the same cloud, seed and step: two halves updated on their own equal the whole set"""
    prm = E.params(E.PRM, 0, 0)
    c = scan_cloud(6, dtype=np.float64, point_step=24, offsets=(0, 8, 16))
    P = E.scan_particles(5001, 7, 0.5, 0.3)
    A = E.attrs(len(P), n_meas=1, mean=0.9)
    outs = []
    for part in (slice(None), slice(0, 2500), slice(2500, None)):
        up = E.updater()
        up.seed, up.step = SEED, 123
        up.setInput(_with_source(c, "device"))
        Pd, Ad = E.to_dev(P[part], A[part])
        up.update(Pd, Ad, E.tsb(), params=prm)
        outs.append(E.from_dev(Ad))
    assert outs[0].tobytes() == np.concatenate(outs[1:]).tobytes()


def test_step_advances_per_update():
    prm = E.params(E.PRM, 0, 0)
    c = scan_cloud(8, nan_frac=0.6)
    P, A = E.scan_particles(800, 9, 0.5, 0.3), E.attrs(800)
    a, b = E.updater(0), E.updater(0)
    a.seed, a.step = SEED, 0xFFFFFFFF
    a.setInput(c)
    Pd, Ad = E.to_dev(P, A)
    a.update(Pd, Ad, E.tsb(), params=prm)
    a.update(Pd, Ad, E.tsb(), params=prm)
    Pe, Ae = E.to_dev(P, A)
    for s in (0xFFFFFFFF, 0):                                                  # the step wraps as the uint32 it is
        b.update(Pe, Ae, E.tsb(), ref.sample(c, 100, SEED, s), prm)
    assert E.from_dev(Ad).tobytes() == E.from_dev(Ae).tobytes()
    assert not np.array_equal(ref.sample(c, 100, SEED, 0)["range"], ref.sample(c, 100, SEED, 1)["range"])
    # the beams an update samples are sampleBeams at (seed, step); without an input and without beams update() raises
    assert a.sampleBeams(c, 100, SEED, 7).tobytes() == ref.sample(c, 100, SEED, 7).tobytes()
    with pytest.raises(rmcl_b200.B2Error):
        E.updater().update(Pd, Ad, E.tsb(), params=prm)


def test_refusals_change_nothing():
    import torch
    c = scan_cloud(10)
    dev = _with_source(c, "device")
    up = E.updater()
    P, A = E.scan_particles(500, 11, 0.5, 0.3), E.attrs(500)
    Pd, Ad = E.to_dev(P, A)
    before = Ad.clone()
    n0 = rmcl_b200.kernel_launch_count()
    out = np.zeros(100, synth.RANGE_MEAS_DTYPE)
    nb = C.c_uint32(777)
    layouts = []
    for k in "xyz":
        L = cloud_layout(c)
        setattr(L, "offset_" + k, B2_CLOUD_NO_FIELD)
        layouts.append((L, c.data.size))
    for dt, big in ((2, 0), (9, 0), (7, 1)):
        L = cloud_layout(c)
        L.datatype, L.is_bigendian = dt, big
        layouts.append((L, c.data.size))
    L = cloud_layout(c)
    L.offset_z = 13
    layouts.append((L, c.data.size))
    need = (c.height - 1) * c.row_step + (c.width - 1) * c.point_step + 12                 # z of the last point ends there
    layouts.append((cloud_layout(c), need - 1))
    for L, nbytes in layouts:
        for ptr, d in ((C.c_void_p(dev.data.data_ptr()), 1), (C.c_void_p(c.data.ctypes.data), 0)):
            rc = _lib().b2_pf_sample_cloud(up._h, ptr, C.c_uint64(nbytes), C.byref(L), C.c_int(d), C.c_uint32(100), C.c_uint64(1), C.c_uint32(0),
                                           C.c_void_p(out.ctypes.data), C.byref(nb))
            assert rc == -1 and nb.value == 777 and not out.view(np.uint8).any()
    bad = synth.pointcloud2(np.ones((4, 3)), 4, 1)
    bad.fields = bad.fields[:2]
    up.setInput(bad)
    with pytest.raises(rmcl_b200.B2Error, match="no x, y or z field"):
        up.update(Pd, Ad, E.tsb(), params=E.params(E.PRM, 0, 0))
    assert up.step == 0
    torch.cuda.synchronize()
    assert rmcl_b200.kernel_launch_count() == n0
    assert torch.equal(Ad, before)
    assert _lib().b2_peek_cuda_error().decode() == ""


def test_cpp_adapter_matches_python(tmp_path):
    """tests/pf_cloud_cpp: rmcl::b200::setInput over a PointCloud2-shaped struct, then two device updates and one host update of
    PCDSensorUpdaterB200 -- byte for byte the Python path"""
    exe = native.adapter("pf_cloud_cpp")
    V, F = E.scene_mesh()
    c = scan_cloud(12, dtype=np.float64, point_step=48, offsets=(3, 17, 29), row_pad=6, extra={"intensity": 44})
    P, A = E.scan_particles(700, 13, 0.5, 0.3), E.attrs(700, n_meas=2, mean=0.8)
    prm = E.params(E.PRM, 0, 0)
    step = 77
    with open(tmp_path / "in.bin", "wb") as f:
        np.array([len(V), len(F)], np.uint32).tofile(f)
        V.astype(np.float32).tofile(f)
        F.astype(np.uint32).tofile(f)
        np.array([len(P), step], np.uint32).tofile(f)
        np.array([SEED], np.uint64).tofile(f)
        np.asarray(E.tsb()).tofile(f)
        np.array(E.PRM, np.float32).tofile(f)
        P.tofile(f)
        A.tofile(f)
        np.array([c.width, c.height, c.point_step, c.row_step, 0, len(c.fields)], np.uint32).tofile(f)
        for fl in c.fields:
            f.write(fl.name.encode().ljust(16, b"\0"))
            np.array([fl.offset, fl.datatype], np.uint32).tofile(f)
        c.data.tofile(f)
    out = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "REFUSED update" in out.stdout and "no x, y or z field" in out.stdout
    up = E.updater()
    up.seed, up.step = SEED, step
    up.setInput(c)
    Pd, Ad = E.to_dev(P, A)
    up.update(Pd, Ad, E.tsb(), params=prm)
    a1 = E.from_dev(Ad)
    up.update(Pd, Ad, E.tsb(), params=prm)
    a2 = E.from_dev(Ad)
    a3 = up.update(P, A, E.tsb(), params=prm)
    assert (tmp_path / "out.bin").read_bytes() == a1.tobytes() + a2.tobytes() + a3.tobytes()
    assert up.step == step + 3
