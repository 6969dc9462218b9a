"""GPU tests of the filter's pose hypotheses (b2_pf_cluster_stats: k_pf_residual_stats, k_pf_cluster_insert, k_pf_cluster_hook,
k_pf_cluster_flatten, the cluster sorts, k_pf_cluster_rank, k_pf_cluster_labels, the member sort, k_pf_cluster_gather and the two estimate
kernels per recorded cluster) against the C restatement of tests/pf_cluster_ref, fed the device's weight_max.

Counts, weights, keys and every label are exact; each record's stats equals, byte for byte, estimateStats of that cluster's members alone."""
import math
import os
import subprocess

import numpy as np
import pytest

import pf_cluster_ref as ref
from conftest import gpu_map
from test_gpu_pf_residual import _dev, _np, _out
from test_pf_cluster import RES_Z, attrs_of, blob, cfg, poses_in_bins, snake
from test_pf_residual import CFG, particles

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NONE = 0xFFFFFFFF
_up = None


def _updater():
    global _up
    if _up is None:
        import rmcl_b200
        _up = rmcl_b200.PCDSensorUpdaterB200(gpu_map("cube29"))
    return _up


def _case(n, seed, kind):
    """uniform: |x|, |y| <= 20 m, all headings; bimodal: two Gaussians 12 m apart holding 60 % / 40 % of the particles; converged: sigma 0.3 m, 5 deg"""
    P, A = particles(n, "lognormal", seed=seed)
    rng = np.random.default_rng(seed + 1)
    P["t"][:, 2] *= np.float32(1.0 / 20.0)
    if kind != "uniform":
        mode = (rng.uniform(size=n) < 0.4) if kind == "bimodal" else np.zeros(n, bool)
        yaw = rng.normal(0.0, math.radians(5.0), n) + np.where(mode, 2.0, -1.0)
        P["t"][:, 0] = rng.normal(0.0, 0.3, n) + np.where(mode, 12.0, 0.0)
        P["t"][:, 1] = rng.normal(0.0, 0.3, n)
        P["R"] = np.stack([np.zeros(n), np.zeros(n), np.sin(yaw / 2), np.cos(yaw / 2)], axis=1).astype(np.float32)
        A["likelihood"]["mean"] = rng.uniform(0.5, 1.0, n).astype(np.float32)
    return P, A


def _run(up, P, A, c, dev=None, labels=True):
    import torch
    Pd, Ad = dev if dev is not None else _dev(P, A)
    lab = torch.full((len(P),), 7, dtype=torch.int32, device="cuda") if labels else None
    r, recs = up.estimateClusters(Pd, Ad, c, lab)
    return r, recs, (lab.cpu().numpy().view(np.uint32) if labels else None)


def _compare(P, A, c, up=None, stats=True):
    up = up or _updater()
    Pd, Ad = _dev(P, A)
    r, recs, lab = _run(up, P, A, c, dev=(Pd, Ad))
    want = ref.clusters(P, A, c, S=float(r["weight_sum"]), L_max=float(r["weight_max"]))
    assert want is not None
    assert (int(r["n_clusters"]), int(r["bins"]), int(r["n_clustered"]), int(r["weight_total"])) == \
           (want["n_clusters"], want["bins"], want["n_clustered"], want["weight_total"])
    assert np.array_equal(lab, want["labels"])
    k = min(want["n_clusters"], c.max_records)
    assert int(r["n_records"]) == k == len(recs) and 1 <= int(r["rounds"]) <= 64
    assert np.array_equal(recs["weight_int"], want["weight_int"][:k]) and np.array_equal(recs["key"], want["key"][:k])
    assert np.array_equal(recs["bins"], want["cbins"][:k])
    assert np.array_equal(recs["weight"], want["weight_int"][:k].astype(np.float64) / np.float64(want["weight_total"]))
    assert np.array_equal(recs["stats"]["nparticles"], want["members"][:k])
    if stats:                                                       # each record is estimateStats of the cluster's members in index order
        import torch
        for j in range(k):
            idx = torch.from_numpy(np.flatnonzero(lab == j)).cuda()
            alone = up.estimateStats(Pd[idx].contiguous(), Ad[idx].contiguous(), max_induction_particles=len(idx))
            assert recs["stats"][j].tobytes() == alone.tobytes(), j
    return r, recs, lab


@pytest.mark.parametrize("kind", ["uniform", "bimodal", "converged"])
@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 1000, 65537, 1_000_000])
def test_device_matches_restatement(n, kind):
    P, A = _case(n, n, kind)
    r, recs, _ = _compare(P, A, cfg())
    if n >= 65537 and kind == "bimodal":                            # a stray particle of a tail may be a cluster of its own
        assert abs(float(recs["weight"][0]) - 0.6) < 0.01 and abs(float(recs["weight"][1]) - 0.4) < 0.01
    if n >= 65537 and kind == "converged":
        assert float(recs["weight"][0]) > 0.99


def test_settings_and_families():
    P, A = _case(200_000, 8, "uniform")
    for kw in ({"res_z": 0.1}, {"res_yaw": math.radians(1.0)}, {"res_yaw": 7.0}, {"res_yaw": math.pi}, {"res_xy": 0.05, "max_records": 16},
               {"res_xy": 4.0, "max_records": 1}):
        _compare(P, A, cfg(**kw))
    for family in ("uniform", "dominant", "half_zero"):
        P, A = particles(100_000, family, seed=3)
        P["t"][::1001, 1] = np.nan
        _compare(P, A, cfg(res_xy=0.25))


def test_crafted_topologies():
    K, c = 36, cfg(res_z=RES_Z)

    def run(cells, L=None, **kw):
        P = poses_in_bins(cells, K)
        return _compare(P, attrs_of(np.ones(len(cells)) if L is None else L), cfg(res_z=RES_Z, **kw))

    assert int(run(blob(0, 0) + blob(4, 0))[0]["n_clusters"]) == 2                 # one empty column between them
    assert int(run([(0, 0, 0, 5), (1, 1, 1, 6)])[0]["n_clusters"]) == 1            # touching diagonally in all four dimensions
    assert int(run([(0, 0, 0, 5), (1, 1, 1, 7)])[0]["n_clusters"]) == 2
    ring = [(0, 0, 0, s) for s in range(K) if s not in (10, 20)]                   # a ring in yaw through the wrap, cut twice
    r, recs, _ = run(ring)
    assert int(r["n_clusters"]) == 2 and list(recs["bins"]) == [25, 9]
    cells = blob(0, 0) + blob(4, 0) + [(3, 1, 0, 5)]                               # a zero-likelihood particle in the gap
    L = np.ones(len(cells)); L[-1] = 0.0
    r, _, lab = run(cells, L)
    assert int(r["n_clusters"]) == 2 and lab[-1] == NONE and int(r["n_clustered"]) == 18
    L[-1] = 1.0
    assert int(run(cells, L)[0]["n_clusters"]) == 1
    P = poses_in_bins(cells, K)
    P["t"][-1, 2] = np.inf
    r, _, lab = _compare(P, attrs_of(L), c)
    assert int(r["n_clusters"]) == 2 and lab[-1] == NONE
    cells = blob(10, 0, side=1) + blob(0, 0, side=1) + blob(5, 0, side=1) + blob(5, 5, side=1) * 2     # equal weights: the smaller key first
    r, recs, lab = run(cells)
    assert list(recs["weight_int"]) == [2 ** 33, 2 ** 32, 2 ** 32, 2 ** 32] and list(lab) == [3, 1, 2, 0, 0]
    for sectors in (1, 2):                                                         # K = 1, 2: offsets that coincide change nothing
        Pk = poses_in_bins([(0, 0, 0, s) for s in range(sectors)] + [(2, 0, 0, 0)], sectors)
        assert int(_compare(Pk, attrs_of(np.ones(len(Pk))), cfg(res_yaw=2 * math.pi / sectors))[0]["n_clusters"]) == 2


def test_snake_of_100000_bins():
    """a one-bin-wide path of 100 199 bins is one cluster, within the cap on rounds"""
    cells = snake()
    r, recs, _ = _compare(poses_in_bins(cells, 36), attrs_of(np.ones(len(cells))), cfg(), stats=False)
    assert int(r["n_clusters"]) == 1 and int(recs["bins"][0]) == len(cells) == 100_199 and int(r["rounds"]) <= 64


def test_all_poses_non_finite_and_refused_sets():
    P, A = _case(1000, 2, "uniform")
    P["t"][:, 0] = np.nan
    r, recs, lab = _run(_updater(), P, A, cfg())
    assert int(r["n_clusters"]) == 0 and len(recs) == 0 and np.all(lab == NONE) and float(r["weight_sum"]) > 0
    for bad in (0.0, -1e-3, float("nan"), float("inf")):
        P, A = _case(1000, 2, "uniform")
        if bad == 0.0:
            A["likelihood"]["mean"] = 0.0
        else:
            A["likelihood"]["mean"][500] = bad
        r, recs, lab = _run(_updater(), P, A, cfg())
        assert int(r["n_clusters"]) == 0 and int(r["bins"]) == 0 and len(recs) == 0 and np.all(lab == 7)      # nothing written but the result


def test_repeatable_and_alternating_with_kld():
    import rmcl_b200
    P, A = _case(100_000, 6, "uniform")
    P["t"][:, :2] *= np.float32(0.3)
    up, c, kld = _updater(), cfg(), rmcl_b200.KLDConfig.defaults()
    Pd, Ad = _dev(P, A)

    def clusters(u):
        r, recs, lab = _run(u, P, A, c, dev=(Pd, Ad))
        return r.tobytes() + recs.tobytes() + lab.tobytes()

    def kld_run(u):
        Pn, An = _out(500_000)
        r = u.resampleKLD(Pd, Ad, Pn, An, kld, CFG, seed=5, step=9)
        gP, gA = _np(Pn, An)
        return r.tobytes() + gP.tobytes() + gA.tobytes()

    a = clusters(up)
    k0 = kld_run(up)
    assert clusters(up) == a and kld_run(up) == k0 and clusters(up) == a
    other = rmcl_b200.PCDSensorUpdaterB200(gpu_map("cube29"))
    assert kld_run(other) == k0 and clusters(other) == a
    r, recs, _ = _run(up, P, A, c, dev=(Pd, Ad), labels=False)      # labels are optional
    assert r.tobytes() + recs.tobytes() == a[:len(r.tobytes() + recs.tobytes())]


def test_refusals_launch_nothing_and_write_nothing():
    import ctypes as C
    import torch
    import rmcl_b200
    from rmcl_b200.api import _devptr
    from rmcl_b200.synth import CLUSTER_RECORD_DTYPE, CLUSTER_RESULT_DTYPE
    up, lib, chk = _updater(), rmcl_b200.load_library(), rmcl_b200.api._chk
    P, A = _case(300, 1, "uniform")
    Pd, Ad = _dev(P, A)
    lab = torch.full((300,), 7, dtype=torch.int32, device="cuda")
    out, recs = np.zeros((), CLUSTER_RESULT_DTYPE), np.zeros(16, CLUSTER_RECORD_DTYPE)
    out["rounds"], recs["key"] = 99, 5

    def call(h=True, p=Pd, a=Ad, n=300, k=True, rec=True, o=True, **kw):
        kc = cfg(**kw)
        ptr = lambda t: None if t is None else _devptr(t)
        return chk(lib.b2_pf_cluster_stats(up._h if h else None, ptr(p), ptr(a), C.c_uint32(n), C.byref(kc) if k else None,
                                           C.c_void_p(recs.ctypes.data) if rec else None, _devptr(lab), C.c_void_p(out.ctypes.data) if o else None))

    def refused(what, **kw):
        before = rmcl_b200.kernel_launch_count()
        with pytest.raises(rmcl_b200.B2Error) as e:
            call(**kw)
        assert e.value.code == -1 and what in str(e.value), str(e.value)
        assert rmcl_b200.kernel_launch_count() == before
        assert int(out["rounds"]) == 99 and np.all(recs["key"] == 5) and bool((lab == 7).all())
        assert lib.b2_peek_cuda_error().decode() == ""

    refused("'h'", h=False)
    refused("poses_dev", p=None)
    refused("attrs_dev", a=None)
    refused("cfg", k=False)
    refused("records_host", rec=False)
    refused("out_host", o=False)
    refused("particles", n=0)
    refused("particles", n=2 ** 30 + 1)
    for v in (0.0, -0.5, float("nan"), float("inf")):
        refused("res_xy", res_xy=v)
    for v in (-0.1, float("nan"), float("inf")):
        refused("res_z", res_z=v)
    for v in (0.0, -0.1, float("nan"), float("inf"), 2 * math.pi / 40000):
        refused("yaw sectors", res_yaw=v)
    for v in (0, 17, 2 ** 32 - 1):
        refused("max_records", max_records=v)
    call()                                                          # the same arguments, valid: it runs
    assert int(out["n_clusters"]) >= 1 and int(out["rounds"]) >= 1


def _pose_error(stats, gx, gy, yaw):
    x, y, z, w = (float(v) for v in stats["orientation"])
    e_yaw = math.atan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z)) - yaw
    return math.hypot(float(stats["position"][0]) - gx, float(stats["position"][1]) - gy), abs((e_yaw + math.pi) % (2 * math.pi) - math.pi)


def test_the_hypotheses_collapse_as_the_filter_converges():
    """End to end on building:200000, the cycle of test_gpu_pf_kld's end-to-end case (a uniform initialisation around the true pose, then sensor
    update -> motion -> resampleKLD with a sharp sensor model) with estimateClusters after every sensor update: the occupied bins fall, and at
    the end the best hypothesis holds more than 90 % of the weight and lies within 0.1 m and 2 deg of the true pose."""
    import torch
    import rmcl_b200
    from rmcl_b200 import synth
    gmap = gpu_map("building:200000")
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gmap)
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(m); h.find(Tgt)
    beams = synth.pf_beams(h.modelView()["points"], 180)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    gx, gy, gz = (float(v) for v in Tgt["t"])
    yaw = math.radians(30.0)
    n_max = 1_000_000
    bufs = [(torch.empty((n_max, 8), dtype=torch.float32, device="cuda"), torch.empty((n_max, 9), dtype=torch.float32, device="cuda")) for _ in range(2)]
    up.initSamplesUniform(*bufs[0], [gx - 2.0, gy - 2.0, gz, 0.0, 0.0, yaw - 1.0], [gx + 2.0, gy + 2.0, gz, 0.0, 0.0, yaw + 1.0], 7)
    prm, kld = rmcl_b200.PFParams.defaults(), rmcl_b200.KLDConfig.defaults()
    prm.dist_sigma = 0.05
    still = synth.make_transform((0.0, 0.0, 0.0), (0.0, 0.0, 0.0))
    n, cur, trace = n_max, 0, []
    for step in range(31):
        P, A = bufs[cur][0][:n], bufs[cur][1][:n]
        up.update(P, A, Tsb, beams, prm)
        r, recs = up.estimateClusters(P, A)
        assert int(recs["weight_int"].sum()) <= int(r["weight_total"]) and int(r["n_clustered"]) <= n
        trace.append((n, int(r["n_clusters"]), int(r["bins"]), round(float(recs["weight"][0]), 3)))
        if step == 30:
            break
        up.motionUpdate(P, A, still, 0.02)
        n, cur = int(up.resampleKLD(P, A, *bufs[1 - cur], kld, rmcl_b200.GladiatorConfig.defaults(), seed=11, step=step)["n_particles"]), 1 - cur
    e_t, e_yaw = _pose_error(recs["stats"][0], gx, gy, yaw)
    print(f"clusters: (n, n_clusters, bins, weight of rank 0) per cycle {trace}; rank 0: translation error {e_t:.3f} m, yaw error {math.degrees(e_yaw):.2f} deg")
    assert trace[0][2] >= 10 * trace[-1][2], trace
    assert float(recs["weight"][0]) > 0.9 and e_t < 0.1 and e_yaw < math.radians(2.0), (trace[-1], e_t, math.degrees(e_yaw))


def test_two_modes_give_two_records_and_the_global_mean_lies_at_neither():
    """a bimodal set from two initSamples calls, 60 % / 40 %, 12 m apart: two records at the two modes, while estimateStats lies between them"""
    import torch
    import rmcl_b200
    from rmcl_b200 import synth
    up = _updater()
    n, n_a = 200_000, 120_000
    P, A = torch.empty((n, 8), dtype=torch.float32, device="cuda"), torch.empty((n, 9), dtype=torch.float32, device="cuda")
    cov = np.diag([0.09, 0.09, 0.0, 0.0, 0.0, math.radians(5.0) ** 2]).reshape(36)
    modes = [synth.make_transform((-6.0, 1.0, 0.0), (0.0, 0.0, 0.5)), synth.make_transform((6.0, 1.0, 0.0), (0.0, 0.0, -2.0))]
    up.initSamples(P[:n_a], A[:n_a], modes[0], cov, 3)
    up.initSamples(P[n_a:], A[n_a:], modes[1], cov, 4)
    A[:, 0] = 1.0                                                   # likelihood.mean: equal weights
    r, recs = up.estimateClusters(P, A)
    assert int(r["n_clusters"]) >= 2 and int(r["n_clustered"]) == n
    assert abs(float(recs["weight"][0]) - 0.6) < 0.01 and abs(float(recs["weight"][1]) - 0.4) < 0.01, recs["weight"]
    for rec, mode, yaw in zip(recs[:2], modes, (0.5, -2.0)):
        e_t, e_yaw = _pose_error(rec["stats"], float(mode["t"][0]), float(mode["t"][1]), yaw)
        assert e_t < 0.05 and e_yaw < math.radians(1.0), (e_t, e_yaw)
    whole = up.estimateStats(P, A, max_induction_particles=n)
    for mode in modes:
        assert math.hypot(float(whole["position"][0]) - float(mode["t"][0]), float(whole["position"][1]) - float(mode["t"][1])) > 4.0


def test_cpp_classes_match_python(tmp_path):
    """tests/pf_cluster_cpp/pf_cluster_cpp.cpp, compiled here against include/rmcl_b200/rcc_b200.hpp, clusters device particles through
    PCDSensorUpdaterB200::estimateClusters with its cluster_config: byte for byte what the Python path gives"""
    import rmcl_b200
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "pf_cluster_cpp")
    lib_dir = os.path.dirname(rmcl_b200.lib_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "pf_cluster_cpp", "pf_cluster_cpp.cpp"), "-L" + lib_dir, "-lrmcl_b200",
                           "-L" + os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + lib_dir])
    P, A = _case(20_000, 12, "uniform")
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(np.array([len(P)], np.uint32).tobytes())
        f.write(P.tobytes()); f.write(A.tobytes())
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "REFUSED" in r.stdout and "max_records" in r.stdout
    rec, recs, lab = _run(_updater(), P, A, rmcl_b200.ClusterConfig.defaults())
    assert int(rec["n_clusters"]) > 8 and len(recs) == 8
    assert np.fromfile(out, np.uint8).tobytes() == rec.tobytes() + recs.tobytes() + lab.tobytes()
