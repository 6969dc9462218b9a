"""CPU tests: the product's host+device traversal / math code (rmcl_b200/csrc/*.cuh), run on the CPU through the test-only harness
tests/emul, against the oracle.  Covers the host BVH8 builder, the quantised-box traversal (conservative culling) and the op-for-op
arithmetic of find / P2L / Umeyama / ICP step / PF evaluation -- everything except the CUDA launch plumbing, which the -m gpu tests cover."""
import numpy as np
import pytest

from conftest import mesh, oracle_scene, random_rays

_EMUL = {}


def emul_scene(name):
    import pyemul
    if name not in _EMUL:
        V, F = mesh(name)
        _EMUL[name] = pyemul.Scene(V, F)
    return _EMUL[name]


@pytest.fixture(scope="module")
def pe():
    import pyemul
    pyemul.lib()
    return pyemul


@pytest.mark.parametrize("name,lo,hi", [("cube29", -9.5, 9.5), ("uvsphere:40:60", -6.0, 6.0), ("building:60000", 1.0, 2.9), ("indoor:20000", 0.2, 2.8)])
def test_traversal_bit_exact(pe, po, name, lo, hi):
    osc, esc = oracle_scene(name), emul_scene(name)
    inf = esc.info()
    assert inf["n_tris"] == len(mesh(name)[1]) and inf["max_depth"] < 30
    o, d = random_rays(20000, lo, hi, seed=2)
    t1, f1, n1, h1 = osc.intersect(o, d, brute=False)
    t2, f2, n2, h2, st = esc.intersect(o, d)
    assert np.array_equal(f1, f2) and np.array_equal(t1, t2) and np.array_equal(n1, n2) and np.array_equal(h1, h2)
    assert 1.0 < st[0] < 60.0
    # axis-aligned rays (idir clamp path) and finite tfar
    rng = np.random.default_rng(5)
    ax = np.eye(3, dtype=np.float32)[rng.integers(0, 3, 3000)] * rng.choice([-1.0, 1.0], (3000, 1)).astype(np.float32)
    a = osc.intersect(o[:3000], ax, tfar=3.0)
    b = esc.intersect(o[:3000], ax, tfar=3.0)
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[0], b[0])


def test_find_all_models_bit_exact(pe, po, synth):
    osc, esc = oracle_scene("indoor:20000"), emul_scene("indoor:20000")
    Tbm, Tsb = synth.indoor_gt_pose(), synth.scenario_tsb()
    sph = synth.SphericalModel(-0.5, 1.0 / 31, 32, -np.pi, 2 * np.pi / 64, 64, 0.1, 30.0)
    pin = synth.PinholeModel(80, 60, 65.0, 65.0, 39.5, 29.5, 0.3, 10.0)
    rng = np.random.default_rng(1)
    dirs = rng.normal(size=(500, 3)).astype(np.float32)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    o1 = synth.O1DnModel(50, 10, np.array([0.1, 0.0, 0.05], np.float32), dirs, 0.1, 20.0)
    on = synth.OnDnModel(50, 10, rng.uniform(-0.2, 0.2, (500, 3)).astype(np.float32), dirs, 0.1, 20.0)
    for m in (sph, pin, o1, on):
        o, d = po.model_rays(m)
        r1 = osc.simulate(Tbm, Tsb, o, d, m.range_max)
        r2 = esc.find(Tbm, Tsb, o, d, m.range_max)
        for k in r1:
            assert np.array_equal(r1[k], r2[k], equal_nan=True), (type(m).__name__, k)
        assert 0.3 < r1["hits"].mean() <= 1.0


def test_sim_options_parity(pe, po, synth):
    """SURVEY.md A.3 leaves three rmagine simulate() semantics open (tfar = range.max vs inf, closest hit below range.min, miss fill): both
    settings of each exist as a switch in the oracle and in the product's find_one; every combination agrees bit for bit, and each switch
    changes what it should."""
    osc, esc = oracle_scene("building:60000"), emul_scene("building:60000")
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 15, 16, -np.pi, 2 * np.pi / 256, 256, 2.0, 6.0)      # short range: both limits bite
    o, d = po.model_rays(m)
    Tbm, Tsb = synth.building_gt_pose(), synth.scenario_tsb()
    base = osc.simulate(Tbm, Tsb, o, d, m.range_max, m.range_min)
    seen = {}
    for opts in range(8):
        tf, mn, fill = opts & 1, (opts >> 1) & 1, (opts >> 2) & 1
        a = osc.simulate(Tbm, Tsb, o, d, m.range_max, m.range_min, tfar_mode=tf, min_mode=mn, miss_fill=fill)
        b = esc.find(Tbm, Tsb, o, d, m.range_max, m.range_min, sim_opts=opts)
        for k in a:
            assert np.array_equal(a[k], b[k], equal_nan=True), (opts, k)
        seen[opts] = a
    assert seen[0]["hits"].tobytes() == base["hits"].tobytes()
    assert seen[1]["hits"].sum() > seen[0]["hits"].sum() and (seen[1]["ranges"][seen[1]["hits"] > 0] > m.range_max).any()       # tfar = inf: far hits appear
    near = (seen[0]["hits"] > 0) & (seen[0]["ranges"] < m.range_min)
    assert near.any() and (seen[2]["hits"][near] == 0).all() and (seen[2]["hits"][~near] == seen[0]["hits"][~near]).all()       # hits below range.min become misses
    miss = seen[4]["hits"] == 0
    assert miss.any() and (seen[4]["points"][miss] == 0).all() and np.isnan(seen[0]["points"][miss]).all()                      # zero fill vs NaN fill
    assert (seen[4]["ranges"][miss] == np.float32(m.range_max + 1)).all()


def test_icp_chain_parity(pe, po, synth):
    osc, esc = oracle_scene("building:60000"), emul_scene("building:60000")
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 256, 256, 0.5, 120.0)
    o, d = po.model_rays(m)
    Tgt, Tsb = synth.building_gt_pose(), synth.scenario_tsb()
    ranges = synth.noisy_ranges(osc.simulate(Tgt, Tsb, o, d, m.range_max)["ranges"], m.range_max)
    dp, dm, _ = po.dataset_from_ranges(o, d, ranges, m.range_min, m.range_max)
    Tbo = synth.make_transform((0.05, 0.02, 0.0), (0, 0, 0.1))
    Tom = synth.compose(synth.compose(Tgt, synth.scenario_pose_offset()), synth.inverse(Tbo))
    a = osc.micp_correct_once(o, d, m.range_max, dp, dm, Tom, Tbo, Tsb, iterations=5, max_dist=1.0, adaptive_max_dist_min=0.15, f64_accum=True)
    b = esc.correct_once(o, d, m.range_max, dp, dm, Tom, Tbo, Tsb, 5, 1.0)
    assert a[2]["n_meas"] == b[2]["n_meas"] and a[2]["n_meas"] > 5000
    assert np.abs(a[0]["t"] - b[0]["t"]).max() <= 1e-6 and np.abs(a[0]["R"] - b[0]["R"]).max() <= 1e-6
    assert np.abs(a[1]["t"] - b[1]["t"]).max() <= 1e-6 and np.abs(a[1]["R"] - b[1]["R"]).max() <= 1e-6
    # (the chain was bit-identical while the device used the oracle's FP64 Jacobi SVD; the FP32 Newton polar iteration that replaced it
    #  on the critical path agrees to ~1e-7, see DESIGN.md section 2)
    # the lean tail of the cooperative ICP loop (pre-composed frames): same result within float noise
    c = esc.correct_once(o, d, m.range_max, dp, dm, Tom, Tbo, Tsb, 5, 1.0, fast_tail=True)
    assert abs(int(c[2]["n_meas"]) - int(a[2]["n_meas"])) <= 2
    assert np.abs(a[0]["t"] - c[0]["t"]).max() <= 2e-6 and np.abs(a[0]["R"] - c[0]["R"]).max() <= 2e-6
    assert np.abs(a[1]["t"] - c[1]["t"]).max() <= 2e-6 and np.abs(a[1]["R"] - c[1]["R"]).max() <= 2e-6


def _two_sensor_case(po, synth, osc, scale=1):
    """spherical LiDAR + pinhole camera on one robot (different Tsb / Tbo / weights), scans taken at T_gt"""
    Tgt = synth.building_gt_pose()
    m1 = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 15, 16 * scale, -np.pi, 2 * np.pi / (128 * scale), 128 * scale, 0.5, 120.0)
    m2 = synth.PinholeModel(64 * scale, 48 * scale, 52.5 * scale, 52.5 * scale, 31.5 * scale, 23.5 * scale, 0.3, 30.0)
    Tsb1, Tsb2 = synth.scenario_tsb(), synth.make_transform((0.3, 0.1, 0.4), (0.0, 0.1, -0.4))
    Tbo1, Tbo2 = synth.make_transform((0.05, 0.02, 0.0), (0, 0, 0.1)), synth.make_transform((0.04, 0.03, 0.0), (0, 0, 0.09))
    sensors = []
    for m, Tsb, Tbo, w, seed in ((m1, Tsb1, Tbo1, 1.0, 3), (m2, Tsb2, Tbo2, 0.35, 4)):
        o, d = po.model_rays(m)
        # the scan is what the sensor sees from the TRUE base pose: Tbm_gt = T_gt (map <- base)
        r = synth.noisy_ranges(osc.simulate(Tgt, Tsb, o, d, m.range_max)["ranges"], m.range_max, seed=seed)
        dp, dm, _ = po.dataset_from_ranges(o, d, r, m.range_min, m.range_max)
        sensors.append(dict(model=m, origs=o, dirs=d, range_max=m.range_max, dataset_points=dp, dataset_mask=dm, Tbo=Tbo, Tsb=Tsb, max_dist=1.0,
                            adaptive_max_dist_min=0.15, weight=w, ranges=r))
    # Tom such that Tom * Tbo1 = T_gt o offset
    Tom = synth.compose(synth.compose(Tgt, synth.scenario_pose_offset()), synth.inverse(Tbo1))
    return sensors, Tom


def test_multi_sensor_loop_parity(pe, po, synth):
    """micp_localization.cpp:915-964 over two sensors: the product's fused loop (icp_tail: pre-composed frames, weighted merge with the
    u32 *= double truncation) against the oracle's statement-by-statement restatement."""
    osc, esc = oracle_scene("building:60000"), emul_scene("building:60000")
    sensors, Tom = _two_sensor_case(po, synth, osc)
    a = osc.micp_correct_once_multi(sensors, Tom, 5, 0.0, f64_accum=True)
    b = esc.micp_multi(sensors, Tom, 5)
    assert a[2]["n_meas"] > 2000 and abs(int(a[2]["n_meas"]) - int(b[2]["n_meas"])) <= 2
    for i in (0, 1):
        assert np.abs(a[i]["t"] - b[i]["t"]).max() <= 2e-6 and min(np.abs(a[i]["R"] - b[i]["R"]).max(), np.abs(a[i]["R"] + b[i]["R"]).max()) <= 2e-6
    # the weights matter: a different camera weight changes the update
    sensors[1]["weight"] = 3.0
    c = osc.micp_correct_once_multi(sensors, Tom, 5, 0.0, f64_accum=True)
    d = esc.micp_multi(sensors, Tom, 5)
    assert np.abs(c[1]["t"] - a[1]["t"]).max() > 1e-5
    assert np.abs(c[1]["t"] - d[1]["t"]).max() <= 2e-6
    # one sensor through the multi path == the single-sensor call
    e = osc.micp_correct_once_multi(sensors[:1], Tom, 5, 0.0, f64_accum=True)
    s0 = sensors[0]
    f = osc.micp_correct_once(s0["origs"], s0["dirs"], s0["range_max"], s0["dataset_points"], s0["dataset_mask"], Tom, s0["Tbo"], s0["Tsb"], 5, 1.0, 0.15, 0.0, f64_accum=True)
    assert e[0].tobytes() == f[0].tobytes() and e[2].tobytes() == f[2].tobytes()


def test_pf_bit_exact(pe, po, synth):
    osc, esc = oracle_scene("building:60000"), emul_scene("building:60000")
    m = synth.c1_sensor()
    o, d = po.model_rays(m)
    Tsb = synth.scenario_tsb()
    pts = osc.simulate(synth.building_gt_pose(), Tsb, o, d, 80.0)["points"]
    beams = synth.pf_beams(pts, 40)
    P, A = synth.pf_particles(300)
    for ng in (0, 1):
        prm = po.PFParams.defaults(ng)
        a = osc.pf_update(P, A, Tsb, beams, prm)
        b = esc.pf_update(P, A, Tsb, beams, prm)
        assert a.tobytes() == b.tobytes()


def test_umeyama_fast_path_and_fallback(pe, po):
    """Device Umeyama (Newton polar iteration, SVD fallback) against the oracle's Jacobi SVD: goldens, reflection, rank-deficient, zero."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "umeyama.npz"))
    for s, T in zip(g["stats"], g["T"]):
        out = pe.umeyama(s)
        assert np.abs(out["t"] - T["t"]).max() <= 1e-6 and min(np.abs(out["R"] - T["R"]).max(), np.abs(out["R"] + T["R"]).max()) <= 1e-6
    rng = np.random.default_rng(3)
    for k in range(200):
        s = np.zeros((), po.CROSS_STATS)
        A = rng.normal(size=(3, 3))
        if k % 4 == 1:
            A[:, 2] *= -1e-3                      # det < 0: reflection branch
        if k % 4 == 2:
            A[2, :] = 0.0                         # rank 2
        if k % 4 == 3:
            A = np.diag(rng.uniform(0.5, 2.0, 3)) + 1e-3 * A      # near-SPD (the ICP case)
        s["covariance"] = A.T.reshape(-1).astype(np.float32)
        s["dataset_mean"], s["model_mean"], s["n_meas"] = rng.normal(size=3), rng.normal(size=3), 100
        a, b = po.umeyama(s), pe.umeyama(s)
        sv = np.linalg.svd(s["covariance"].reshape(3, 3).T.astype(np.float64), compute_uv=False)
        if sv[1] < 1e-3 * sv[0] or sv[2] < 1e-6 * sv[0]:
            continue                              # rotation not unique: nothing to compare
        q1, q2 = np.asarray(a["R"], np.float64), np.asarray(b["R"], np.float64)
        tol = 2e-6 if sv[2] > 1e-3 * sv[0] else 1e-3
        assert min(np.abs(q1 - q2).max(), np.abs(q1 + q2).max()) <= tol, (k, sv)
    z = np.zeros((), po.CROSS_STATS)
    I = pe.umeyama(z)
    assert np.allclose(I["R"], [0, 0, 0, 1]) and np.allclose(I["t"], 0)


@pytest.mark.parametrize("name,lo,hi", [("cube29", [-12] * 3, [12] * 3), ("building:60000", [-2, -2, -1], [62, 42, 4]), ("uvsphere:40:60", [-7] * 3, [7] * 3)])
def test_cpc_bit_exact(pe, po, synth, name, lo, hi):
    """Closest-point traversal of the 8-wide BVH (trace.cuh:closest_point) == the oracle's definition, bit for bit."""
    osc, esc = oracle_scene(name), emul_scene(name)
    rng = np.random.default_rng(5)
    q = rng.uniform(lo, hi, (20000, 3)).astype(np.float32)
    q[::997] = np.nan
    Tbm, Tsb = synth.make_transform([0.3, -0.2, 0.1], [0.1, 0.05, 0.7]), synth.make_transform([0.1, 0, 0.2], [0, 0, 0.1])
    a, b = osc.cpc_find(Tbm, Tsb, q, 0.8), esc.cpc_find(Tbm, Tsb, q, 0.8)
    for k in ("points", "normals", "hits", "face_ids", "dists"):
        assert np.array_equal(a[k], b[k], equal_nan=True), k
    assert 0 < a["hits"].mean() < 1


def test_pf_cpc_bit_exact(pe, po, synth):
    """PF sensor update with correspondence_type == 1 (evaluate_cpc, PCDSensorUpdaterEmbree.cpp:88-95): attrs bit-identical to the oracle."""
    osc, esc = oracle_scene("building:60000"), emul_scene("building:60000")
    m = synth.c1_sensor()
    o, d = po.model_rays(m)
    Tsb = synth.scenario_tsb()
    pts = osc.simulate(synth.building_gt_pose(), Tsb, o, d, 80.0)["points"]
    beams = synth.pf_beams(pts, 40)
    P, A = synth.pf_particles(300)
    prm = po.PFParams.defaults(0, 1)
    a, b = osc.pf_update(P, A, Tsb, beams, prm), esc.pf_update(P, A, Tsb, beams, prm)
    assert a.tobytes() == b.tobytes()
    assert not np.array_equal(a["likelihood"]["mean"], osc.pf_update(P, A, Tsb, beams, po.PFParams.defaults(0, 0))["likelihood"]["mean"])


def test_gladiator_bit_exact(pe, po, synth):
    """Device resampling code (kernels.cuh: philox4x32_10, gladiator_draws, gladiator_one) on the CPU == the oracle, bit for bit."""
    from test_oracle import _glad_particles
    n = 20000
    P, A = _glad_particles(synth, n)
    cfg = po.GladiatorConfig(0.03, 0.03, 0.01, 0.002, 0.002, 0.01, 0.3, 0.2)
    raw, nrm = po.pf_gladiator_randoms(99, 7, 1000, n - 1000)
    Pn, An = po.pf_gladiator_resample(P, A, 1000, n - 1000, raw, nrm, cfg)
    Pe, Ae, rawe, nrme = pe.gladiator(P, A, 1000, n - 1000, cfg, 99, 7)
    assert np.array_equal(raw, rawe) and np.array_equal(nrm, nrme)
    assert Pn.tobytes() == Pe.tobytes() and An.tobytes() == Ae.tobytes()


def test_segmentation_bit_exact(pe, po, synth):
    from test_oracle import _segmentation_case
    sc, m, o, d, T, Tsb, sim, real = _segmentation_case(po, synth)
    ra = po.segment(o, d, m.range_min, m.range_max, real, sim["ranges"], sim["normals"], 0.15, 0.1)
    rb = pe.segment(o, d, m.range_min, m.range_max, real, sim["ranges"], sim["normals"], 0.15, 0.1)
    assert all(np.array_equal(x, y) for x, y in zip(ra, rb))


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_random_soup_bit_exact(pe, po, seed):
    """Triangle soups with the awkward cases mixed in -- degenerate (zero-area) triangles, duplicates, slivers, coplanar sheets, coordinates
    from millimetres to hundreds of metres: ray hits and closest points of the device traversal code equal the oracle's brute force."""
    import pyemul
    rng = np.random.default_rng(100 + seed)
    n = 400
    scale = [1e-3, 1.0, 300.0, 1.0][seed]
    c = rng.uniform(-1, 1, (n, 1, 3)) * scale
    tri = c + rng.normal(0, 0.15 * scale, (n, 3, 3))
    tri[:20, 2] = tri[:20, 1]                                   # zero-area (two equal vertices)
    tri[20:40] = tri[40:60]                                     # exact duplicates (tie -> lower face id)
    tri[60:80, :, 2] = 0.25 * scale                             # a coplanar sheet
    tri[80:100, 2] = tri[80:100, 0] + (tri[80:100, 1] - tri[80:100, 0]) * 0.5 + rng.normal(0, 1e-6 * scale, (20, 3))   # slivers
    V = tri.reshape(-1, 3).astype(np.float32)
    F = np.arange(3 * n, dtype=np.uint32).reshape(n, 3)
    osc, esc = po.Scene(V, F), pyemul.Scene(V, F)
    o = (rng.uniform(-1.5, 1.5, (4000, 3)) * scale).astype(np.float32)
    d = rng.normal(size=(4000, 3)); d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    d[:300, rng.integers(0, 3)] = 0.0                           # axis-parallel components
    tb, fb, nb, hb = osc.intersect(o, d, brute=True)
    te, fe, ne, he, _ = esc.intersect(o, d)
    assert np.array_equal(hb, he) and np.array_equal(fb, fe) and np.array_equal(tb, te) and np.array_equal(nb, ne)
    assert 0.05 < hb.mean() < 0.99
    I = np.zeros((), pyemul.TRANSFORM); I["R"][3] = 1.0
    q = (rng.uniform(-1.5, 1.5, (3000, 3)) * scale).astype(np.float32)
    q[:200] = V[rng.integers(0, len(V), 200)]                   # queries ON vertices
    a, b = osc.cpc_find(I, I, q, 0.1 * scale, brute=True), esc.cpc_find(I, I, q, 0.1 * scale)
    for k in ("points", "hits", "face_ids", "dists"):
        assert np.array_equal(a[k], b[k], equal_nan=True), k


def test_motion_update_collision_bit_exact(pe, po, synth):
    from test_oracle import _motion_case
    osc, esc = oracle_scene("cube29"), emul_scene("cube29")
    P, A, T = _motion_case(synth)
    for collide in (False, True):
        a = po.pf_motion_update(P, A, T, 0.03, scene=osc if collide else None)
        b = esc.pf_motion(P, A, T, 0.03, collide)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def test_refit_bit_exact(pe, po, synth):
    """b2_mesh_refit's per-node code on the CPU: after the vertices moved, rays and closest points on the refitted tree equal the oracle
    on the moved mesh."""
    import pyemul
    V, F = mesh("building:60000")
    esc = pyemul.Scene(V, F)
    rng = np.random.default_rng(21)
    V2 = (V + rng.normal(0, 0.02, V.shape)).astype(np.float32)
    V2[:, 0] += (0.3 * np.sin(V[:, 1] * 0.2)).astype(np.float32)
    esc.refit(V2, F)
    osc2 = po.Scene(V2, F)
    o, d = random_rays(20000, 1.0, 2.9, seed=22)
    o[:, 0] *= 20; o[:, 1] *= 13
    t1, f1, n1, h1 = osc2.intersect(o, d)
    t2, f2, n2, h2, _ = esc.intersect(o, d)
    assert np.array_equal(h1, h2) and np.array_equal(f1, f2) and np.array_equal(t1, t2) and np.array_equal(n1, n2)
    I = np.zeros((), pyemul.TRANSFORM); I["R"][3] = 1.0
    q = rng.uniform([1, 1, 0.2], [59, 39, 2.8], (5000, 3)).astype(np.float32)
    a, b = osc2.cpc_find(I, I, q, 1.0), esc.cpc_find(I, I, q, 1.0)
    assert np.array_equal(a["face_ids"], b["face_ids"]) and np.array_equal(a["dists"], b["dists"])
