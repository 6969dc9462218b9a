"""b2_micp_pose_covariance on an H100 (pytest -m gpu): pair counts against b2_rcc_cross_statistics, sums against a float64 restatement over
the downloaded buffers, sensors adding up, closed-form degeneracies of simple scenes, consistency with the scatter of noisy corrections,
repeatability, refusals and the C++ mirror (SURVEY appendix I)."""
import ctypes as C
import math
import subprocess

import numpy as np
import pytest

from conftest import gpu_map
import chain_ref
import micp_cov_ref as ref
import native
import pf_estimate_ref

pytestmark = pytest.mark.gpu
DV = 1e2


def _rect(V, F, corner, eu, ev):
    """two triangles spanning corner, corner + eu, corner + eu + ev, corner + ev"""
    c, eu, ev = (np.asarray(a, np.float32) for a in (corner, eu, ev))
    b = len(V)
    V += [c, c + eu, c + eu + ev, c + ev]
    F += [[b, b + 1, b + 2], [b, b + 2, b + 3]]


def _scene(kind):
    V, F = [], []
    if kind in ("box", "room", "walls"):
        lo, hi = {"box": ([-5.0, -4.0, 0.0], [5.0, 4.0, 3.0]), "room": ([-4.0, -4.0, -4.0], [4.0, 4.0, 4.0]), "walls": ([-5.0, -4.0, -30.0], [5.0, 4.0, 30.0])}[kind]
        lo, hi = np.array(lo), np.array(hi)
        dx, dy, dz = hi - lo
        _rect(V, F, lo, (dx, 0, 0), (0, 0, dz)); _rect(V, F, (lo[0], hi[1], lo[2]), (dx, 0, 0), (0, 0, dz))
        _rect(V, F, lo, (0, dy, 0), (0, 0, dz)); _rect(V, F, (hi[0], lo[1], lo[2]), (0, dy, 0), (0, 0, dz))
        if kind != "walls":
            _rect(V, F, lo, (dx, 0, 0), (0, dy, 0)); _rect(V, F, (lo[0], lo[1], hi[2]), (dx, 0, 0), (0, dy, 0))
    elif kind == "corridor":                        # along x, 1 km long: no ray of the sensor reaches an end
        lo, hi = np.array([-500.0, -1.5, 0.0]), np.array([500.0, 1.5, 3.0])
        dx = hi[0] - lo[0]
        _rect(V, F, lo, (dx, 0, 0), (0, 3.0, 0)); _rect(V, F, (lo[0], lo[1], hi[2]), (dx, 0, 0), (0, 3.0, 0))
        _rect(V, F, lo, (dx, 0, 0), (0, 0, 3.0)); _rect(V, F, (lo[0], hi[1], lo[2]), (dx, 0, 0), (0, 0, 3.0))
    elif kind == "floor":
        _rect(V, F, (-200.0, -200.0, 0.0), (400.0, 0, 0), (0, 400.0, 0))
    return np.array(V, np.float32), np.array(F, np.uint32)


_MAPS = {}


def _map(kind):
    import rmcl_b200
    if kind not in _MAPS:
        _MAPS[kind] = rmcl_b200.Map(*_scene(kind), device=0, build_mode=1)
    return _MAPS[kind]


def _scan(h, m, Tbm, sigma, seed):
    """the handle's own ray cast at Tbm as the scan, with N(0, sigma) range noise; misses become range_max + 1"""
    h.find(Tbm)
    mv = h.modelView()
    r = np.where(mv["hits"] > 0, mv["ranges"], np.float32(m.range_max + 1.0)).astype(np.float32)
    if sigma > 0:
        r = np.where(mv["hits"] > 0, r + np.random.default_rng(seed).normal(0.0, sigma, r.shape).astype(np.float32), r).astype(np.float32)
    return r


def _spherical(synth, map_, m, Tsb):
    import rmcl_b200
    h = rmcl_b200.RCCB200Spherical(map_)
    h.setTsb(Tsb); h.setModel(m); h.setParams(1.0, 0.15)
    return h


def _restated(hs, Tbo, w, Td, cp, Tref):
    """per sensor (n accepted, H, R2, Q2) over the downloaded buffers with the product's gate, in float64"""
    out = []
    for k, h in enumerate(hs):
        dv, mv = h.datasetView(), h.modelView()
        Tpre = ref.product_pretransform(Tbo[k], h._Tsb, Td)
        ok, r = ref.product_gate(Tpre, dv["points"], dv["mask"], mv["points"], mv["normals"], mv["hits"], chain_ref.product_gate(h._max_dist, 0.15, cp))
        H, R2, Q2, W = ref.information_np(np.asarray(dv["points"]).reshape(-1, 3)[ok], np.asarray(mv["normals"]).reshape(-1, 3)[ok], r[ok],
                                          *ref.frames(Tref, Tbo[k], h._Tsb, Tpre))
        out.append((int(ok.sum()), w[k] * H, w[k] * R2, w[k] * Q2, w[k] * W))
    return out


def _check_counts_and_sums(hs, Tbo, Td, cp, w=None, Tref=None):
    import rmcl_b200
    w = [1.0] * len(hs) if w is None else list(w)
    Tref = Tbo[0] if Tref is None else Tref
    rec = rmcl_b200.micp_pose_covariance(hs, Tbo, Td, cp, merge_weights=w, Tbo_ref=Tref)
    for k, h in enumerate(hs):
        Tpre = ref.product_pretransform(Tbo[k], h._Tsb, Td)
        assert int(rec["n_pairs"][k]) == int(h.computeCrossStatistics(Tpre, cp)["n_meas"]), k
    parts = _restated(hs, Tbo, w, Td, cp, Tref)
    assert [p[0] for p in parts] == [int(x) for x in rec["n_pairs"][:len(hs)]]
    H = sum(p[1] for p in parts)
    R2, Q2, W = (sum(p[i] for p in parts) for i in (2, 3, 4))
    got = rec["information"].reshape(6, 6)
    assert np.linalg.norm(got - H) <= 1e-5 * np.linalg.norm(H)
    assert abs(rec["residual_sq_sum"] - R2) <= 1e-5 * R2 and abs(rec["weight_sum"] - W) <= 1e-9 * W
    assert abs(rec["length_scale"] ** 2 * rec["weight_sum"] - Q2) <= 1e-5 * Q2
    assert abs(np.trace(got[:3, :3]) - rec["weight_sum"]) <= 1e-5 * rec["weight_sum"]          # unit normals
    assert W > 100
    return rec


def _remember(h, Tsb, max_dist=1.0):
    h._Tsb, h._max_dist = Tsb, max_dist
    return h


@pytest.fixture(scope="module")
def building_c2(synth):
    gm = gpu_map("building:1000000")
    m, Tsb = synth.c2_sensor(), synth.scenario_tsb()
    h = _remember(_spherical(synth, gm, m, Tsb), Tsb)
    Tgt = synth.building_gt_pose()
    h.setRanges(_scan(h, m, Tgt, 0.01, 1))
    Tom = synth.compose(Tgt, synth.scenario_pose_offset())
    return h, m, Tsb, Tgt, Tom


def test_counts_and_sums_c2_building(synth, building_c2):
    """C2 over building:1000000 after micp_correct_once in exec modes 0, 1 and 2 and after a 3-step micp_correct: n_pairs equals
    b2_rcc_cross_statistics(T_snew_sold, cp).n_meas, the sums equal the float64 restatement within 1e-5"""
    import rmcl_b200
    h, m, Tsb, Tgt, Tom = building_c2
    I = synth.make_transform()
    for mode in (2, 1, 0):
        h.setExecMode(mode)
        Tn, Td, Cm = rmcl_b200.micp_correct_once([h], np.stack([I]), Tom, 5, 0.0)
        rec = _check_counts_and_sums([h], np.stack([I]), Td, 0.0)
        assert int(rec["n_pairs"][0]) > 50_000 and int(rec["n_degenerate"]) == 0
    h.setExecMode(2)
    T, cp, steps = rmcl_b200.micp_correct([h], np.stack([I]), Tom, n_corrections=3, convergence_progress=0.0)
    _check_counts_and_sums([h], np.stack([I]), steps[-1]["T_onew_oold"], float(steps[-2]["convergence_progress"]))


def test_repeatable_and_leaves_the_handle_alone(synth, building_c2):
    """repeated calls give the same bytes; a correctOnce after the call equals one without it bit for bit"""
    import rmcl_b200
    h, m, Tsb, Tgt, Tom = building_c2
    Tbo = np.stack([synth.make_transform()])
    first = rmcl_b200.micp_correct_once([h], Tbo, Tom, 5, 0.0)
    recs = [rmcl_b200.micp_pose_covariance([h], Tbo, first[1], 0.0) for _ in range(3)]
    assert recs[0].tobytes() == recs[1].tobytes() == recs[2].tobytes()
    after = rmcl_b200.micp_correct_once([h], Tbo, Tom, 5, 0.0)
    plain = rmcl_b200.micp_correct_once([h], Tbo, Tom, 5, 0.0)
    for a, b, c in zip(first, after, plain):
        assert a.tobytes() == b.tobytes() == c.tobytes()


def test_two_sensors_and_closest_point(synth):
    """two sensors with different Tsb, Tbo and weights: counts and sums per sensor, and the pair equals the weighted sum of each alone (same
    Tbo_ref) within 1e-9; a closest-point handle likewise"""
    import rmcl_b200
    gm = _map("box")
    Tgt = synth.make_transform((1.0, -0.7, 0.2), (0.0, 0.0, 0.3))
    m1, m2 = synth.c1_sensor(), synth.SphericalModel(math.radians(-30.0), math.radians(60.0) / 15, 16, -math.pi, 2 * math.pi / 128, 128, 0.1, 100.0)
    Tsb1, Tsb2 = synth.make_transform((0.1, 0.0, 0.8), (0, 0, 0.05)), synth.make_transform((-0.1, 0.1, 1.0), (0.0, 0.1, -0.4))
    Tbo = np.stack([synth.make_transform((0.02, 0.0, 0.0), (0, 0, 0.01)), synth.make_transform((0.0, 0.03, 0.0), (0, 0, -0.02))])
    hs = []
    for k, (m, Tsb) in enumerate(((m1, Tsb1), (m2, Tsb2))):
        h = _remember(_spherical(synth, gm, m, Tsb), Tsb)
        h.setRanges(_scan(h, m, synth.compose(Tgt, Tbo[k]), 0.01, 10 + k))
        hs.append(h)
    Tom = synth.compose(Tgt, synth.make_transform((0.05, -0.04, 0.02), (0.0, 0.0, 0.02)))          # the scans were taken at Tom = Tgt
    w = [0.7, 1.8]
    Tn, Td, Cm = rmcl_b200.micp_correct_once(hs, Tbo, Tom, 5, 0.0, merge_weights=w)
    both = _check_counts_and_sums(hs, Tbo, Td, 0.0, w)
    alone = [rmcl_b200.micp_pose_covariance([hs[k]], Tbo[k:k + 1], Td, 0.0, merge_weights=[w[k]], Tbo_ref=Tbo[0]) for k in range(2)]
    Hsum = alone[0]["information"] + alone[1]["information"]
    assert np.linalg.norm(both["information"] - Hsum) <= 1e-9 * np.linalg.norm(Hsum)
    for f in ("residual_sq_sum", "weight_sum"):
        assert abs(both[f] - alone[0][f] - alone[1][f]) <= 1e-9 * both[f]
    assert [int(x) for x in both["n_pairs"][:2]] == [int(alone[0]["n_pairs"][0]), int(alone[1]["n_pairs"][0])]
    # a closest-point handle over the first sensor's dataset
    dv = hs[0].datasetView()
    hc = _remember(rmcl_b200.CPCB200(gm), Tsb1)
    hc.setTsb(Tsb1); hc.setParams(1.0, 0.15); hc.setDataset(dv["points"], dv["mask"])
    Tn, Td, Cm = rmcl_b200.micp_correct_once([hc], Tbo[:1], Tom, 5, 0.0)
    _check_counts_and_sums([hc], Tbo[:1], Td, 0.0)


def _corrected(synth, kind, m, Tsb, Tgt, pinhole=False, sigma=0.01):
    import rmcl_b200
    gm = _map(kind)
    if pinhole:
        h = rmcl_b200.RCCB200Pinhole(gm); h.setTsb(Tsb); h.setModel(m); h.setParams(1.0, 0.15)
    else:
        h = _spherical(synth, gm, m, Tsb)
    _remember(h, Tsb)
    h.setRanges(_scan(h, m, Tgt, sigma, 5))
    Tbo = np.stack([synth.make_transform()])
    Tom = synth.compose(Tgt, synth.make_transform((0.03, -0.02, 0.01), (0.0, 0.0, 0.01)))
    Tn, Td, Cm = rmcl_b200.micp_correct_once([h], Tbo, Tom, 5, 0.0)
    return rmcl_b200.micp_pose_covariance([h], Tbo, Td, 0.0, degenerate_variance=DV)


def _span_contains(rec, axis):
    P = rec["eigenvectors"].reshape(6, 6)[[i for i in range(6) if rec["degenerate_mask"] >> i & 1]]
    return float(np.linalg.norm(P @ np.eye(6)[axis]))


def test_geometry_closed_form(synth):
    """box room: no degenerate direction; corridor along x: exactly one, along x, with covariance[0] within 1 % of degenerate_variance;
    walls only: z degenerate; a pinhole looking down at one floor plane: exactly three, spanning x, y and yaw"""
    m = synth.c1_sensor()
    Tsb = synth.make_transform((0.1, 0.0, 0.3))
    box = _corrected(synth, "box", m, Tsb, synth.make_transform((1.0, -0.7, 0.9), (0.0, 0.0, 0.3)))
    assert int(box["n_degenerate"]) == 0 and np.isfinite(box["covariance"]).all()
    cor = _corrected(synth, "corridor", m, Tsb, synth.make_transform((0.0, 0.2, 0.9), (0.0, 0.0, 0.0)))       # body x along the corridor
    assert int(cor["n_degenerate"]) == 1, cor["eigenvalues"]
    v = cor["eigenvectors"].reshape(6, 6)[int(np.log2(int(cor["degenerate_mask"])))]
    assert abs(v[0]) >= 0.999, v
    assert abs(cor["covariance"][0] - DV) <= 0.01 * DV
    walls = _corrected(synth, "walls", m, Tsb, synth.make_transform((1.0, -0.7, 0.9), (0.0, 0.0, 0.3)))
    assert int(walls["n_degenerate"]) >= 1 and _span_contains(walls, 2) >= 0.999, walls["eigenvalues"]
    cam = synth.PinholeModel(64, 48, 40.0, 40.0, 31.5, 23.5, 0.1, 50.0)
    Tsb_down = synth.make_transform((0.0, 0.0, 0.0), (0.0, math.pi / 2, 0.0))       # the optical axis (x) turned to -z
    fl = _corrected(synth, "floor", cam, Tsb_down, synth.make_transform((2.0, 1.0, 2.5), (0.0, 0.0, 0.4)), pinhole=True)
    assert int(fl["n_degenerate"]) == 3, fl["eigenvalues"]
    for axis in (0, 1, 5):
        assert _span_contains(fl, axis) >= 0.999, (axis, fl["eigenvectors"])


def test_consistency_with_noisy_corrections(synth):
    """Closed room, C1, Gaussian range noise sigma 0.05 m, 200 trials of a 3-step micp_correct from the true pose: the scatter of
    ~Tbm_true * Tbm_est has every diagonal within a factor 2 of the mean predicted one, and the mean NEES lies in [3, 12].  The model has one
    sigma2 for all pairs (homoscedastic, SURVEY I8) while the point-to-plane noise of a range error shrinks with the cosine of the incidence,
    so the scene is chosen to show every face at similar incidence: a cube room with the scan tilted (roll 0.6, pitch 0.5 rad) out of line
    with its faces.  (In a flat 10 x 8 x 3 m box with a level scan the floor and ceiling are seen at grazing incidence and z, roll and pitch
    came out 2.3 to 2.8 times over-predicted.)"""
    import rmcl_b200
    m = synth.c1_sensor()
    Tsb = synth.make_transform((0.1, 0.0, 0.3), (0.6, 0.5, 0.0))
    Tgt = synth.make_transform((0.6, -0.4, 0.2), (0.0, 0.0, 0.3))
    h = _remember(_spherical(synth, _map("room"), m, Tsb), Tsb)
    h.find(Tgt)
    mv = h.modelView()
    hit = mv["hits"] > 0
    Tbo = np.stack([synth.make_transform()])
    rng = np.random.default_rng(2024)
    errs, covs = [], []
    for trial in range(200):
        r = np.where(hit, mv["ranges"] + rng.normal(0.0, 0.05, hit.shape), m.range_max + 1.0).astype(np.float32)
        h.setRanges(r)
        T, cp, steps = rmcl_b200.micp_correct([h], Tbo, Tgt, n_corrections=3, convergence_progress=0.0)
        rec = rmcl_b200.micp_pose_covariance([h], Tbo, steps[-1]["T_onew_oold"], float(steps[-2]["convergence_progress"]))
        assert int(rec["n_degenerate"]) == 0
        errs.append(pf_estimate_ref.deviation(Tgt, np.asarray(T).reshape(1))[0])
        covs.append(rec["covariance"].reshape(6, 6))
    E, Cs = np.array(errs), np.array(covs)
    emp = (E * E).mean(0)
    pred = np.array([c.diagonal() for c in Cs]).mean(0)
    ratio = emp / pred
    assert (ratio >= 0.5).all() and (ratio <= 2.0).all(), (emp, pred)
    nees = np.mean([e @ np.linalg.solve(c, e) for e, c in zip(E, Cs)])
    assert 3.0 <= nees <= 12.0, nees


def test_refusals_launch_nothing(synth, building_c2):
    """every refusal returns B2_ERR_INVALID, launches nothing and leaves the output as it was"""
    import rmcl_b200
    h, m, Tsb, Tgt, Tom = building_c2
    lib = rmcl_b200.load_library()
    I = synth.make_transform()
    Tbo = np.stack([I, I])
    w = np.array([1.0, 1.0])
    Td = rmcl_b200.micp_correct_once([h], Tbo[:1], Tom, 5, 0.0)[1]
    cfg = rmcl_b200.api._MicpCovConfig(1e-3, 1e2)
    fresh = _spherical(synth, gpu_map("building:1000000"), m, Tsb)                      # no find yet
    fresh.setRanges(np.full(m.phi_size * m.theta_size, 5.0, np.float32))
    other = _spherical(synth, gpu_map("building:1000000"), m, Tsb)
    other.find(Tgt)
    other.setDataset(np.zeros((10, 3), np.float32), np.ones(10, np.uint8))             # dataset size != model size

    def call(handles, n=None, Tb=Tbo, wt=w, T=Td, ref_=None, c=cfg, out=True, sensors_null=False, Tbo_null=False, T_null=False):
        arr = (C.c_void_p * max(len(handles), 1))(*[x._h for x in handles])
        rec = np.zeros(1, rmcl_b200.MICP_COVARIANCE_DTYPE)
        rec.view(np.uint8)[:] = 0xAB
        before_bytes = rec.tobytes()
        n0 = rmcl_b200.kernel_launch_count()
        Tb = np.ascontiguousarray(Tb); T = np.ascontiguousarray(T); wt = None if wt is None else np.ascontiguousarray(wt, np.float64)
        rc = lib.b2_micp_pose_covariance(None if sensors_null else arr, None if Tbo_null else C.c_void_p(Tb.ctypes.data),
                                         None if wt is None else C.c_void_p(wt.ctypes.data), C.c_uint32(len(handles) if n is None else n),
                                         None if T_null else C.c_void_p(T.ctypes.data), C.c_double(0.0),
                                         None if ref_ is None else C.c_void_p(np.ascontiguousarray(ref_).ctypes.data),
                                         None if c is None else C.byref(c), C.c_void_p(rec.ctypes.data) if out else None)
        assert rmcl_b200.kernel_launch_count() == n0
        assert rec.tobytes() == before_bytes
        return rc

    nan_T = np.array(Td, copy=True); nan_T["t"][0] = np.nan
    one = dict(Tb=Tbo[:1], wt=[1.0])
    for kwargs in (dict(sensors_null=True), dict(Tbo_null=True), dict(T_null=True), dict(c=None), dict(out=False), dict(n=0), dict(n=5),
                   dict(T=nan_T), dict(ref_=nan_T), dict(Tb=np.stack([nan_T])), dict(wt=[-1.0]), dict(wt=[np.inf]),
                   dict(c=rmcl_b200.api._MicpCovConfig(0.0, 1e2)), dict(c=rmcl_b200.api._MicpCovConfig(1.0, 1e2)),
                   dict(c=rmcl_b200.api._MicpCovConfig(np.nan, 1e2)), dict(c=rmcl_b200.api._MicpCovConfig(1e-3, 0.0)),
                   dict(c=rmcl_b200.api._MicpCovConfig(1e-3, np.inf))):
        assert call([h], **{**one, **kwargs}) == -1, kwargs                          # n = 5: refused before a handle is read
    assert call([h, h], Tb=Tbo) == -1                                                # the same handle twice
    assert call([fresh], Tb=Tbo[:1], wt=[1.0]) == -1                                 # no find yet
    assert call([other], Tb=Tbo[:1], wt=[1.0]) == -1                                 # dataset size != model size
    h.correctOnceAsync(Tom, I, 5, 0.0)                                               # calls in flight
    assert call([h], Tb=Tbo[:1], wt=[1.0]) == -1
    h.correctOnceWait()
    assert lib.b2_peek_cuda_error().decode() == ""


def test_cpp_mirror_matches_python(synth, tmp_path):
    """tests/micp_cov_cpp/micp_cov_cpp.cpp, compiled here against include/rmcl_b200/rcc_b200.hpp: rmcl::micp_correct then
    rmcl::micp_pose_covariance give the same bytes as the Python path"""
    import rmcl_b200
    exe = native.adapter("micp_cov_cpp")
    V, F = _scene("box")
    m = synth.c1_sensor()
    Tsb = synth.make_transform((0.1, 0.0, 0.3))
    Tgt = synth.make_transform((1.0, -0.7, 0.9), (0.0, 0.0, 0.3))
    h = _spherical(synth, _map("box"), m, Tsb)
    ranges = _scan(h, m, Tgt, 0.02, 9)
    Tom = synth.compose(Tgt, synth.make_transform((0.05, 0.03, -0.02), (0.0, 0.0, 0.02)))
    hp = _spherical(synth, _map("box"), m, Tsb)
    hp.setRanges(ranges)
    Tbo = np.stack([synth.make_transform()])
    T, cp, steps = rmcl_b200.micp_correct([hp], Tbo, Tom, n_corrections=3)
    rec = rmcl_b200.micp_pose_covariance([hp], Tbo, steps[-1]["T_onew_oold"], float(steps[-2]["convergence_progress"]))
    model = np.array([(m.phi_min, m.phi_inc, m.phi_size, m.theta_min, m.theta_inc, m.theta_size, m.range_min, m.range_max)],
                     dtype=[("a", "<f4"), ("b", "<f4"), ("c", "<u4"), ("d", "<f4"), ("e", "<f4"), ("f", "<u4"), ("g", "<f4"), ("h", "<f4")])
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(np.array([len(V), len(F), len(ranges)], np.uint32).tobytes())
        f.write(V.tobytes()); f.write(F.tobytes()); f.write(model.tobytes())
        f.write(np.ascontiguousarray(Tsb).tobytes()); f.write(np.ascontiguousarray(Tom).tobytes()); f.write(ranges.tobytes())
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "REFUSED" in r.stdout and "tau" in r.stdout
    assert np.fromfile(out, np.uint8).tobytes() == np.ascontiguousarray(T).tobytes() + rec.tobytes()
