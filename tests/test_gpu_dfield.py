"""GPU tests of the truncated distance field (b2_dfield_*, b2_pf_sensor_update_field) against the product's functions compiled for the
host (tests/dfield_ref.py, dfield_ref/dfield_emul.cu): the device build, the lookup and the update are bit-identical to them.  The field's
relation to the oracle and the float64 restatements is pinned by tests/test_dfield.py.

Tolerances.
  * download, query, update: exact (bytes).
  * field update vs closest-point update (fresh attributes, so each mean is the average of the beams' evaluations): per beam at most
    max(exp(-1/2) / (sigma denom) ((sqrt(3)/2) h + 1e-4), exp(-(trunc - sqrt(3) h)^2 / (2 sigma^2)) / denom) apart (DESIGN section 4,
    include/rmcl_b200.h), plus 2e-6 of float merging.
  * PF cycle: after ten rounds both estimates are within 0.3 m / 0.15 rad of the true pose and within 0.3 m of each other."""
import math

import numpy as np
import pytest

import dfield_ref as R
from conftest import gpu_map, mesh

pytestmark = pytest.mark.gpu


def _grid(name, h, trunc):
    V, F = mesh(name)
    lo, hi = R.default_box(V, trunc)
    return R.Grid(lo, hi, h, trunc)


def _product(name):
    V, F = mesh(name)
    return R.ProductField(V, F)


_HOST = {}


def _host_field(name, h, trunc):
    key = (name, h, trunc)
    if key not in _HOST:
        g = _grid(name, h, trunc)
        _HOST[key] = (g,) + _product(name).build(g)
    return _HOST[key]


def _dev(P, A):
    import torch
    return (torch.from_numpy(np.ascontiguousarray(P).view(np.float32).reshape(-1, 8).copy()).cuda(),
            torch.from_numpy(np.ascontiguousarray(A).view(np.float32).reshape(-1, 9).copy()).cuda())


def _np_attrs(Ad):
    from rmcl_b200 import synth
    return Ad.cpu().numpy().reshape(-1).view(synth.PARTICLE_ATTR_DTYPE)


@pytest.mark.parametrize("name,h,trunc", [("indoor:500000", 0.1, 1.0), ("building:1000000", 0.25, 1.0)])
def test_download_equals_the_host_build(name, h, trunc):
    import rmcl_b200
    f = rmcl_b200.DistanceField(gpu_map(name), h, trunc)
    g, index, bricks = _host_field(name, h, trunc)
    inf = f.info()
    assert inf["dims"] == g.dims and inf["brick_dims"] == g.bdims and inf["bricks_total"] == g.n_bricks
    assert np.array_equal(np.asarray(inf["origin"], np.float32), g.lo) and inf["inv_resolution"] == g.inv_h
    assert inf["bricks_allocated"] == len(bricks) and inf["bytes"] == 4 * g.n_bricks + 2916 * len(bricks)
    di, db = f.download()
    assert di.tobytes() == index.tobytes() and db.tobytes() == bricks.tobytes()
    print(f"{name} h {h} trunc {trunc}: {inf['bricks_allocated']} / {inf['bricks_total']} bricks, {inf['bytes'] / 2 ** 20:.1f} MiB, build {inf['build_ms']:.1f} ms")


def test_query_equals_the_host_lookup():
    import rmcl_b200
    import torch
    name, h, trunc = "indoor:500000", 0.1, 1.0
    f = rmcl_b200.DistanceField(gpu_map(name), h, trunc)
    g, index, bricks = _host_field(name, h, trunc)
    rng = np.random.default_rng(7)
    pts = rng.uniform(g.lo - 1.0, g.lo + np.array(g.dims) * g.h + 1.0, (1_000_000, 3)).astype(np.float32)
    pts[:6] = [[np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 0], [1e30, 0, 0], g.lo, g.lo + (np.array(g.dims) - 1).astype(np.float32) * np.float32(g.h)]
    want = R.lookup(g, index, bricks, pts)
    got = f.query(pts)
    assert got.tobytes() == want.tobytes()
    got_d = f.query(torch.from_numpy(pts).cuda())
    assert got_d.cpu().numpy().tobytes() == want.tobytes()


def _pf_case(n, n_beams, seed):
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    P = synth.transforms(n)
    P["t"] = rng.uniform((0.5, 0.5, 0.2), (11.5, 7.5, 2.5), (n, 3)).astype(np.float32)
    yaw = rng.uniform(-np.pi, np.pi, n)
    P["R"][:, 2], P["R"][:, 3] = np.sin(yaw / 2), np.cos(yaw / 2)
    A = np.zeros(n, synth.PARTICLE_ATTR_DTYPE)
    A["likelihood"]["mean"] = rng.uniform(0, 0.2, n).astype(np.float32)
    A["likelihood"]["sigma"] = rng.uniform(0, 0.01, n).astype(np.float32)
    A["likelihood"]["n_meas"] = rng.choice([0, 3, 9999, 10000], n)
    B = np.zeros(n_beams, synth.RANGE_MEAS_DTYPE)
    d = rng.normal(size=(n_beams, 3))
    B["dir"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    B["range"] = rng.uniform(0.1, 9.0, n_beams).astype(np.float32)
    B["orig"] = rng.normal(0, 0.05, (n_beams, 3)).astype(np.float32)
    return P, A, B, synth.scenario_tsb()


@pytest.mark.parametrize("n,n_beams", [(1, 0), (0, 5), (1, 1), (31, 33), (127, 180), (128, 1000), (129, 32), (4096, 180), (65_537, 17), (1_000_000, 7)])
def test_update_equals_the_host_update(n, n_beams):
    import rmcl_b200
    name, h, trunc = "indoor:500000", 0.1, 1.0
    f = rmcl_b200.DistanceField(gpu_map(name), h, trunc)
    g, index, bricks = _host_field(name, h, trunc)
    up = rmcl_b200.PCDSensorUpdaterB200(gpu_map(name))
    up.setDistanceField(f)
    P, A, B, Tsb = _pf_case(max(n, 1), n_beams, n + n_beams)
    P, A = P[:n], A[:n]
    prm = rmcl_b200.PFParams.defaults(correspondence_type=1)              # ignored by the field update
    want = R.pf_update(g, index, bricks, P, A, Tsb, B, prm)
    if n == 0:
        import torch
        Pd, Ad = torch.zeros((0, 8), device="cuda"), torch.zeros((0, 9), device="cuda")
    else:
        Pd, Ad = _dev(P, A)
    up.update(Pd, Ad, Tsb, B, prm)
    assert _np_attrs(Ad).tobytes() == want.tobytes()
    if n > 2:
        # slices concatenate to the whole
        k = n // 3
        Ps, As = _dev(P, A)
        up.update(Ps[:k], As[:k], Tsb, B, prm)
        up.update(Ps[k:], As[k:], Tsb, B, prm)
        assert _np_attrs(As).tobytes() == want.tobytes()


def _c3_scene():
    import rmcl_b200
    from rmcl_b200 import synth
    gmap = gpu_map("building:1000000")
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gmap)
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(m); h.find(Tgt)
    beams = synth.pf_beams(h.modelView()["points"], 180)
    return gmap, Tsb, Tgt, beams


def test_c3_field_update_within_the_bound_of_the_closest_point_update():
    import rmcl_b200
    from rmcl_b200 import synth
    gmap, Tsb, _, beams = _c3_scene()
    h, trunc = 0.1, 6.0
    f = rmcl_b200.DistanceField(gmap, h, trunc)
    P, _ = synth.pf_particles(100_000)
    A = np.zeros(len(P), synth.PARTICLE_ATTR_DTYPE)
    cp = rmcl_b200.PFParams.defaults(correspondence_type=1)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    Pd, Ad = _dev(P, A)
    up.update(Pd, Ad, Tsb, beams, cp)
    want = _np_attrs(Ad)
    up.setDistanceField(f)
    Pd, Ad = _dev(P, A)
    up.update(Pd, Ad, Tsb, beams, cp)
    got = _np_attrs(Ad)
    assert np.array_equal(got["likelihood"]["n_meas"], want["likelihood"]["n_meas"])
    sq = float(np.float32(cp.dist_sigma) ** 2)
    denom = math.sqrt(2 * sq * math.pi)
    c = math.sqrt(3.0) / 2.0 * h
    per_beam = max(math.exp(-0.5) / (math.sqrt(sq) * denom) * (c + 1e-4), math.exp(-(trunc - 2 * c) ** 2 / (2 * sq)) / denom)
    diff = np.abs(got["likelihood"]["mean"].astype(np.float64) - want["likelihood"]["mean"].astype(np.float64))
    print(f"C3 |field - closest point| mean: max {diff.max():.3e}, median {np.median(diff):.3e}, bound {per_beam:.3e}")
    assert diff.max() <= per_beam + 2e-6


def test_handles_in_any_destruction_order():
    import rmcl_b200
    from rmcl_b200 import synth
    V, F = synth.cube(9)
    pts = np.array([[0, 0, 0], [9.5, 0, 0], [30, 0, 0]], np.float32)
    # field before map ... and map before field
    m = rmcl_b200.Map(V, F)
    f = rmcl_b200.DistanceField(m, 0.5, 2.0)
    want = f.query(pts)
    m.close()
    assert f.query(pts).tobytes() == want.tobytes()
    assert want[0] == np.float32(2.0) and abs(float(want[1]) - 0.5) < 1e-6 and want[2] == np.float32(2.0)
    f.close()
    # PF handle before field, field before PF handle
    m = rmcl_b200.Map(V, F)
    f = rmcl_b200.DistanceField(m, 0.5, 2.0)
    up = rmcl_b200.PCDSensorUpdaterB200(m)
    up.setDistanceField(f)
    del m
    P, A = synth.pf_particles(64, footprint=(8.0, 8.0), z=0.0)
    B = np.zeros(8, synth.RANGE_MEAS_DTYPE); B["dir"][:, 0] = 1.0; B["range"] = 1.0
    Pd, Ad = _dev(P, A)
    up.update(Pd, Ad, synth.scenario_tsb(), B)
    up.close()
    assert f.query(pts).tobytes() == want.tobytes()
    up2 = rmcl_b200.PCDSensorUpdaterB200(f.map)
    up2.setDistanceField(f)
    f_ref = f
    del f
    up2.update(Pd, Ad, synth.scenario_tsb(), B)                             # the updater keeps the field alive
    f_ref.close()
    with pytest.raises(Exception):
        up2.update(P, A, synth.scenario_tsb(), B)                           # host particles with a field: refused
    up2.setDistanceField(None)


def test_refusals_on_a_map():
    import rmcl_b200
    from rmcl_b200 import synth
    m = gpu_map("cube29")
    for args in [(0.0, 1.0), (0.1, float("nan")), (-1.0, 1.0), (0.1, 0.0)]:
        with pytest.raises(rmcl_b200.B2Error) as e:
            rmcl_b200.DistanceField(m, *args)
        assert e.value.code == -1
    for lo, hi in [((0, 0, 0), (0, 1, 1)), ((0, 0, np.nan), (1, 1, 1)), ((0, 0, 0), (1e9, 1, 1))]:
        with pytest.raises(rmcl_b200.B2Error):
            rmcl_b200.DistanceField(m, 0.1, 1.0, lo, hi)
    with pytest.raises(rmcl_b200.B2Error):
        rmcl_b200.DistanceField(m, 0.01, 1.0, (-1e4, -1e4, -1e4), (1e4, 1e4, 1e4))     # more than 2^32 - 2 bricks
    # the field then still builds and the explicit box is used as given
    f = rmcl_b200.DistanceField(m, 0.5, 1.0, (-12, -12, -12), (12, 12, 12))
    inf = f.info()
    assert inf["origin"] == (-12.0, -12.0, -12.0) and inf["dims"] == (49, 49, 49)


def _tracking(use_field, seed=77):
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    from test_pf_init import RVIZ_COV
    gmap, Tsb, Tgt, beams = _c3_scene()
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    if use_field:
        up.setDistanceField(rmcl_b200.DistanceField(gmap, 0.05, 1.0))
    n = 100_000
    Pd = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    Ad = torch.empty((n, 9), dtype=torch.float32, device="cuda")
    yaw_gt = 2.0 * np.arctan2(float(Tgt["R"][2]), float(Tgt["R"][3]))
    start = synth.make_transform(np.asarray(Tgt["t"], np.float64) + [0.3, 0.4, 0.0], (0.0, 0.0, yaw_gt + 0.2))
    up.initSamples(Pd, Ad, start, RVIZ_COV, seed)
    glad, prm = rmcl_b200.GladiatorConfig.defaults(), rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.2
    still = synth.make_transform()
    for step in range(10):
        up.motionUpdate(Pd, Ad, still, 0.01)
        up.update(Pd, Ad, Tsb, beams, prm)
        Pn, An = torch.empty_like(Pd), torch.empty_like(Ad)
        up.resample(Pd, Ad, Pn, An, glad, seed=seed, step=step)
        Pd, Ad = Pn, An
    rec = up.estimateStats(Pd, Ad)
    pos = np.asarray(rec["position"], np.float64)
    q = rec["orientation"]
    dyaw = abs((2.0 * np.arctan2(q[2], q[3]) - yaw_gt + np.pi) % (2 * np.pi) - np.pi)
    return pos, float(np.linalg.norm(pos[:2] - np.asarray(Tgt["t"][:2], np.float64))), float(dyaw)


def test_pf_cycle_with_the_field_converges_like_ray_casting():
    """init 0.5 m / 0.2 rad off the true pose of building:1000000, ten rounds of motion (standing still), sensor update and Gladiator
    resampling, then the estimate: with the field (h 0.05 m, trunc 1 m) and with ray casting, dist_sigma 0.2 m"""
    p_rc, e_rc, y_rc = _tracking(False)
    p_df, e_df, y_df = _tracking(True)
    print(f"ray casting: {e_rc:.3f} m, {y_rc:.3f} rad; field: {e_df:.3f} m, {y_df:.3f} rad; apart {np.linalg.norm(p_rc[:2] - p_df[:2]):.3f} m")
    assert e_rc < 0.3 and y_rc < 0.15 and e_df < 0.3 and y_df < 0.15
    assert np.linalg.norm(p_rc[:2] - p_df[:2]) < 0.3
