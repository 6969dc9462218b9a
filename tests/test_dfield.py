"""CPU tests of the truncated distance field (b2_dfield_*, b2_pf_sensor_update_field): the product's df_* functions compiled for the host
(tests/dfield_ref/dfield_emul.cu) against the oracle's closest point and float64 numpy restatements (tests/dfield_ref.py).

Tolerances.
  * node values, allocation, bounded query: exact (bit patterns).
  * lookup: the product interpolates in float32 (three lerps of values <= trunc, each op rounded), the restatement in float64 over the same
    stored nodes and the same cell and t: within 8 ulp of trunc.
  * accuracy contract: |field - min(d, trunc)| <= (sqrt(3)/2) h + 1e-5 (1 + max |coordinate|): node positions and distances carry float
    rounding of the coordinates' size.
  * update: float32 transform, evaluation and merge against float64: mean and sigma within 2e-6, n_meas exact."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import dfield_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C_HALF_SQRT3 = math.sqrt(3.0) / 2.0


def _meshes():
    from rmcl_b200 import synth
    return {"cube": synth.cube(5), "uvsphere": synth.uvsphere(12, 8), "indoor": synth.indoor(2000)}


MESHES = None


def _mesh(name):
    global MESHES
    if MESHES is None:
        MESHES = _meshes()
    return MESHES[name]


def _field(name, h, trunc, lo=None, hi=None):
    V, F = _mesh(name)
    if lo is None:
        lo, hi = R.default_box(V, trunc)
    g = R.Grid(lo, hi, h, trunc)
    assert g.refused is None, g.refused
    pf = R.ProductField(V, F)
    index, bricks = pf.build(g)
    return V, F, g, pf, index, bricks


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---------------------------------------------------------------- 1. node values ------------------------------------------------------
@pytest.mark.parametrize("name,h,trunc", [("cube", 0.5, 1.5), ("uvsphere", 0.4, 1.0), ("indoor", 0.25, 0.5)])
def test_node_values_equal_the_oracle_clamped(name, h, trunc):
    """every stored node equals orc_closest_point's distance clamped at trunc, through the oracle's BVH for all nodes and by brute force
    for a sample; the cube's grid puts nodes on its faces (origin -11.5, h 0.5) and at exactly trunc from them"""
    V, F, g, _, index, bricks = _field(name, h, trunc)
    ref = R.RefField(V, F)
    ids = np.flatnonzero(index.reshape(-1) != R.NOBRICK)
    assert len(ids) == len(bricks) and np.array_equal(index.reshape(-1)[ids], np.arange(len(ids)))     # slots in brick order
    P = R.node_points(g, ids).reshape(-1, 3)
    got = bricks.reshape(-1)
    assert np.array_equal(_bits(ref.values(P, g.trunc)), _bits(got))
    rng = np.random.default_rng(1)
    k = rng.choice(len(P), min(len(P), 4000), replace=False)
    assert np.array_equal(_bits(ref.values(P[k], g.trunc, brute=True)), _bits(got[k]))
    assert (got <= np.float32(trunc)).all() and (got >= 0).all()
    if name == "cube":
        assert (got == 0).any() and (got == np.float32(trunc)).any()
        exact = np.abs(np.abs(P).max(1) - 11.5) == 0                              # nodes exactly trunc off a face, outside the cube
        assert exact.any()


def test_far_nodes_and_an_explicit_box():
    """a box far larger than the map: far bricks are not allocated, every allocated node still equals the oracle"""
    V, F, g, _, index, bricks = _field("cube", 1.0, 2.0, lo=(-40, -40, -40), hi=(40, 40, 40))
    ref = R.RefField(V, F)
    ids = np.flatnonzero(index.reshape(-1) != R.NOBRICK)
    assert 0 < len(ids) < g.n_bricks
    assert np.array_equal(_bits(ref.values(R.node_points(g, ids).reshape(-1, 3), g.trunc)), _bits(bricks.reshape(-1)))
    un = np.flatnonzero(index.reshape(-1) == R.NOBRICK)
    assert (ref.values(R.node_points(g, un).reshape(-1, 3), g.trunc, brute=True) == np.float32(g.trunc)).all()


# ---------------------------------------------------------------- 2. allocation margin -----------------------------------------------
@pytest.mark.parametrize("name,h,trunc", [("cube", 0.5, 1.5), ("cube", 0.3, 0.7), ("uvsphere", 0.25, 0.6), ("indoor", 0.2, 0.3)])
def test_unallocated_bricks_hold_trunc(name, h, trunc):
    """every node of every unallocated brick has value exactly trunc, and the allocation is the rule: centre distance < trunc + 8h.  The
    box is the map's grown by trunc + 24h, so that there are bricks whose centres sit just outside that margin (within h of it); the 64
    unallocated bricks nearest the margin are checked by brute force, all of them through the oracle's BVH"""
    V, _ = _mesh(name)
    lo, hi = R.default_box(V, trunc + 24 * h)
    V, F, g, _, index, _ = _field(name, h, trunc, lo, hi)
    ref = R.RefField(V, F)
    flat = index.reshape(-1)
    un = np.flatnonzero(flat == R.NOBRICK)
    assert len(un) > 0
    assert (ref.values(R.node_points(g, un).reshape(-1, 3), g.trunc) == np.float32(g.trunc)).all()
    dc = ref.dist(R.brick_centres(g))
    ta = np.float32(g.trunc) + np.float32(8.0) * np.float32(g.h)
    assert np.array_equal(flat != R.NOBRICK, dc < ta)
    assert ((dc >= ta) & (dc < ta + np.float32(g.h))).any()
    nearest = un[np.argsort(dc[un])[:64]]
    assert (ref.values(R.node_points(g, nearest).reshape(-1, 3), g.trunc, brute=True) == np.float32(g.trunc)).all()


# ---------------------------------------------------------------- 3. bounded query ---------------------------------------------------
@pytest.mark.parametrize("name", ["cube", "uvsphere", "indoor"])
def test_bounded_query_equals_unbounded_below_trunc(name):
    V, F = _mesh(name)
    pf = R.ProductField(V, F)
    rng = np.random.default_rng(2)
    lo, hi = V.min(0) - 2.0, V.max(0) + 2.0
    pts = [rng.uniform(lo, hi, (20000, 3))]
    tri = V[F[rng.integers(0, len(F), 5000)]]
    w = rng.dirichlet((1, 1, 1), 5000)
    pts.append(np.einsum("nk,nkd->nd", w, tri))                                  # on the surface
    pts.append(tri[:, 0])                                                        # on vertices
    pts = np.concatenate(pts).astype(np.float32)
    for trunc in (0.05, 0.5, 1.5):
        d2u, fu = pf.closest(pts)
        d2b, fb = pf.closest(pts, bounded=True, trunc=trunc)
        t2 = np.float32(trunc) * np.float32(trunc)
        below = d2u < t2
        assert below.any() and (~below).any()
        assert np.array_equal(_bits(d2u[below]), _bits(d2b[below])) and np.array_equal(fu[below], fb[below])
        # at or beyond trunc both clamp to trunc
        cu = np.minimum(np.sqrt(d2u[~below]), np.float32(trunc))
        cb = np.minimum(np.sqrt(d2b[~below]), np.float32(trunc))
        assert (cu == np.float32(trunc)).all() and (cb == np.float32(trunc)).all()


# ---------------------------------------------------------------- 4. lookup ------------------------------------------------------------
def _lookup_points(g, rng):
    lo = g.lo.astype(np.float64)
    h = g.h
    dims = np.array(g.dims)
    top = lo + (dims - 1) * h
    n = 20000
    out = [rng.uniform(lo, top, (n, 3))]
    i = rng.integers(0, dims, (n, 3))
    nodes = (g.lo + i.astype(np.float32) * np.float32(h)).astype(np.float64)    # on nodes
    out.append(nodes)
    face = nodes.copy(); face[:, 0] = rng.uniform(lo[0], top[0], n); face[:, 1] = rng.uniform(lo[1], top[1], n)     # on cell faces (z = node)
    out.append(face)
    edge = nodes.copy(); edge[:, 0] = rng.uniform(lo[0], top[0], n)             # on cell edges along x
    out.append(edge)
    bnd = rng.uniform(lo, top, (n, 3)); k = rng.integers(0, 3, n); side = rng.integers(0, 2, n)
    bnd[np.arange(n), k] = np.where(side == 0, lo[k], top[k])                   # on the box boundary
    out.append(bnd)
    outside = rng.uniform(lo - 3.0, top + 3.0, (n, 3))
    out.append(outside)
    pts = np.concatenate(out).astype(np.float32)
    special = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.nan, np.nan, np.nan], [1e30, 0, 0], [-1e30, 1e30, 0]], np.float32)
    return np.concatenate([pts, special])


@pytest.mark.parametrize("name,h,trunc", [("cube", 0.5, 1.5), ("indoor", 0.25, 0.5)])
def test_lookup_matches_the_float64_restatement(name, h, trunc):
    _, _, g, _, index, bricks = _field(name, h, trunc)
    rng = np.random.default_rng(3)
    pts = _lookup_points(g, rng)
    got = R.lookup(g, index, bricks, pts)
    want = R.lookup64(g, index, bricks, pts)
    fin = np.isfinite(pts).all(1)
    assert np.isinf(got[~fin]).all() and (got[~fin] > 0).all()
    tol = 8 * float(np.spacing(np.float32(trunc)))
    assert np.abs(got[fin].astype(np.float64) - want[fin]).max() <= tol
    # finite points outside the box give exactly trunc
    G = (pts[fin] - g.lo) * np.float32(g.inv_h)
    outside = ~((G >= 0).all(1) & (G <= (np.array(g.dims) - 1).astype(np.float32)).all(1))
    assert outside.any() and (got[fin][outside] == np.float32(trunc)).all()
    # at a node the lookup returns the node (t = 0 on every axis)
    ids = np.flatnonzero(index.reshape(-1) != R.NOBRICK)[:50]
    P = R.node_points(g, ids)[:, :8, :8, :8].reshape(-1, 3)
    Gp = (P - g.lo) * np.float32(g.inv_h)
    exact = (Gp == np.round(Gp)).all(1)
    assert exact.any()
    assert np.array_equal(_bits(R.lookup(g, index, bricks, P[exact])), _bits(bricks[:50, :8, :8, :8].reshape(-1)[exact]))


# ---------------------------------------------------------------- 5. accuracy contract ------------------------------------------------
@pytest.mark.parametrize("name,h,trunc", [("cube", 0.5, 1.5), ("uvsphere", 0.4, 1.0)])
def test_accuracy_bound(name, h, trunc):
    V, F, g, _, index, bricks = _field(name, h, trunc)
    ref = R.RefField(V, F)
    rng = np.random.default_rng(4)
    dims = np.array(g.dims)
    pts = rng.uniform(g.lo, g.lo + (dims - 1) * g.h, (100_000, 3)).astype(np.float32)
    got = R.lookup(g, index, bricks, pts).astype(np.float64)
    d = ref.dist(pts, brute=True).astype(np.float64)
    eps = 1e-5 * (1.0 + float(np.abs(pts).max()))
    err = np.abs(got - np.minimum(d, trunc))
    assert err.max() <= C_HALF_SQRT3 * h + eps, err.max()


# ---------------------------------------------------------------- 6. the update ------------------------------------------------------
def _pf_case(n, n_beams, seed):
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    P = synth.transforms(n)
    P["t"] = rng.uniform((1.0, 1.0, 0.5), (11.0, 7.0, 2.0), (n, 3)).astype(np.float32)
    yaw = rng.uniform(-np.pi, np.pi, n)
    P["R"][:, 2], P["R"][:, 3] = np.sin(yaw / 2), np.cos(yaw / 2)
    A = np.zeros(n, synth.PARTICLE_ATTR_DTYPE)
    A["likelihood"]["mean"] = rng.uniform(0, 0.2, n).astype(np.float32)
    A["likelihood"]["sigma"] = rng.uniform(0, 0.01, n).astype(np.float32)
    A["likelihood"]["n_meas"] = rng.choice([0, 5, 9990, 10000], n)
    B = np.zeros(n_beams, synth.RANGE_MEAS_DTYPE)
    d = rng.normal(size=(n_beams, 3))
    d[:, 2] *= 0.3
    B["dir"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    B["range"] = rng.uniform(0.2, 8.0, n_beams).astype(np.float32)
    B["orig"] = rng.normal(0, 0.05, (n_beams, 3)).astype(np.float32)
    if n_beams > 3:
        B["range"][0] = np.nan
        B["range"][1] = np.inf
    return P, A, B, synth.scenario_tsb()


def test_update_matches_numpy_and_the_closest_point_update():
    import rmcl_b200
    from oracle import pyoracle as po
    h, trunc = 0.1, 6.0
    V, F, g, _, index, bricks = _field("indoor", h, trunc)
    P, A, B, Tsb = _pf_case(300, 60, 5)
    prm = rmcl_b200.PFParams.defaults()
    got = R.pf_update(g, index, bricks, P, A, Tsb, B, prm)
    q = R.beam_points64(P, Tsb, B)
    e = R.lookup64(g, index, bricks, q.reshape(-1, 3).astype(np.float32)).reshape(q.shape[:2])
    ev = R.evaluate64(e, prm.dist_sigma)
    mean, sig, nm = R.merge64(A, ev)
    assert np.array_equal(got["likelihood"]["n_meas"], nm)
    assert np.abs(got["likelihood"]["mean"] - mean).max() <= 2e-6
    assert np.abs(got["likelihood"]["sigma"] - sig).max() <= 2e-6
    # against the closest-point update on fresh attributes (the mean is then the plain average of the evaluations): within the per-beam
    # bound exp(-1/2) / (sigma denom) (sqrt(3)/2) h where the distance is below trunc - (sqrt(3)/2) h, otherwise both evaluations are
    # at most the Gaussian at trunc - sqrt(3) h
    A0 = np.zeros_like(A)
    osc = po.Scene(V, F)
    cpc = osc.pf_update(P, A0, Tsb, B, po.PFParams.defaults(ng_mode=0, correspondence_type=1))
    fld = R.pf_update(g, index, bricks, P, A0, Tsb, B, prm)
    assert np.array_equal(cpc["likelihood"]["n_meas"], fld["likelihood"]["n_meas"])
    d = R.RefField(V, F).dist(q.reshape(-1, 3).astype(np.float32)).reshape(q.shape[:2]).astype(np.float64)
    sq = float(np.float32(prm.dist_sigma) ** 2)
    denom = math.sqrt(2 * sq * math.pi)
    c = C_HALF_SQRT3 * h
    near = math.exp(-0.5) / (math.sqrt(sq) * denom) * (c + 1e-4)
    far = math.exp(-max(0.0, trunc - 2 * c) ** 2 / (2 * sq)) / denom
    per_beam = np.where(d < trunc - c, near, far)
    per_beam[~np.isfinite(q).all(2)] = 0.0                                      # NaN / inf end points: both evaluate to 0
    bound = per_beam.mean(1) + 2e-6
    diff = np.abs(fld["likelihood"]["mean"].astype(np.float64) - cpc["likelihood"]["mean"].astype(np.float64))
    assert (diff <= bound).all(), (diff - bound).max()


def test_update_edge_counts():
    """zero beams leave the attributes as they are; one beam; the MAX_N_MEAS clamp"""
    import rmcl_b200
    _, _, g, _, index, bricks = _field("indoor", 0.25, 1.0)
    prm = rmcl_b200.PFParams.defaults()
    P, A, B, Tsb = _pf_case(50, 5, 6)
    assert R.pf_update(g, index, bricks, P, A, Tsb, B[:0], prm).tobytes() == A.tobytes()
    got = R.pf_update(g, index, bricks, P, A, Tsb, B[2:3], prm)
    assert np.array_equal(got["likelihood"]["n_meas"], np.minimum(A["likelihood"]["n_meas"].astype(np.int64) + 1, 10000))


# ---------------------------------------------------------------- 7. refusals ---------------------------------------------------------
@pytest.mark.parametrize("lo,hi,h,trunc", [
    ((0, 0, 0), (1, 1, 1), 0.0, 1.0), ((0, 0, 0), (1, 1, 1), -0.1, 1.0), ((0, 0, 0), (1, 1, 1), float("nan"), 1.0), ((0, 0, 0), (1, 1, 1), float("inf"), 1.0),
    ((0, 0, 0), (1, 1, 1), 0.1, 0.0), ((0, 0, 0), (1, 1, 1), 0.1, float("nan")), ((0, 0, 0), (1, 1, 1), 0.1, float("inf")), ((0, 0, 0), (1, 1, 1), 0.1, -1.0),
    ((0, 0, 0), (0, 1, 1), 0.1, 1.0), ((0, 2, 0), (1, 1, 1), 0.1, 1.0), ((0, 0, float("nan")), (1, 1, 1), 0.1, 1.0), ((0, 0, 0), (1, float("inf"), 1), 0.1, 1.0),
    ((0, 0, 0), (2 ** 24, 1, 1), 1.0, 1.0), ((0, 0, 0), (1.1e6, 1, 1), 1.0 / 16.0, 1.0), ((0, 0, 0), (20000, 20000, 20000), 0.5, 1.0)])
def test_grid_refusals(lo, hi, h, trunc):
    """the grid's refusals (b2_dfield_create returns B2_ERR_INVALID for each before anything is allocated): h, trunc, bounds, more than
    2^24 nodes on an axis (counting the last brick's far face), more than 2^32 - 2 bricks"""
    g = R.Grid(np.array(lo, np.float32), np.array(hi, np.float32), h, trunc)
    assert g.refused, (lo, hi, h, trunc)


def test_grid_limits_accepted():
    g = R.Grid(np.zeros(3, np.float32), np.array([8 * (2 ** 21 - 1), 1, 1], np.float32), 1.0, 1.0)       # 2^24 - 7 nodes: fits
    assert g.refused is None and g.dims[0] == 8 * (2 ** 21 - 1) + 1 and g.bdims == (2 ** 21 - 1, 1, 1)
    g = R.Grid(np.zeros(3, np.float32), np.array([0.1, 0.1, 0.1], np.float32), 1.0, 1.0)                  # smaller than one cell
    assert g.refused is None and g.dims == (2, 2, 2) and g.bdims == (1, 1, 1)


def test_abi_null_arguments_are_refused():
    """null arguments are refused with B2_ERR_INVALID before a device is touched; a compute entry point never runs without a device"""
    import rmcl_b200
    lib = rmcl_b200.load_library()
    prm = rmcl_b200.api._DfieldParams(0.1, 1.0, None, None)
    out = C.c_void_p(1234)
    assert lib.b2_dfield_create(None, C.byref(prm), C.byref(out)) == -1 and out.value is None
    assert lib.b2_dfield_create(C.c_void_p(8), None, C.byref(out)) == -1
    assert lib.b2_dfield_create(C.c_void_p(8), C.byref(prm), None) == -1
    dist = np.full(4, 7.0, np.float32)
    assert lib.b2_dfield_query(None, None, C.c_uint32(4), C.c_void_p(dist.ctypes.data), C.c_int(0)) == -1 and (dist == 7.0).all()
    assert lib.b2_dfield_get_info(None, None) == -1
    assert lib.b2_dfield_download(None, None, None) == -1
    assert lib.b2_pf_sensor_update_field(None, None, None, None, C.c_uint32(0), None, None, C.c_uint32(0), None) == -1
    assert lib.b2_dfield_destroy(None) == 0
    # one of the two bounds only
    lo = np.zeros(3, np.float32)
    half = rmcl_b200.api._DfieldParams(0.1, 1.0, lo.ctypes.data, None)
    assert lib.b2_dfield_create(C.c_void_p(8), C.byref(half), C.byref(out)) == -1
    bad = rmcl_b200.api._DfieldParams(float("nan"), 1.0, None, None)
    assert lib.b2_dfield_create(C.c_void_p(8), C.byref(bad), C.byref(out)) == -1
    assert sorted(set(rmcl_b200.api.EXPORTS)) == sorted(rmcl_b200.api.EXPORTS)
    assert C.sizeof(rmcl_b200.api._DfieldParams) == 24 and C.sizeof(rmcl_b200.api._DfieldInfo) == 80


def test_no_device_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import rmcl_b200
    from rmcl_b200 import synth
    V, F = synth.cube(3)
    with pytest.raises(rmcl_b200.B2Error):
        rmcl_b200.DistanceField(rmcl_b200.Map(V, F), 0.1, 1.0)


def test_updater_refuses_numpy_with_a_field():
    """with a field set, update() on numpy arrays raises B2Error before anything is launched or sampled (no device needed)"""
    import rmcl_b200
    from rmcl_b200 import synth
    up = rmcl_b200.PCDSensorUpdaterB200.__new__(rmcl_b200.PCDSensorUpdaterB200)
    up._h, up._input, up.config, up.step = None, object(), rmcl_b200.PFParams.defaults(), 3
    up._field = rmcl_b200.DistanceField.__new__(rmcl_b200.DistanceField)
    P, A = synth.pf_particles(4)
    with pytest.raises(rmcl_b200.B2Error):
        up.update(P, A, synth.scenario_tsb())
    assert up.step == 3
    up._field._h = None
    with pytest.raises(TypeError):
        up.setDistanceField(object())


def test_cpp_field_api_compiles(tmp_path):
    """the C++ mirror (B200DistanceField, PCDSensorUpdaterB200::setDistanceField) compiles standalone"""
    import subprocess
    src = tmp_path / "df.cpp"
    src.write_text('#include "rmcl_b200/rcc_b200.hpp"\n'
                   "int main() {\n"
                   "  auto map = std::make_shared<rmcl::B200Map>(\"none.ply\");\n"
                   "  auto f = std::make_shared<rmcl::B200DistanceField>(map, 0.1f, 1.0f);\n"
                   "  rmcl::PCDSensorUpdaterB200 up(map);\n"
                   "  up.setDistanceField(f);\n"
                   "  float d; float p[3] = {0, 0, 0}; f->query(p, 1, &d);\n"
                   "  b2_dfield_info i = f->info(); (void)i;\n"
                   "  up.setDistanceField(nullptr);\n"
                   "  return 0; }\n")
    subprocess.check_call(["g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)])
