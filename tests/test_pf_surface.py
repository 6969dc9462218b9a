"""The surface constraint (b2_pf_project_to_surface, PCDSensorUpdaterB200.projectToSurface) on the CPU.

* The product's pf_surface_one, compiled for the host over its host-built BVH, is byte-identical in poses and attributes to the C
  restatement of the rule (tests/pf_surface_ref/), whose answers are the same by brute force as through the oracle's BVH.
* Float64 checks of the geometry, independent of the restatement: on a tilted plane the result lies on the plane within the float bound
  below, its z-axis is the plane's normal and its heading change is the minimal rotation; no particle on a lattice edge or vertex is lost;
  projecting twice moves nothing beyond the bound."""
import math

import numpy as np
import pytest

from pf_surface_ref import ProductScene, RefScene, quat_mul64, quat_rotate64
from rmcl_b200 import synth
from rmcl_b200.api import SurfaceConfig
from rmcl_b200.synth import PARTICLE_ATTR_DTYPE, TRANSFORM_DTYPE

TERRAIN_TRIS = 20000
# the tilted plane z = PLANE_A x + PLANE_B y over [-8, 8]^2, 32 x 32 quads (dyadic vertices): slope atan(|(A, B)|) = 15.6 deg
PLANE_A, PLANE_B, PLANE_HALF = 0.25, 0.125, 8.0
PLANE_SLOPE = math.atan(math.hypot(PLANE_A, PLANE_B))
# Bound on the distance of t' from the plane (float64, m).  g.z = (t.z + probe_above) - t_hit is two roundings of values <= S = 16 m
# (<= 1 ulp(S)); t_hit = T / det from the Moeller-Trumbore chains, whose terms are <= S |e|^2 over det ~ |e|^2: <= 8 ulp(S); the offset
# base_height * n adds <= 2 ulp(S).  16 ulp(16 m) = 16 * 2^-19 = 3.1e-5 m.
PLANE_BOUND = 16 * 2.0 ** -19


def _plane():
    V, F = synth._grid_rect([-PLANE_HALF, -PLANE_HALF, 0.0], [2 * PLANE_HALF, 0, 0], [0, 2 * PLANE_HALF, 0], 32, 32)
    V[:, 2] = PLANE_A * V[:, 0] + PLANE_B * V[:, 1]
    return V.astype(np.float32), F.astype(np.uint32)


def _plane_normal():
    n = np.array([-PLANE_A, -PLANE_B, 1.0])
    return n / np.linalg.norm(n)


_SCENES = {}


def _scenes(name):
    if name not in _SCENES:
        V, F = synth.terrain(TERRAIN_TRIS) if name == "terrain" else _plane()
        _SCENES[name] = (ProductScene(V, F), RefScene(V, F))
    return _SCENES[name]


def _particles(xyz, rpy=None, seed=0):
    """poses at xyz (n, 3) with Euler angles rpy (n, 3, default 0) and random attributes, stamps and likelihoods (n_meas < 10000)"""
    rng = np.random.default_rng(seed)
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    n = len(xyz)
    P = np.zeros(n, TRANSFORM_DTYPE)
    P["t"] = xyz.astype(np.float32)
    rpy = np.zeros((n, 3)) if rpy is None else np.asarray(rpy, np.float64).reshape(n, 3)
    P["R"] = np.array([synth.quat_from_rpy(*r) for r in rpy], np.float32)
    P["stamp"] = rng.integers(1, 2**32, n, dtype=np.uint64).astype(np.uint32)
    A = np.zeros(n, PARTICLE_ATTR_DTYPE)
    A["likelihood"]["mean"] = rng.uniform(0.1, 1.0, n)
    A["likelihood"]["sigma"] = rng.uniform(0.0, 0.1, n)
    A["likelihood"]["n_meas"] = rng.integers(0, 5000, n)
    A["state_sigma"] = rng.uniform(0.0, 1.0, (n, 6))
    return P, A


def _cfg(probe_above=0.5, probe_below=1.0, base_height=0.0, max_slope=0.6, align=1):
    return SurfaceConfig(probe_above, probe_below, base_height, max_slope, align)


def _marked(A):
    return (A["likelihood"]["n_meas"] == 10000) & (A["likelihood"]["mean"] == 0.0) & (A["likelihood"]["sigma"] == 0.0)


def _terrain_height(x, y):
    """the walkable height at (x, y) seen from just above the lattice parts (floor, ramp, mezzanine top, stairs) -- NaN elsewhere"""
    r, m, st = synth.TERRAIN_RAMP, synth.TERRAIN_MEZZANINE, synth.TERRAIN_STAIRS
    z = np.zeros_like(x, dtype=np.float64)
    on_ramp = (x >= r["x0"]) & (x <= r["x0"] + r["run"]) & (y >= r["y0"]) & (y <= r["y1"])
    z[on_ramp] = (x[on_ramp] - r["x0"]) * r["rise"] / r["run"]
    on_mez = (x >= m["x0"]) & (x <= m["x1"]) & (y >= m["y0"]) & (y <= m["y1"])
    z[on_mez] = m["top"]
    on_st = (x >= st["x0"]) & (x < st["x0"] + st["steps"] * st["tread"]) & (y >= st["y0"]) & (y <= st["y1"])
    z[on_st] = (np.floor((x[on_st] - st["x0"]) / st["tread"]) + 1) * st["riser"]
    return z


def _random_cases(seed):
    """particles above, below and beside the terrain with any orientation"""
    rng = np.random.default_rng(seed)
    n = 3000
    xyz = np.stack([rng.uniform(-2, 66, n), rng.uniform(-2, 34, n), rng.uniform(-1.0, 4.5, n)], 1)
    rpy = np.stack([rng.uniform(-math.pi, math.pi, n), rng.uniform(-1.5, 1.5, n), rng.uniform(-math.pi, math.pi, n)], 1)
    return _particles(xyz, rpy, seed)


def _lattice_cases(seed):
    """particles exactly on lattice vertices and edges (cell 1 m at this size: the diagonal of every cell runs from (i, j) to (i+1, j+1)),
    a little above the walkable height, with small tilts"""
    rng = np.random.default_rng(seed)
    n = 1500
    i, j = rng.integers(0, 48, n).astype(np.float64), rng.integers(0, 32, n).astype(np.float64)
    f = rng.integers(0, 64, n) / 64.0
    kind = rng.integers(0, 4, n)
    x = np.where(kind == 0, i, np.where(kind == 1, i + f, np.where(kind == 2, i, i + f)))
    y = np.where(kind == 0, j, np.where(kind == 1, j, np.where(kind == 2, j + f, j + f)))
    z = _terrain_height(x, y) + rng.integers(0, 8, n) / 32.0
    rpy = np.stack([rng.normal(0, 0.05, n), rng.normal(0, 0.05, n), rng.uniform(-math.pi, math.pi, n)], 1)
    return _particles(np.stack([x, y, z], 1), rpy, seed)


def _mezzanine_cases(seed):
    rng = np.random.default_rng(seed)
    m = synth.TERRAIN_MEZZANINE
    n = 800
    xyz = np.stack([rng.uniform(m["x0"] + 0.1, m["x1"] - 0.1, n), rng.uniform(m["y0"] + 0.1, m["y1"] - 0.1, n), rng.uniform(0.0, 0.3, n)], 1)
    return _particles(xyz, np.stack([np.zeros(n), np.zeros(n), rng.uniform(-3, 3, n)], 1), seed)


def _stairs_cases(seed):
    """on and between the steps, with x exactly on the risers for a third of them"""
    rng = np.random.default_rng(seed)
    st = synth.TERRAIN_STAIRS
    n = 1200
    k = rng.integers(0, st["steps"], n)
    x = st["x0"] + k * st["tread"] + np.where(rng.integers(0, 3, n) == 0, 0.0, rng.uniform(0, st["tread"], n))
    y = rng.uniform(st["y0"], st["y1"], n)
    z = (k + 1) * st["riser"] + rng.uniform(-0.1, 0.3, n)
    return _particles(np.stack([x, y, z], 1), np.stack([np.zeros(n), np.zeros(n), rng.uniform(-3, 3, n)], 1), seed)


def _special_cases():
    """upside-down particles (1 + c exactly 0 and just around it) and non-finite poses"""
    xyz, rpy = [], []
    for x, y in ((10.0, 10.0), (30.0, 8.0), (12.5, 2.0), (56.3, 7.1)):
        for roll in (math.pi, math.pi - 1e-4, math.pi - 3e-3, -math.pi + 1e-7):
            xyz.append((x, y, 0.2 + _terrain_height(np.array([x]), np.array([y]))[0]))
            rpy.append((roll, 0.0, 0.7))
    P, A = _particles(xyz, rpy, 3)
    nan, inf = np.float32("nan"), np.float32("inf")
    bad = np.repeat(P[:1], 6)
    bad["t"][0, 0] = nan
    bad["t"][1, 2] = nan
    bad["t"][2, 1] = inf
    bad["t"][3, 2] = -inf
    bad["R"][4] = nan
    bad["t"][5] = nan
    return np.concatenate([P, bad]), np.concatenate([A, np.repeat(A[:1], 6)])


CONFIGS = [_cfg(align=1), _cfg(align=0), _cfg(base_height=0.3, align=1), _cfg(base_height=0.3, align=0)]
CFG_IDS = ["align1", "align0", "align1_h0.3", "align0_h0.3"]


def _agree(scene, P, A, cfg, brute_too=False):
    prod, ref = _scenes(scene)
    Pp, Ap = prod.project(P, A, cfg)
    Pr, Ar = ref.project(P, A, cfg)
    assert Pp.tobytes() == Pr.tobytes()
    assert Ap.tobytes() == Ar.tobytes()
    if brute_too:
        Pb, Ab = ref.project(P, A, cfg, brute=1)
        assert Pb.tobytes() == Pr.tobytes() and Ab.tobytes() == Ar.tobytes()
    return Pp, Ap


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
@pytest.mark.parametrize("case", ["random", "lattice", "stairs", "special"])
def test_product_matches_restatement_on_terrain(case, cfg):
    P, A = {"random": lambda: _random_cases(1), "lattice": lambda: _lattice_cases(2), "stairs": lambda: _stairs_cases(4),
            "special": _special_cases}[case]()
    Pp, Ap = _agree("terrain", P, A, cfg, brute_too=True)
    # the stamp and everything but the likelihood of a marked particle stay; a marked particle keeps its pose
    assert np.array_equal(Pp["stamp"], P["stamp"])
    assert Ap["state_sigma"].tobytes() == A["state_sigma"].tobytes()
    m = _marked(Ap)
    assert Pp[m].tobytes() == P[m].tobytes()
    assert Ap[~m].tobytes() == A[~m].tobytes()


def test_special_cases_outcomes():
    """upside-down particles land upright (roll pi: the half-turn branch); non-finite poses, a NaN orientation included, are marked and keep
    their pose"""
    P, A = _special_cases()
    for cfg in (_cfg(), _cfg(align=0)):
        Pp, Ap = _agree("terrain", P, A, cfg)
        assert not _marked(Ap[:16]).any() and _marked(Ap[16:]).all()
        assert Pp[16:].tobytes() == P[16:].tobytes()
    up = quat_rotate64(Pp["R"][:16], np.array([0.0, 0.0, 1.0]))
    assert (up[:, 2] < -0.99).all()                                            # align 0 (the last run) keeps them upside down
    Pp, _ = _agree("terrain", P, A, _cfg())
    up = quat_rotate64(Pp["R"][:16], np.array([0.0, 0.0, 1.0]))
    assert (up[:, 2] > 0.95).all()                                             # on ground normals of at most 17.4 deg (the bumps)


@pytest.mark.parametrize("probe_above", [0.5, 3.5])
def test_under_the_mezzanine(probe_above):
    """a probe that starts below the slab's underside (2.75 m) finds the floor; one that starts above its top lands on it (a stated limit)"""
    P, A = _mezzanine_cases(5)
    for cfg in (_cfg(probe_above=probe_above, probe_below=1.0, align=1), _cfg(probe_above=probe_above, probe_below=1.0, base_height=0.3, align=0)):
        Pp, Ap = _agree("terrain", P, A, cfg, brute_too=True)
        assert not _marked(Ap).any()
        want = 0.0 if probe_above < synth.TERRAIN_MEZZANINE["bottom"] else synth.TERRAIN_MEZZANINE["top"]
        assert np.abs(Pp["t"][:, 2] - (want + cfg.base_height)).max() <= 1e-6


def test_stair_risers_are_never_ground():
    """particles on the risers' x land on a tread (the riser's face is parallel to the ray); with max_slope pi/2 the vertical risers still
    cannot be hit by a vertical ray, so the outcome does not change"""
    P, A = _stairs_cases(6)
    st = synth.TERRAIN_STAIRS
    Pp, Ap = _agree("terrain", P, A, _cfg(probe_above=0.5, probe_below=1.0, align=1))
    Pq, Aq = _agree("terrain", P, A, _cfg(probe_above=0.5, probe_below=1.0, align=1, max_slope=float(np.float32(math.pi / 2))))
    assert Pp.tobytes() == Pq.tobytes() and Ap.tobytes() == Aq.tobytes()
    ok = ~_marked(Ap)
    z = Pp["t"][ok, 2].astype(np.float64)
    assert np.all(np.isclose(z / st["riser"], np.round(z / st["riser"]), atol=1e-6))       # every landing is on a tread (or the floor)
    n = quat_rotate64(Pp["R"][ok], np.array([0.0, 0.0, 1.0]))
    assert np.abs(n[:, 2] - 1.0).max() <= 1e-6


@pytest.mark.parametrize("scene,slope", [("plane", PLANE_SLOPE), ("terrain", math.atan2(3.0, 17.0))])
def test_slopes_just_under_and_over_max_slope(scene, slope):
    rng = np.random.default_rng(7)
    n = 500
    if scene == "plane":
        x, y = rng.uniform(-7, 7, n), rng.uniform(-7, 7, n)
        z = PLANE_A * x + PLANE_B * y + 0.2
    else:
        r = synth.TERRAIN_RAMP
        x, y = rng.uniform(r["x0"] + 0.5, r["x0"] + r["run"] - 0.5, n), rng.uniform(r["y0"] + 0.1, r["y1"] - 0.1, n)
        z = (x - r["x0"]) * r["rise"] / r["run"] + 0.2
    P, A = _particles(np.stack([x, y, z], 1), seed=8)
    for ms, lost in ((slope + 1e-4, False), (slope - 1e-4, True)):
        Pp, Ap = _agree(scene, P, A, _cfg(max_slope=ms), brute_too=True)
        assert (_marked(Ap) == lost).all()


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_product_matches_restatement_on_plane(cfg):
    rng = np.random.default_rng(9)
    n = 2000
    xyz = np.stack([rng.uniform(-9, 9, n), rng.uniform(-9, 9, n), rng.uniform(-4, 4, n)], 1)
    rpy = np.stack([rng.uniform(-math.pi, math.pi, n), rng.uniform(-1.5, 1.5, n), rng.uniform(-math.pi, math.pi, n)], 1)
    P, A = _particles(xyz, rpy, 9)
    _agree("plane", P, A, cfg, brute_too=True)


def _on_plane(seed, n=2000, tilt=0.3):
    rng = np.random.default_rng(seed)
    x, y = rng.uniform(-7.5, 7.5, n), rng.uniform(-7.5, 7.5, n)
    z = PLANE_A * x + PLANE_B * y + rng.uniform(-0.4, 0.45, n)
    rpy = np.stack([rng.normal(0, tilt, n), rng.normal(0, tilt, n), rng.uniform(-math.pi, math.pi, n)], 1)
    return _particles(np.stack([x, y, z], 1), rpy, seed)


@pytest.mark.parametrize("base_height", [0.0, 0.3])
def test_plane_geometry_float64(base_height):
    """t' on the plane within PLANE_BOUND (plus base_height along n); R' e_z = n within 1e-6 rad; R' = R_min R with R_min scipy's
    minimal rotation taking R e_z onto n (heading changed as little as possible)"""
    from scipy.spatial.transform import Rotation
    P, A = _on_plane(10)
    Pp, Ap = _scenes("plane")[0].project(P, A, _cfg(base_height=base_height, align=1))
    assert not _marked(Ap).any()
    n = _plane_normal()
    t = Pp["t"].astype(np.float64)
    dist = (t - base_height * n) @ n - 0.0                                       # the plane passes through the origin
    assert np.abs(dist).max() <= PLANE_BOUND
    up = quat_rotate64(Pp["R"], np.array([0.0, 0.0, 1.0]))
    ang = np.arctan2(np.linalg.norm(np.cross(up, n), axis=1), up @ n)
    assert ang.max() <= 1e-6
    a = quat_rotate64(P["R"], np.array([0.0, 0.0, 1.0]))
    axis = np.cross(a, n)
    angle = np.arctan2(np.linalg.norm(axis, axis=1), a @ n)
    rmin = Rotation.from_rotvec(axis / np.linalg.norm(axis, axis=1, keepdims=True) * angle[:, None])
    want = (rmin * Rotation.from_quat(P["R"].astype(np.float64))).as_quat()
    got = Pp["R"].astype(np.float64)
    err = np.minimum(np.abs(got - want).max(1), np.abs(got + want).max(1))
    assert err.max() <= 2e-6
    # align 0 keeps R bit for bit and moves t straight down onto the plane
    Pq, _ = _scenes("plane")[0].project(P, A, _cfg(base_height=base_height, align=0))
    assert Pq["R"].tobytes() == P["R"].tobytes()
    assert Pq["t"][:, :2].tobytes() == P["t"][:, :2].tobytes()
    zq = Pq["t"][:, 2].astype(np.float64) - base_height
    assert np.abs(zq - (PLANE_A * Pq["t"][:, 0].astype(np.float64) + PLANE_B * Pq["t"][:, 1].astype(np.float64))).max() <= PLANE_BOUND


def _on_upper_rim(x, y):
    """on the +x or +y border of the ramp, the mezzanine top or the stairs, with nothing else within the probe under it.  A vertical ray
    exactly in the plane of a triangle box's upper face fails the tracer's box validation (its slab interval on that axis ends at 0), so
    there only the neighbour on the upper side can be hit, and a rim has none (SURVEY F6)."""
    r, m, st = synth.TERRAIN_RAMP, synth.TERRAIN_MEZZANINE, synth.TERRAIN_STAIRS
    ramp = (x >= r["x0"]) & (x <= r["x0"] + r["run"]) & (y == r["y1"])
    mez = (x >= m["x0"]) & (x <= m["x1"]) & (y >= m["y0"]) & (y <= m["y1"]) & ((x == m["x1"]) | (y == m["y1"]))
    stairs = (x >= st["x0"]) & (x <= st["x0"] + st["steps"] * st["tread"]) & (y == st["y1"])
    return ramp | mez | stairs


def test_lattice_edges_and_vertices_are_not_lost():
    """on the dyadic lattice of the terrain every particle exactly on an inner edge or vertex finds its surface, at its exact height;
    exactly on a surface's upper rim it is off surface unless the surface below is within the probe"""
    P, A = _lattice_cases(11)
    rim = _on_upper_rim(P["t"][:, 0].astype(np.float64), P["t"][:, 1].astype(np.float64))
    assert 0 < rim.sum() < len(P) // 10
    P, A = P[~rim], A[~rim]
    for cfg in (_cfg(align=1), _cfg(align=0, base_height=0.25)):
        Pp, Ap = _scenes("terrain")[0].project(P, A, cfg)
        assert not _marked(Ap).any()
        x, y = P["t"][:, 0].astype(np.float64), P["t"][:, 1].astype(np.float64)
        want = _terrain_height(x, y) + cfg.base_height                          # flat parts: n = e_z
        off_ramp = ~((x > synth.TERRAIN_RAMP["x0"]) & (x < synth.TERRAIN_RAMP["x0"] + synth.TERRAIN_RAMP["run"]) & (y <= synth.TERRAIN_RAMP["y1"]))
        assert np.abs(Pp["t"][off_ramp, 2] - want[off_ramp]).max() == 0.0


@pytest.mark.parametrize("align,base_height", [(1, 0.0), (0, 0.0), (0, 0.3)])
def test_projecting_twice_moves_nothing_beyond_the_bound(align, base_height):
    """idempotent within PLANE_BOUND where the rule is (with align 1 and base_height > 0 a second call slides the particle along the slope
    by base_height n.xy: that case is left out)"""
    P, A = _on_plane(12)
    prod = _scenes("plane")[0]
    cfg = _cfg(align=align, base_height=base_height)
    P1, A1 = prod.project(P, A, cfg)
    P2, A2 = prod.project(P1, A1, cfg)
    assert A2.tobytes() == A1.tobytes()
    assert np.abs(P2["t"].astype(np.float64) - P1["t"]).max() <= PLANE_BOUND
    err = np.minimum(np.abs(P2["R"].astype(np.float64) - P1["R"]).max(1), np.abs(P2["R"].astype(np.float64) + P1["R"]).max(1))
    assert err.max() <= 1e-6


def test_synth_terrain_layout():
    V, F = synth.terrain(TERRAIN_TRIS)
    assert 0.98 * TERRAIN_TRIS <= len(F) <= TERRAIN_TRIS
    b = synth.TERRAIN_BUMPS
    bump = (V[:, 0] >= b["x0"]) & (V[:, 1] <= b["y0"] + b["size"])
    lat = V[~bump].astype(np.float64) * 2.0 ** 10
    assert np.array_equal(lat, np.round(lat))                                     # dyadic
    assert np.abs(V[bump, 2] - synth.terrain_bump_z(V[bump, 0], V[bump, 1])).max() <= 1e-6
    assert math.degrees(math.atan2(synth.TERRAIN_RAMP["rise"], synth.TERRAIN_RAMP["run"])) == pytest.approx(10.0, abs=0.01)


def test_quat_helpers():
    q = np.array(synth.quat_from_rpy(0.3, -0.2, 1.1), np.float64)
    p = np.array(synth.quat_from_rpy(-0.1, 0.4, 0.2), np.float64)
    v = np.array([0.3, -1.0, 2.0])
    assert np.allclose(quat_rotate64(quat_mul64(q, p), v), quat_rotate64(q, quat_rotate64(p, v)))
