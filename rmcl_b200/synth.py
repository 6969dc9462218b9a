"""Deterministic synthetic inputs for the ray-casting-correspondence path (SURVEY.md section 8d).

Meshes (float32 vertices, uint32 faces, CCW seen from the side a sensor can stand on), sensor models,
pose/particle generators.  Pure numpy; used by tests, bench.py and __graft_entry__.smoke().
No geometry queries happen here -- scans are produced by whichever tracer the caller uses.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

# --------------------------------------------------------------------------------------------------
# mesh helpers
# --------------------------------------------------------------------------------------------------


def _grid_rect(origin, eu, ev, nu, nv):
    """Rectangle origin + s*eu + t*ev, s,t in [0,1], split into nu x nv quads x 2 triangles.
    Winding is CCW when looking against eu x ev (normal = eu x ev)."""
    origin = np.asarray(origin, np.float64)
    eu = np.asarray(eu, np.float64)
    ev = np.asarray(ev, np.float64)
    s = np.linspace(0.0, 1.0, nu + 1)
    t = np.linspace(0.0, 1.0, nv + 1)
    S, T = np.meshgrid(s, t, indexing="xy")            # (nv+1, nu+1)
    V = origin[None, None, :] + S[..., None] * eu[None, None, :] + T[..., None] * ev[None, None, :]
    V = V.reshape(-1, 3)
    j, i = np.meshgrid(np.arange(nv), np.arange(nu), indexing="ij")
    a = (j * (nu + 1) + i).ravel()
    b = a + 1
    c = a + (nu + 1)
    d = c + 1
    F = np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, c], 1)], 0)
    # interleave so the two triangles of a quad are adjacent
    F = F.reshape(2, -1, 3).transpose(1, 0, 2).reshape(-1, 3)
    return V, F


def _merge(parts):
    vs, fs, off = [], [], 0
    for V, F in parts:
        vs.append(V)
        fs.append(F + off)
        off += V.shape[0]
    return np.concatenate(vs, 0).astype(np.float32), np.concatenate(fs, 0).astype(np.uint32)


def _split_to_count(V, F, target):
    """Split the first (target - len(F)) triangles at the midpoint of edge (v1,v2): +1 triangle each. Exact face count."""
    extra = target - F.shape[0]
    if extra <= 0:
        return V, F
    if extra > F.shape[0]:
        raise ValueError("cannot reach target by single splits")
    V = V.astype(np.float64)
    f = F[:extra].astype(np.int64)
    mid = 0.5 * (V[f[:, 1]] + V[f[:, 2]])
    mid_idx = V.shape[0] + np.arange(extra)
    t1 = np.stack([f[:, 0], f[:, 1], mid_idx], 1)
    t2 = np.stack([f[:, 0], mid_idx, f[:, 2]], 1)
    Vn = np.concatenate([V, mid], 0)
    Fn = np.concatenate([t1, t2, F[extra:].astype(np.int64)], 0)
    return Vn.astype(np.float32), Fn.astype(np.uint32)


def cube(n: int, side: float = 20.0):
    """Axis-aligned cube centred at the origin, 6 faces x n x n quads x 2 -> 12 n^2 triangles, normals pointing INWARD
    (the sensor stands inside).  C1 uses n=29 -> 10 092 triangles."""
    h = side / 2.0
    parts = [
        _grid_rect([-h, -h, -h], [side, 0, 0], [0, side, 0], n, n),   # floor z=-h, normal +z
        _grid_rect([-h, -h, h], [0, side, 0], [side, 0, 0], n, n),    # ceiling, normal -z
        _grid_rect([-h, -h, -h], [0, 0, side], [side, 0, 0], n, n),   # y=-h, normal +y
        _grid_rect([-h, h, -h], [side, 0, 0], [0, 0, side], n, n),    # y=+h, normal -y
        _grid_rect([-h, -h, -h], [0, side, 0], [0, 0, side], n, n),   # x=-h, normal +x
        _grid_rect([h, -h, -h], [0, 0, side], [0, side, 0], n, n),    # x=+h, normal -x
    ]
    return _merge(parts)


def uvsphere(A: int, B: int, radius: float = 10.0):
    """Latitude/longitude sphere with A rings x B slices of quads -> 2AB triangles (tiny polar holes instead of
    degenerate cap triangles).  Mirrors make_sphere_map of rmcl_ros/src/benchmarks/lidar_corrector_embree_benchmark.cpp:38-71."""
    eps = 1e-3
    pol = np.linspace(eps, math.pi - eps, A + 1)
    az = np.linspace(0.0, 2.0 * math.pi, B + 1)
    P, Z = np.meshgrid(pol, az, indexing="ij")
    V = np.stack([radius * np.sin(P) * np.cos(Z), radius * np.sin(P) * np.sin(Z), radius * np.cos(P)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(A), np.arange(B), indexing="ij")
    a = (i * (B + 1) + j).ravel()
    b = a + 1
    c = a + (B + 1)
    d = c + 1
    F = np.concatenate([np.stack([a, c, d], 1), np.stack([a, d, b], 1)], 0)
    F = F.reshape(2, -1, 3).transpose(1, 0, 2).reshape(-1, 3)
    return V.astype(np.float32), F.astype(np.uint32)


def _rects_to_mesh(rects, n_faces):
    """rects: list of (origin, eu, ev).  Uniform cell size chosen so the face count is just below n_faces, then
    single-triangle splits make it exact."""
    dims = [(np.linalg.norm(eu), np.linalg.norm(ev)) for _, eu, ev in rects]

    def count(c):
        return sum(2 * max(1, math.ceil(w / c)) * max(1, math.ceil(h / c)) for w, h in dims)

    lo, hi = 1e-4, 100.0
    for _ in range(80):                      # smallest cell with count <= n_faces
        mid = 0.5 * (lo + hi)
        if count(mid) > n_faces:
            lo = mid
        else:
            hi = mid
    c = hi
    parts = [_grid_rect(o, eu, ev, max(1, math.ceil(w / c)), max(1, math.ceil(h / c))) for (o, eu, ev), (w, h) in zip(rects, dims)]
    V, F = _merge(parts)
    V, F = _split_to_count(V, F, n_faces)
    assert F.shape[0] == n_faces, (F.shape[0], n_faces)
    return V, F


def building(n_faces: int = 1_000_000):
    """One closed storey 60 x 40 x 3 m, interior walls every 5 m in x and y with 1.2 m door gaps, exactly n_faces triangles."""
    X, Y, Z = 60.0, 40.0, 3.0
    rects = [
        ([0, 0, 0], [X, 0, 0], [0, Y, 0]),        # floor (normal +z)
        ([0, 0, Z], [0, Y, 0], [X, 0, 0]),        # ceiling (normal -z)
        ([0, 0, 0], [0, 0, Z], [X, 0, 0]),        # y=0
        ([0, Y, 0], [X, 0, 0], [0, 0, Z]),        # y=Y
        ([0, 0, 0], [0, Y, 0], [0, 0, Z]),        # x=0
        ([X, 0, 0], [0, 0, Z], [0, Y, 0]),        # x=X
    ]
    door = 1.2
    # walls parallel to y at x = 5,10,...,55: segments between door gaps centred in every 5 m bay
    for xi in range(1, 12):
        x = 5.0 * xi
        for yj in range(8):
            y0, y1 = 5.0 * yj, 5.0 * (yj + 1)
            c = 0.5 * (y0 + y1)
            for (a, b) in ((y0, c - door / 2), (c + door / 2, y1)):
                rects.append(([x, a, 0], [0, b - a, 0], [0, 0, Z]))
            rects.append(([x, c - door / 2, 2.1], [0, door, 0], [0, 0, Z - 2.1]))   # lintel above the door
    for yj in range(1, 8):
        y = 5.0 * yj
        for xi in range(12):
            x0, x1 = 5.0 * xi, 5.0 * (xi + 1)
            c = 0.5 * (x0 + x1)
            for (a, b) in ((x0, c - door / 2), (c + door / 2, x1)):
                rects.append(([a, y, 0], [b - a, 0, 0], [0, 0, Z]))
            rects.append(([c - door / 2, y, 2.1], [door, 0, 0], [0, 0, Z - 2.1]))
    rects = [(np.array(o, float), np.array(u, float), np.array(v, float)) for o, u, v in rects]
    return _rects_to_mesh(rects, n_faces)


def _box_rects(lo, hi):
    lo = np.array(lo, float)
    hi = np.array(hi, float)
    d = hi - lo
    return [
        (lo, [0, d[1], 0], [d[0], 0, 0]),                                   # bottom (normal -z)
        ([lo[0], lo[1], hi[2]], [d[0], 0, 0], [0, d[1], 0]),                # top (+z)
        (lo, [d[0], 0, 0], [0, 0, d[2]]),                                   # y=lo (normal -y)
        ([lo[0], hi[1], lo[2]], [0, 0, d[2]], [d[0], 0, 0]),                # y=hi (+y)
        (lo, [0, 0, d[2]], [0, d[1], 0]),                                   # x=lo (-x)
        ([hi[0], lo[1], lo[2]], [0, d[1], 0], [0, 0, d[2]]),                # x=hi (+x)
    ]


def indoor(n_faces: int = 500_000):
    """One 12 x 8 x 3 m room with box furniture, exactly n_faces triangles (C4)."""
    X, Y, Z = 12.0, 8.0, 3.0
    rects = [
        ([0, 0, 0], [X, 0, 0], [0, Y, 0]),
        ([0, 0, Z], [0, Y, 0], [X, 0, 0]),
        ([0, 0, 0], [0, 0, Z], [X, 0, 0]),
        ([0, Y, 0], [X, 0, 0], [0, 0, Z]),
        ([0, 0, 0], [0, Y, 0], [0, 0, Z]),
        ([X, 0, 0], [0, 0, Z], [0, Y, 0]),
    ]
    boxes = [((2.0, 1.0, 0.0), (4.0, 2.0, 0.8)), ((8.0, 5.0, 0.0), (9.0, 7.5, 2.0)), ((5.0, 3.5, 0.0), (6.5, 4.5, 0.45)),
             ((10.5, 0.5, 0.0), (11.5, 3.0, 1.2)), ((0.5, 5.5, 0.0), (1.5, 7.5, 1.8))]
    for lo, hi in boxes:
        rects += _box_rects(lo, hi)
    rects = [(np.array(o, float), np.array(u, float), np.array(v, float)) for o, u, v in rects]
    return _rects_to_mesh(rects, n_faces)


# terrain(): the geometry its users need to know (m).  The ramp rises TERRAIN_RAMP["rise"] over TERRAIN_RAMP["run"] along +x, 10.008 deg.
TERRAIN_FLOOR = ((0.0, 0.0, 48.0, 32.0), (48.0, 16.0, 64.0, 32.0))                   # z = 0: (x0, y0, x1, y1) rectangles
TERRAIN_RAMP = {"x0": 4.0, "y0": 0.0, "y1": 4.0, "run": 17.0, "rise": 3.0}           # from z = 0 at x0 to the mezzanine at x0 + run
TERRAIN_MEZZANINE = {"x0": 21.0, "y0": 0.0, "x1": 37.0, "y1": 16.0, "top": 3.0, "bottom": 2.75}
TERRAIN_STAIRS = {"x0": 40.0, "y0": 20.0, "y1": 24.0, "steps": 8, "tread": 0.5, "riser": 0.25}   # up along +x, a wall behind the top
TERRAIN_BUMPS = {"x0": 48.0, "y0": 0.0, "size": 16.0, "height": 0.4, "period": 8.0}


def terrain_bump_z(x, y):
    """height of the bump field: height * (sin(2 pi u / period) sin(2 pi v / period))^2 over its square, 0 on its border (steepest 17.4 deg)"""
    b = TERRAIN_BUMPS
    k = 2.0 * math.pi / b["period"]
    return b["height"] * (np.sin(k * (np.asarray(x) - b["x0"])) * np.sin(k * (np.asarray(y) - b["y0"]))) ** 2


def _terrain_lattice(s):
    """the parts of terrain() on the dyadic lattice, with cell size s = 2^-k"""
    def n(length):
        return max(1, int(round(length / s)))
    parts = []
    for x0, y0, x1, y1 in TERRAIN_FLOOR:
        parts.append(_grid_rect([x0, y0, 0.0], [x1 - x0, 0, 0], [0, y1 - y0, 0], n(x1 - x0), n(y1 - y0)))
    r = TERRAIN_RAMP
    # ramp cells: run / 2^j along the slope (vertices x0 + run i / 2^j, rise i / 2^j stay dyadic)
    parts.append(_grid_rect([r["x0"], r["y0"], 0.0], [r["run"], 0, r["rise"]], [0, r["y1"] - r["y0"], 0], n(16.0), n(r["y1"] - r["y0"])))
    m = TERRAIN_MEZZANINE
    dx, dy, dz = m["x1"] - m["x0"], m["y1"] - m["y0"], m["top"] - m["bottom"]
    parts.append(_grid_rect([m["x0"], m["y0"], m["top"]], [dx, 0, 0], [0, dy, 0], n(dx), n(dy)))          # top (+z)
    parts.append(_grid_rect([m["x0"], m["y0"], m["bottom"]], [0, dy, 0], [dx, 0, 0], n(dy), n(dx)))       # underside (-z)
    parts.append(_grid_rect([m["x0"], m["y0"], m["bottom"]], [dx, 0, 0], [0, 0, dz], n(dx), 1))           # y = y0
    parts.append(_grid_rect([m["x0"], m["y1"], m["bottom"]], [0, 0, dz], [dx, 0, 0], 1, n(dx)))           # y = y1
    parts.append(_grid_rect([m["x0"], m["y0"], m["bottom"]], [0, 0, dz], [0, dy, 0], 1, n(dy)))           # x = x0
    parts.append(_grid_rect([m["x1"], m["y0"], m["bottom"]], [0, dy, 0], [0, 0, dz], n(dy), 1))           # x = x1
    st = TERRAIN_STAIRS
    w = st["y1"] - st["y0"]
    for k in range(st["steps"]):
        x = st["x0"] + k * st["tread"]
        parts.append(_grid_rect([x, st["y0"], k * st["riser"]], [0, w, 0], [0, 0, st["riser"]], n(w), n(st["riser"])))      # riser (vertical)
        parts.append(_grid_rect([x, st["y0"], (k + 1) * st["riser"]], [st["tread"], 0, 0], [0, w, 0], n(st["tread"]), n(w)))  # tread
    top = st["steps"] * st["riser"]
    parts.append(_grid_rect([st["x0"] + st["steps"] * st["tread"], st["y0"], 0.0], [0, 0, top], [0, w, 0], n(top), n(w)))  # back wall
    return parts


def terrain(n_tris: int = 1_000_000):
    """A mesh map for the surface constraint (PCDSensorUpdaterB200.projectToSurface): a flat floor at z = 0 (TERRAIN_FLOOR), a ramp
    (TERRAIN_RAMP, 3 m over 17 m) up to a mezzanine slab whose top is at 3 m over part of the floor (TERRAIN_MEZZANINE, 0.25 m thick),
    stairs with vertical risers (TERRAIN_STAIRS) and a field of smooth bumps (TERRAIN_BUMPS, terrain_bump_z) in the floor's missing corner.
    Every vertex except the bumps' is on a dyadic lattice (cell 2^-k, exact in float32), so points on its edges and vertices are exact.
    About n_tris triangles, at most n_tris: the finest lattice with at most n_tris / 2 triangles, the rest an nb x nb bump grid."""
    def count(parts):
        return sum(F.shape[0] for _, F in parts)
    s = 1.0
    parts = _terrain_lattice(s)
    if count(parts) + 2 * 4 * 4 > n_tris:
        raise ValueError(f"terrain needs at least {count(parts) + 32} triangles")
    while True:
        finer = _terrain_lattice(s / 2)
        if count(finer) > n_tris // 2:
            break
        s, parts = s / 2, finer
    b = TERRAIN_BUMPS
    nb = int(math.isqrt((n_tris - count(parts)) // 2))
    V, F = _grid_rect([b["x0"], b["y0"], 0.0], [b["size"], 0, 0], [0, b["size"], 0], nb, nb)
    V[:, 2] = terrain_bump_z(V[:, 0], V[:, 1])
    V[np.isin(V[:, 0], (b["x0"], b["x0"] + b["size"])) | np.isin(V[:, 1], (b["y0"], b["y0"] + b["size"])), 2] = 0.0     # the border meets the floor
    return _merge(parts + [(V, F)])


# --------------------------------------------------------------------------------------------------
# sensor models (field names follow rmagine / rmcl_msgs ScanInfo, DepthInfo: rmcl_ros/src/util/conversions.cpp:22-60)
# --------------------------------------------------------------------------------------------------


@dataclass
class SphericalModel:
    phi_min: float
    phi_inc: float
    phi_size: int
    theta_min: float
    theta_inc: float
    theta_size: int
    range_min: float
    range_max: float

    @property
    def size(self):
        return self.phi_size * self.theta_size

    @property
    def height(self):
        return self.phi_size

    @property
    def width(self):
        return self.theta_size


@dataclass
class PinholeModel:
    width: int
    height: int
    fx: float
    fy: float
    cx: float
    cy: float
    range_min: float
    range_max: float

    @property
    def size(self):
        return self.width * self.height


@dataclass
class O1DnModel:
    width: int
    height: int
    orig: np.ndarray            # (3,)
    dirs: np.ndarray            # (H*W, 3)
    range_min: float
    range_max: float

    @property
    def size(self):
        return self.width * self.height


@dataclass
class OnDnModel:
    width: int
    height: int
    origs: np.ndarray           # (H*W, 3)
    dirs: np.ndarray            # (H*W, 3)
    range_min: float
    range_max: float

    @property
    def size(self):
        return self.width * self.height


def c1_sensor():
    """C1: 32 x 32 spherical, phi in [-45,+45] deg, theta in [-pi, pi), range [0.1, 100]."""
    return SphericalModel(math.radians(-45.0), math.radians(90.0) / 31.0, 32, -math.pi, 2.0 * math.pi / 32.0, 32, 0.1, 100.0)


def c2_sensor():
    """C2: 128 x 1024 VLP/OS-128 style, phi from -25 deg in 40/127 deg steps, range [0.5, 120]."""
    return SphericalModel(math.radians(-25.0), math.radians(40.0) / 127.0, 128, -math.pi, 2.0 * math.pi / 1024.0, 1024, 0.5, 120.0)


def vlp16_900():
    """rmagine's vlp16_900(): 16 rows -15..+15 deg, 900 columns over 360 deg, range [0.5, 130] (benchmark sets range.min = 0)."""
    return SphericalModel(math.radians(-15.0), math.radians(2.0), 16, -math.pi, 2.0 * math.pi / 900.0, 900, 0.5, 130.0)


def c4_sensor():
    """C4: 640 x 480 depth camera, fx=fy=525, cx=319.5, cy=239.5, range [0.3, 10]."""
    return PinholeModel(640, 480, 525.0, 525.0, 319.5, 239.5, 0.3, 10.0)


# --------------------------------------------------------------------------------------------------
# transforms (numpy float32 [qx,qy,qz,qw,tx,ty,tz,stamp]; 32 bytes like rm::Transform)
# --------------------------------------------------------------------------------------------------

TRANSFORM_DTYPE = np.dtype([("R", np.float32, 4), ("t", np.float32, 3), ("stamp", np.uint32)])
CROSS_STATS_DTYPE = np.dtype([("dataset_mean", np.float32, 3), ("model_mean", np.float32, 3), ("covariance", np.float32, 9), ("n_meas", np.uint32)])
GAUSSIAN1D_DTYPE = np.dtype([("mean", np.float32), ("sigma", np.float32), ("n_meas", np.uint32)])
PARTICLE_ATTR_DTYPE = np.dtype([("likelihood", GAUSSIAN1D_DTYPE), ("state_sigma", np.float32, 6)])
RANGE_MEAS_DTYPE = np.dtype([("orig", np.float32, 3), ("dir", np.float32, 3), ("range", np.float32), ("cov", np.float32, 9)])
assert TRANSFORM_DTYPE.itemsize == 32 and CROSS_STATS_DTYPE.itemsize == 64
assert PARTICLE_ATTR_DTYPE.itemsize == 36 and RANGE_MEAS_DTYPE.itemsize == 64
# rmcl_msgs/ParticleStats as b2_particle_stats (include/rmcl_b200.h): what PCDSensorUpdaterB200.estimateStats returns
LIKELIHOOD_STATS_DTYPE = np.dtype([("min", np.float64), ("max", np.float64), ("mean", np.float64), ("sigma", np.float64)])
PARTICLE_STATS_DTYPE = np.dtype([("position", np.float64, 3), ("orientation", np.float64, 4), ("covariance", np.float64, 36), ("shift", np.float64),
                                 ("trans_bb_min", np.float64, 3), ("trans_bb_max", np.float64, 3), ("likelihood", LIKELIHOOD_STATS_DTYPE), ("nparticles", np.uint64)])
assert PARTICLE_STATS_DTYPE.itemsize == 440
# b2_residual_result: what PCDSensorUpdaterB200.resampleResidual returns
RESIDUAL_RESULT_DTYPE = np.dtype([("n_particles", np.uint64), ("draws", np.uint64), ("weight_sum", np.float64), ("weight_max", np.float64)])
assert RESIDUAL_RESULT_DTYPE.itemsize == 32
# b2_kld_result: what PCDSensorUpdaterB200.resampleKLD returns
KLD_RESULT_DTYPE = np.dtype([("n_particles", np.uint64), ("bins", np.uint64), ("weight_sum", np.float64), ("weight_max", np.float64)])
assert KLD_RESULT_DTYPE.itemsize == 32
# b2_recovery_state / b2_recovery_result: what PCDSensorUpdaterB200.recoveryObserve / recoveryInject return
RECOVERY_STATE_DTYPE = np.dtype([("w_avg", np.float64), ("w_slow", np.float64), ("w_fast", np.float64), ("p_inject", np.float64)])
assert RECOVERY_STATE_DTYPE.itemsize == 32
RECOVERY_RESULT_DTYPE = np.dtype([("p_inject", np.float64), ("n_replaced", np.uint64), ("n_failed", np.uint64)])
assert RECOVERY_RESULT_DTYPE.itemsize == 24
# b2_cluster_record / b2_cluster_result: what PCDSensorUpdaterB200.estimateClusters returns
CLUSTER_RECORD_DTYPE = np.dtype([("stats", PARTICLE_STATS_DTYPE), ("weight", np.float64), ("weight_int", np.uint64), ("bins", np.uint64), ("key", np.uint64)])
assert CLUSTER_RECORD_DTYPE.itemsize == 472
CLUSTER_RESULT_DTYPE = np.dtype([("n_clusters", np.uint64), ("n_records", np.uint64), ("bins", np.uint64), ("n_clustered", np.uint64), ("weight_total", np.uint64),
                                 ("rounds", np.uint64), ("weight_sum", np.float64), ("weight_max", np.float64)])
assert CLUSTER_RESULT_DTYPE.itemsize == 64
# b2_search_record: what PCDSensorUpdaterB200.globalSearch returns per kept peak
SEARCH_RECORD_DTYPE = np.dtype([("pose", TRANSFORM_DTYPE), ("score", np.float32), ("i", np.uint32), ("j", np.uint32), ("k", np.uint32)])
assert SEARCH_RECORD_DTYPE.itemsize == 48
# b2_search_bnb_result: the counts of PCDSensorUpdaterB200.globalSearchBnB
SEARCH_BNB_RESULT_DTYPE = np.dtype([("n_candidates", np.uint64), ("n_bounded", np.uint64), ("n_leaves", np.uint64), ("n_peaks", np.uint64), ("n_records", np.uint64),
                                    ("n_bounded_pass", np.uint64, (16,)), ("n_level", np.uint64, (25,)), ("best_score", np.float32), ("threshold", np.float32),
                                    ("n_passes", np.uint32), ("depth", np.uint32)])
assert SEARCH_BNB_RESULT_DTYPE.itemsize == 384


def quat_from_rpy(roll, pitch, yaw):
    """ZYX Euler -> quaternion (x,y,z,w), float64."""
    cr, sr = math.cos(roll / 2), math.sin(roll / 2)
    cp, sp = math.cos(pitch / 2), math.sin(pitch / 2)
    cy, sy = math.cos(yaw / 2), math.sin(yaw / 2)
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


def make_transform(t=(0, 0, 0), rpy=(0, 0, 0)):
    T = np.zeros((), TRANSFORM_DTYPE)
    T["R"] = quat_from_rpy(*rpy).astype(np.float32)
    T["t"] = np.asarray(t, np.float32)
    return T


def transforms(n):
    T = np.zeros((n,), TRANSFORM_DTYPE)
    T["R"][:, 3] = 1.0
    return T


def _qmul(a, b):
    ax, ay, az, aw = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bx, by, bz, bw = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], -1)


def _qrot(q, v):
    p = np.concatenate([v, np.zeros(v.shape[:-1] + (1,))], -1)
    qc = q * np.array([-1, -1, -1, 1.0])
    return _qmul(_qmul(q, p), qc)[..., :3]


def compose(a, b):
    """a * b in float64, returned as TRANSFORM_DTYPE (host-side convenience for tests/bench set-up only)."""
    qa, qb = np.asarray(a["R"], np.float64), np.asarray(b["R"], np.float64)
    ta, tb = np.asarray(a["t"], np.float64), np.asarray(b["t"], np.float64)
    q = _qmul(qa, qb)
    t = _qrot(qa, tb) + ta
    out = np.zeros(np.broadcast(a, b).shape, TRANSFORM_DTYPE)
    out["R"] = (q / np.linalg.norm(q, axis=-1, keepdims=True)).astype(np.float32)
    out["t"] = t.astype(np.float32)
    return out


def transform_points(T, pts):
    """T * p for an (n, 3) array, float64 inside, float32 out (host-side convenience for tests / bench set-up only)."""
    q, t = np.asarray(T["R"], np.float64), np.asarray(T["t"], np.float64)
    return (_qrot(q, np.asarray(pts, np.float64)) + t).astype(np.float32)


def inverse(a):
    qa, ta = np.asarray(a["R"], np.float64), np.asarray(a["t"], np.float64)
    qi = qa * np.array([-1, -1, -1, 1.0])
    out = np.zeros(np.shape(a), TRANSFORM_DTYPE)
    out["R"] = qi.astype(np.float32)
    out["t"] = (-_qrot(qi, ta)).astype(np.float32)
    return out


# --------------------------------------------------------------------------------------------------
# scenario constants (SURVEY.md 8d)
# --------------------------------------------------------------------------------------------------


def scenario_tsb():
    return make_transform((0.2, 0.0, 0.5), (0.0, 0.0, math.radians(10.0)))


def scenario_pose_offset():
    return make_transform((0.1, -0.05, 0.2), (0.0, 0.0, math.radians(3.0)))


def building_gt_pose():
    """Base 0.5 m above the floor (sensor ends up 1.0 m above it with scenario_tsb), near the footprint centre, yaw 30 deg."""
    return make_transform((31.3, 21.7, 0.5), (0.0, 0.0, math.radians(30.0)))


def indoor_gt_pose():
    return make_transform((6.3, 3.1, 0.7), (0.0, 0.0, math.radians(30.0)))


def noisy_ranges(ranges, range_max, seed=42, sigma=0.01, drop=0.02):
    """+N(0, sigma) range noise, `drop` of the beams set to range_max + 1 (mask coverage)."""
    rng = np.random.default_rng(seed)
    r = np.asarray(ranges, np.float32).copy()
    r += rng.normal(0.0, sigma, r.shape).astype(np.float32)
    k = rng.random(r.shape) < drop
    r[k] = np.float32(range_max + 1.0)
    return r


def pf_particles(n, footprint=(60.0, 40.0), z=0.5, seed=42, margin=0.3):
    """Uniform x,y over the footprint, constant z, yaw U[-pi,pi), roll=pitch=0 (mirrors rmcl_localization.cpp:287-320);
    attrs: likelihood = Gaussian1D::Identity() with mean forced to 1.0 (:323-327), i.e. {1, 0, 0}."""
    rng = np.random.default_rng(seed)
    P = transforms(n)
    P["t"][:, 0] = rng.uniform(margin, footprint[0] - margin, n).astype(np.float32)
    P["t"][:, 1] = rng.uniform(margin, footprint[1] - margin, n).astype(np.float32)
    P["t"][:, 2] = z
    yaw = rng.uniform(-math.pi, math.pi, n)
    P["R"][:, 2] = np.sin(yaw / 2).astype(np.float32)
    P["R"][:, 3] = np.cos(yaw / 2).astype(np.float32)
    A = np.zeros((n,), PARTICLE_ATTR_DTYPE)
    A["likelihood"]["mean"] = 1.0
    A["state_sigma"] = 0.1
    return P, A


def pf_beams(points, k, seed=42):
    """First k indices of a seeded permutation of the finite scan points -> RangeMeasurement array in the sensor frame
    (replaces the random_device sampling of PCDSensorUpdaterEmbree.cpp:276-327; cov = 0.1 I)."""
    pts = np.asarray(points, np.float32).reshape(-1, 3)
    finite = np.flatnonzero(np.isfinite(pts).all(1))
    rng = np.random.default_rng(seed)
    sel = rng.permutation(finite)[:k]
    p = pts[sel]
    rngs = np.sqrt((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1] + p[:, 2] * p[:, 2]).astype(np.float32)).astype(np.float32)
    B = np.zeros((len(sel),), RANGE_MEAS_DTYPE)
    B["dir"] = (p / rngs[:, None]).astype(np.float32)
    B["range"] = rngs
    B["cov"][:, [0, 4, 8]] = 0.1
    return B


# --------------------------------------------------------------------------------------------------
# sensor_msgs/PointCloud2 (field names of the ROS message; PointField datatypes: 2 UINT8, 7 FLOAT32, 8 FLOAT64)
# --------------------------------------------------------------------------------------------------

@dataclass
class PointField:
    name: str
    offset: int
    datatype: int
    count: int = 1


@dataclass
class PointCloud2:
    width: int
    height: int
    fields: list
    is_bigendian: bool
    point_step: int
    row_step: int
    data: np.ndarray            # uint8 (or a CUDA uint8 tensor)
    is_dense: bool = False


def pointcloud2(points, width, height, *, dtype=np.float32, point_step=16, offsets=(0, 4, 8), extra=None, row_pad=0, seed=0):
    """An organised cloud of `points` ((height*width, 3) in the sensor frame, row-major; NaN marks a miss, e.g. the points of a spherical
    scan's find with misses left as NaN): x, y, z as `dtype` (float32 or float64) at `offsets` inside `point_step` bytes, `row_pad` bytes
    after each row.  `extra` maps further field names to offsets: a field named "mask" is one UINT8 (random 0/1, as a filter node would
    write it), any other a FLOAT32 of random values.  Bytes no field covers are random as well, so nothing reads them unnoticed."""
    rng = np.random.default_rng(seed)
    P = np.asarray(points, np.float64).reshape(height, width, 3)
    dt = np.dtype(dtype).newbyteorder("<")
    fields = [PointField(n, int(o), 8 if dt.itemsize == 8 else 7) for n, o in zip("xyz", offsets)]
    for name, o in (extra or {}).items():
        fields.append(PointField(name, int(o), 2 if name == "mask" else 7))
    for f in fields:
        if f.offset + (1 if f.datatype == 2 else 4 if f.datatype == 7 else 8) > point_step:
            raise ValueError(f"field {f.name} does not fit into point_step {point_step}")
    row_step = width * point_step + row_pad
    buf = rng.integers(0, 256, height * row_step, dtype=np.uint8)
    rows = buf.reshape(height, row_step)[:, :width * point_step].reshape(height, width, point_step)
    with np.errstate(over="ignore"):                # a double beyond float range stays inf in a FLOAT32 cloud
        for k, f in enumerate(fields[:3]):
            rows[:, :, f.offset:f.offset + dt.itemsize] = P[:, :, k].astype(dt)[..., None].view(np.uint8)
    for f in fields[3:]:
        if f.datatype == 2:
            rows[:, :, f.offset] = rng.integers(0, 2, (height, width), dtype=np.uint8)
        else:
            rows[:, :, f.offset:f.offset + 4] = rng.uniform(0, 100, (height, width)).astype("<f4")[..., None].view(np.uint8)
    return PointCloud2(width, height, fields, False, point_step, row_step, buf)
