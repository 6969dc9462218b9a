"""The find's ray casting (k_rcc_find, k_intersect), its closest points (k_cpc_find) and the device Umeyama (k_umeyama_batch) at their
numerical and launch edges, against a float64 restatement of the same operations.

The oracle restates the device's FP32 hit definition op for op, so bit-equality with it shows that the two agree, not that either is right:
a mistake written into both (the frame change Tbm * Tsb, the sensor-frame normal and its flip toward the sensor, the miss encoding, the MT
acceptance rule with its AABB validation, Ericson's region tests) stays invisible to it.  Here a plain numpy float64 model checks them:
rays from the handle's own float32 model tables (b2_rcc_debug_model_tables) posed in float64 with unit quaternions, brute-force
Moller-Trumbore over every triangle, brute-force point-to-triangle distance, an SVD Umeyama.  The oracle takes the device's place in the
CPU test at the top, so the model and its bounds are checked against the FP32 definition on a machine without a GPU.

Admissible rays instead of loose tolerances.  u = 2^-24; for a ray (origin o, direction d, both in the map frame) and a face crossed at t:
  kappa = |e1| |e2| / |Ng|        1 / sin of the face's angle at v0 (MT's products are bounded by |e1| |e2|, its determinant is |Ng| |d| cos)
  S     = |o| + t |d| + E         E = max |vertex coordinate| of the scene
  tol   = K_T u kappa S / |cos|   length along the ray (t in units of |d|: tol / |d|)
  m     = EDGE_MARGIN + K_T u kappa S      distance across the ray
K_T = 32: the map-frame origin carries <= 6 u |o| from the FP32 pose (tf_mul, tf_apply), the direction <= 6 u (q_rot), and MT's t (FMA
cross and dot products, 2 u |a| |b| per cross component, 3 u per dot, u per edge difference and the division) <= 18 u kappa (t |d| + diam)
/ cos; the sum is <= 24 u kappa S / cos, with a third spare.
A ray is admissible if its float64 closest hit
  * is at least m from every edge of every face it crosses at or before that hit (float64 signed distance to the nearest edge, times |cos|),
  * has |cos| >= COS_MIN(kappa, rho), rho = 1 + diam / (t |d|)  (diam = longest edge of the face),
  * is separated by more than the t tolerance from the second-nearest float64 hit on a different, non-duplicate face,
  * lies more than m from tfar (and from range_min where that cuts) and from the origin.
COS_MIN is derived, not tuned.  The validation accepts MT's t only if tn <= fl(t C1) and tf >= fl(t C2), C1/C2 = 1 -+ 2^-14, for the
slab interval [tn, tf] of the face's AABB, which contains the true t* (for an axis-aligned face tn* = tf* = t*).  MT's FP32 error is
|t - t*| <= K_MT u kappa rho t / |cos| (K_MT = 24 covers the 18 above plus the division), formula F's slab ends are off by <= 3 u rho t
(fl(plane - o), fl(1/d), the product), and fl(t C1) loses u t.  The validation therefore cannot reject a true hit when
  K_MT u kappa rho / |cos| + 3 u rho + u <= 2^-14,   i.e.   |cos| >= COS_MIN = K_MT u kappa rho / (2^-14 - 3 u rho - u)
(about 0.034 for a right isosceles face seen from afar).  The bound is a worst case: MT's measured error on admissible rays stays below
4 u where the slab interval is tight (faces with flat AABBs, whose MT products do not cancel), so the validation would still accept every
admissible hit here with C1/C2 = 1 -+ 2^-22; at 1 -+ 2^-23 it rejects admissible hits and this file fails.

Admissible rays: hit / miss and face id exact (exact duplicates of a face resolve to the smallest id by the (t, face) rule); |t - t64| <= tol;
the sensor-frame point within tol + 2 u S of o + t64 d; the normal unit within 8 u, within K_N u kappa (K_N = 16: the FP32 cross product
of the edges, the normalisations and the rotation) of the float64 face normal, and dot(dir, n) <= 0.
Every ray: a reported hit is a real crossing of the reported face (t within its tol, signed edge distance >= -m), never of a zero-area
face, and no robust float64 hit (inside by m, |cos| >= COS_MIN, after m) lies before it by more than its tol; misses use the exact encoding.
Rays the model cannot redraw (a raster sensor model's table) are kept: their inadmissible rays take the every-ray checks only and are counted.

Closest points: |d - d64| <= K_D u kappa S, S = |q| + d + E (K_D = 16: the query's FP32 transform <= 6 u |q|, the region tests and the
closest point <= 8 u kappa (|q| + E), d2 and its square root); kappa is the larger of the reported face's and the float64 closest face's
(the reported distance is the minimum of FP32 candidates, so it is off by at most the error of one of the two; a sliver's barycentrics are
ill-conditioned, and the sphere's polar slivers (kappa ~ 10^3) show it), 1 for a zero-area face (its closest point is a segment's).  No
margin: the distance is continuous in the query.  The point within the same bound of
the float64 closest point on the reported face; the face id only where the float64 runner-up on another face is farther by > 2 bounds;
the normal the rotated unit Ng within K_N u kappa, no flip; hits = d <= max_dist where |d64 - max_dist| exceeds the bound.
Umeyama: the rotation of the float32 C's float64 SVD with S = diag(1, 1, sign det(U) det(V)); the device's rotation angle from it
<= K_R u |C| / g (K_R = 16), g = min(s1 + s2, s1 + s s3, s2 + s s3), s = sign det C: the polar factor moves by <= 2 |E| / g under a
perturbation E, and the FP32 Newton steps perturb by a few u |C|; cases with g = 0 are skipped.  The translation mm - R dm within
angle |dm| + 8 u (|mm| + |dm|).

Printed per case: rays redrawn, inadmissible rays kept, the largest error as a fraction of each bound, and (not asserted) how many rays
crossing a face within the edge margin missed it and every face behind the edge: evidence for a watertightness issue.
"""
import ctypes as C
import subprocess
import time

import numpy as np
import pytest

import native

U = 2.0 ** -24
K_T = 32.0
K_MT = 24.0
K_N = 16.0
K_D = 16.0
K_R = 16.0
EDGE_MARGIN = 1e-4
KEEP = 0.5                     # crossings kept by the model: signed edge distance (across the ray) above -KEEP
NOFACE = 0xFFFFFFFF
FIND_BLOCK = 64                # threads per k_rcc_find / k_cpc_find block
PERM_MAX_TILES = 11520         # the find's tile schedule covers at most this many tiles
_T0 = time.time()


def cos_min(kappa, rho):
    den = 2.0 ** -14 - 3 * U * rho - U
    return np.where(den > 0, K_MT * U * kappa * rho / np.where(den > 0, den, 1.0), np.inf)


# =====================================================================================================================================
# scenes
# =====================================================================================================================================
def degenerate_mesh():
    """inside a coarse cube: a triangle fan (shared edges), zero-area faces (collinear, repeated vertex), exact duplicates, slivers
    narrower than the edge margin, and two coplanar overlapping triangles"""
    from rmcl_b200 import synth
    V, F = synth.cube(3)
    vs, fs = [V.astype(np.float64)], [F.astype(np.int64)]
    n = len(V)

    def add(tris):
        nonlocal n
        tris = np.asarray(tris, np.float64).reshape(-1, 3, 3)
        vs.append(tris.reshape(-1, 3))
        fs.append(n + np.arange(3 * len(tris)).reshape(-1, 3))
        n += 3 * len(tris)
    ang = np.linspace(0, 2 * np.pi, 9)[:-1]
    ring = np.stack([3 * np.cos(ang) + 1.0, 3 * np.sin(ang) - 1.0, np.full(8, -5.0)], 1)
    ring[:, 2] += 0.5 * np.sin(3 * ang)                                          # a non-planar fan
    c = np.array([1.0, -1.0, -4.0])
    fan = [(c, ring[k], ring[(k + 1) % 8]) for k in range(8)]
    add(fan)
    add([((1, 1, 2), (2, 2, 2), (3, 3, 2)), ((-2, 3, 1), (-2, 3, 1), (0, 4, 1)), ((4, -6, 0), (5, -5, 1), (6, -4, 2))])      # zero area
    add([fan[2], fan[5]])                                                        # exact duplicates (same vertex order)
    add([((-4, -4, 3), (4, -4, 3), (0, -4 + 2e-5, 3)), ((-6, 5, -2), (-6, 5.00001, 6), (-6, 5, 6))])                          # slivers
    add([((-3, 0, 4), (3, 0, 4), (0, 3, 4)), ((-2, 1, 4), (2, 1, 4), (0, -2, 4))])                                            # coplanar overlap
    # a panel of faces one ulp off z = const at coordinates that are not round numbers: flat AABBs (the validation's slab interval is tight)
    # without the exact products of the cube's walls
    rng = np.random.default_rng(7)
    xs, ys = np.sort(rng.uniform(-8.7, 8.9, 7)), np.sort(rng.uniform(-2.3, 8.1, 7))
    zc = np.float32(-7.3071)
    Z = np.where(rng.random((7, 7)) < 0.5, zc, np.nextafter(zc, np.float32(0)))
    for i in range(6):
        for j in range(6):
            p = [(xs[i + a], ys[j + b], Z[i + a, j + b]) for a, b in ((0, 0), (1, 0), (1, 1), (0, 1))]
            add([(p[0], p[1], p[2]), (p[0], p[2], p[3])])
    Vd = np.concatenate(vs).astype(np.float32)
    Fd = np.concatenate(fs).astype(np.uint32)
    return Vd, Fd


_SC = {}


def mesh(name):
    from rmcl_b200 import synth
    if name == "cube":
        return synth.cube(8)
    if name == "sphere":
        return synth.uvsphere(12, 24)
    if name == "indoor":
        return synth.indoor(3000)
    if name == "degenerate":
        return degenerate_mesh()
    if name == "building":
        return synth.building(200000)
    raise KeyError(name)


class Scene64:
    """float64 view of a float32 mesh (the named scene's, or V, F given), with a grouping of the faces for culling large scenes"""

    def __init__(self, name, V=None, F=None):
        if V is None:
            V, F = mesh(name)
        self.name, self.V, self.F = name, V, F
        v = V.astype(np.float64)
        self.v0, self.v1, self.v2 = v[F[:, 0]], v[F[:, 1]], v[F[:, 2]]
        self.e1, self.e2 = self.v1 - self.v0, self.v2 - self.v0
        self.Ng = np.cross(self.e1, self.e2)
        self.nNg = np.linalg.norm(self.Ng, axis=1)
        self.l0 = np.linalg.norm(self.v2 - self.v1, axis=1)
        self.l1 = np.linalg.norm(self.e2, axis=1)
        self.l2 = np.linalg.norm(self.e1, axis=1)
        self.zero = self.nNg == 0
        with np.errstate(divide="ignore", invalid="ignore"):
            self.kappa = np.where(self.zero, np.inf, self.l1 * self.l2 / self.nNg)
        self.diam = np.maximum(np.maximum(self.l0, self.l1), self.l2)
        self.E = float(np.abs(v).max())
        self.bmax = np.abs(V).max(0)                                               # BvhView bx, by, bz
        key = np.ascontiguousarray(np.stack([self.v0, self.v1, self.v2], 1).reshape(len(F), 9))
        _, first, inv = np.unique(key, axis=0, return_index=True, return_inverse=True)
        self.dup = first[inv.reshape(-1)]                                          # smallest face id with the same ordered vertices
        self.groups = self._groups(np.arange(len(F)), 256) if len(F) > 4096 else [np.arange(len(F))]
        lo = [np.minimum(np.minimum(self.v0[g], self.v1[g]), self.v2[g]).min(0) for g in self.groups]
        hi = [np.maximum(np.maximum(self.v0[g], self.v1[g]), self.v2[g]).max(0) for g in self.groups]
        pad = 1e-3 * (1 + self.E)
        self.glo, self.ghi = np.array(lo) - pad, np.array(hi) + pad

    def _groups(self, idx, size):
        if len(idx) <= size:
            return [idx]
        c = (self.v0[idx] + self.v1[idx] + self.v2[idx]) / 3
        ax = int(np.argmax(c.max(0) - c.min(0)))
        o = idx[np.argsort(c[:, ax], kind="stable")]
        h = len(o) // 2
        return self._groups(o[:h], size) + self._groups(o[h:], size)


def scene(name):
    if name not in _SC:
        _SC[name] = Scene64(name)
    return _SC[name]


def gpu_map(name):
    import rmcl_b200
    key = "map:" + name
    if key not in _SC:
        sc = scene(name)
        _SC[key] = rmcl_b200.Map(sc.V, sc.F, device=0)
    return _SC[key]


def oracle_scene(po, name):
    key = "orc:" + name
    if key not in _SC:
        sc = scene(name)
        _SC[key] = po.Scene(sc.V, sc.F)
    return _SC[key]


# =====================================================================================================================================
# float64 model: poses, crossings, closest hits, admissibility
# =====================================================================================================================================
def quat(T):
    q = np.asarray(T["R"], np.float64)
    return q / np.linalg.norm(q)


def qmat(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def sensor_to_map(Tbm, Tsb):
    """T_sm = Tbm * Tsb in float64 with unit quaternions -> (R, t)"""
    Rb, Rs = qmat(quat(Tbm)), qmat(quat(Tsb))
    return Rb @ Rs, Rb @ np.asarray(Tsb["t"], np.float64) + np.asarray(Tbm["t"], np.float64)


def crossings(sc, o, d, chunk=128):
    """every float64 ray-triangle crossing with det != 0, finite t and signed edge distance (across the ray) above -KEEP:
    dict of flat arrays ray, face, t, edc, cos"""
    out = {k: [] for k in ("ray", "face", "t", "edc", "cos")}
    n = len(o)
    nd = np.linalg.norm(d, axis=1)
    for a in range(0, n, chunk):
        oo, dd = o[a:a + chunk], d[a:a + chunk]
        ok_r = np.isfinite(oo).all(1) & np.isfinite(dd).all(1) & (nd[a:a + chunk] > 0)
        if len(sc.groups) == 1:
            pairs = [(np.flatnonzero(ok_r), sc.groups[0])]
        else:
            with np.errstate(divide="ignore", invalid="ignore"):
                inv = 1.0 / dd
                t1 = (sc.glo[None] - oo[:, None]) * inv[:, None]
                t2 = (sc.ghi[None] - oo[:, None]) * inv[:, None]
            tn = np.where(np.isnan(t1) | np.isnan(t2), -np.inf, np.minimum(t1, t2)).max(2)
            tf = np.where(np.isnan(t1) | np.isnan(t2), np.inf, np.maximum(t1, t2)).min(2)
            hitg = (tn <= tf) & (tf >= 0) & ok_r[:, None]
            pairs = [(np.flatnonzero(hitg[:, g]), sc.groups[g]) for g in np.flatnonzero(hitg.any(0))]
        for rows, fi in pairs:
            if len(rows) == 0:
                continue
            ro, rd = oo[rows][:, None, :], dd[rows][:, None, :]
            e1, e2, v0 = sc.e1[fi], sc.e2[fi], sc.v0[fi]
            with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                pv = np.cross(rd, e2)
                det = np.einsum("rtk,tk->rt", pv, e1)
                tv = ro - v0
                Uu = np.einsum("rtk,rtk->rt", tv, pv) / det
                qv = np.cross(tv, e1)
                Vv = np.einsum("rtk,rtk->rt", np.broadcast_to(rd, qv.shape), qv) / det
                t = np.einsum("tk,rtk->rt", e2, qv) / det
                W = 1.0 - Uu - Vv
                nn = sc.nNg[fi]
                ed = np.minimum(np.minimum(W * nn / sc.l0[fi], Uu * nn / sc.l1[fi]), Vv * nn / sc.l2[fi])
                cs = np.abs(np.einsum("rk,tk->rt", rd[:, 0, :], sc.Ng[fi])) / (nn * nd[a + rows][:, None])
                edc = ed * cs
            keep = np.isfinite(t) & np.isfinite(edc) & (edc > -KEEP) & (det != 0) & (nn > 0)
            r, f = np.nonzero(keep)
            out["ray"].append(a + rows[r])
            out["face"].append(fi[f])
            out["t"].append(t[r, f])
            out["edc"].append(edc[r, f])
            out["cos"].append(cs[r, f])
    res = {k: (np.concatenate(v) if v else np.zeros(0, np.int64 if k in ("ray", "face") else np.float64)) for k, v in out.items()}
    o_ = np.argsort(res["ray"], kind="stable")
    return {k: v[o_] for k, v in res.items()}


def trace_model(sc, o, d, tfar=np.inf, range_min=None):
    """closest float64 hit (t > 0, t <= tfar) per ray, its admissibility and what the checks need.
    range_min: where a hit below it is cut (min_mode 1), it must also not lie near it."""
    n = len(o)
    cr = crossings(sc, o, d)
    nd, no = np.linalg.norm(d, axis=1), np.linalg.norm(o, axis=1)
    t, face = np.full(n, np.inf), np.full(n, NOFACE, np.int64)
    adm = np.ones(n, bool)
    why = np.zeros(n, np.int64)
    near_edge = np.zeros(n, bool)
    bounds = np.split(np.arange(len(cr["ray"])), np.searchsorted(cr["ray"], np.arange(1, n)))
    tf = float(tfar)
    for r in range(n):
        ix = bounds[r]
        if not (np.isfinite(o[r]).all() and np.isfinite(d[r]).all() and nd[r] > 0):
            continue                                                               # no crossing: an exact miss
        ct, cf, ce, cc = cr["t"][ix], cr["face"][ix], cr["edc"][ix], cr["cos"][ix]
        kap = sc.kappa[cf]
        S = no[r] + np.abs(ct) * nd[r] + sc.E
        tolt = K_T * U * kap * S / np.maximum(cc, 1e-300) / nd[r]
        m = EDGE_MARGIN + K_T * U * kap * S
        inside = (ce >= 0) & (ct > 0) & (ct <= tf if not np.isnan(tf) else np.zeros(len(ct), bool))
        if inside.any():
            j = np.flatnonzero(inside)
            j = j[np.lexsort((cf[j], ct[j]))][0]
            t[r], face[r] = ct[j], cf[j]
            tlim = ct[j]
        else:
            j = -1
            tlim = tf if np.isfinite(tf) else np.inf
        bad = 0
        if ((np.abs(ce) < m) & (ct > -tolt) & (ct <= tlim + tolt)).any():
            bad = 1                                                                  # an edge crossed at or before the hit
        if ((np.abs(ct) * nd[r] < m) & (ce > -m)).any():
            bad = bad or 2                                                           # the origin on a surface
        if np.isfinite(tf) and ((np.abs(ct - tf) <= tolt + m / nd[r]) & (ce > -m)).any():
            bad = bad or 3                                                           # a crossing at tfar
        if range_min is not None and ((np.abs(ct - range_min) <= tolt + m / nd[r]) & (ce > -m) & (ct <= tlim + tolt)).any():
            bad = bad or 4
        if j >= 0:
            near_edge[r] = abs(ce[j]) < m[j]
            rho = 1.0 + sc.diam[cf[j]] / (ct[j] * nd[r])
            if cc[j] < cos_min(kap[j], rho):
                bad = bad or 5
            other = inside & (sc.dup[cf] != sc.dup[cf[j]]) & (np.abs(ct - ct[j]) <= tolt + tolt[j])
            if other.any():
                bad = bad or 6
        adm[r] = bad == 0
        why[r] = bad
    return dict(t=t, face=face, adm=adm, why=why, near_edge=near_edge, cr=cr, bounds=bounds, nd=nd, no=no)


def check_hits(sc, ref, t_dev, f_dev, tfar=np.inf, range_min=None, what=""):
    """t_dev (inf / anything on a miss), f_dev (NOFACE on a miss) against the model; -> dict of worst ratios and counts"""
    n = len(t_dev)
    f_dev = f_dev.astype(np.int64)
    hit = f_dev != NOFACE
    cr, bounds, nd = ref["cr"], ref["bounds"], ref["nd"]
    adm = ref["adm"]
    worst_t = 0.0
    assert not (hit & np.isin(f_dev, np.flatnonzero(sc.zero))).any(), (what, "a zero-area face reported")
    # admissible rays: exact hit / miss and face, t within tol
    a = np.flatnonzero(adm)
    mism = a[(f_dev[a] != np.where(np.isfinite(ref["t"][a]), ref["face"][a], NOFACE))]
    assert len(mism) == 0, (what, "face / hit differs on admissible rays", mism[:5], f_dev[mism[:5]], ref["face"][mism[:5]], ref["t"][mism[:5]])
    for r in range(n):
        ix = bounds[r]
        ct, cf, ce, cc = cr["t"][ix], cr["face"][ix], cr["edc"][ix], cr["cos"][ix]
        S = ref["no"][r] + np.abs(ct) * nd[r] + sc.E if len(ix) else np.zeros(0)
        tolt = K_T * U * sc.kappa[cf] * S / np.maximum(cc, 1e-300) / nd[r] if len(ix) else np.zeros(0)
        m = EDGE_MARGIN + K_T * U * sc.kappa[cf] * S if len(ix) else np.zeros(0)
        if hit[r]:
            k = np.flatnonzero(cf == f_dev[r])
            assert len(k) == 1, (what, r, "reported face is not crossed", int(f_dev[r]))
            k = k[0]
            assert abs(t_dev[r] - ct[k]) <= tolt[k] and ce[k] >= -m[k] and 0 < t_dev[r] <= tfar, (what, r, t_dev[r], ct[k], tolt[k], ce[k], m[k])
            if adm[r]:
                worst_t = max(worst_t, abs(t_dev[r] - ct[k]) / tolt[k])
            limit = t_dev[r]
        else:
            limit = tfar
            if range_min is not None and ((ce >= 0) & (ct > 0) & (ct < range_min + tolt)).any():
                continue                                                             # min_mode: the closest hit is below range_min
        if len(ix) and not np.isnan(limit):
            rho = 1.0 + sc.diam[cf] / (np.maximum(ct, 1e-300) * nd[r])
            robust = (ce >= m) & (cc >= cos_min(sc.kappa[cf], rho)) & (ct * nd[r] > m) & (ct < limit - tolt)
            if hit[r]:
                robust &= ct < limit - tolt[np.flatnonzero(cf == f_dev[r])[0]]
            assert not robust.any(), (what, r, "a robust float64 hit lies before the reported one", ct[robust][:3], cf[robust][:3], limit, int(f_dev[r]))
    # near-edge rays that missed everything up to the model's hit: watertightness evidence
    ne = np.flatnonzero(ref["near_edge"])
    holes = int(np.sum(~hit[ne] | (t_dev[ne] > ref["t"][ne] * (1 + 1e-5))))
    return dict(worst_t=worst_t, holes=holes, near_edge=len(ne), inadmissible=int((~adm).sum()), n=n, hits=int(hit.sum()))


# =====================================================================================================================================
# find: rays, model buffers
# =====================================================================================================================================
def model_tables(h):
    import rmcl_b200
    lib = rmcl_b200.load_library()
    n = C.c_uint32()
    assert lib.b2_rcc_debug_model_tables(h._h, None, None, C.byref(n)) == 0
    d = np.zeros((n.value, 3), np.float32)
    assert lib.b2_rcc_debug_model_tables(h._h, C.c_void_p(d.ctypes.data), None, C.byref(n)) == 0
    return d


def rays_of(Tbm, Tsb, orig_s, dir_s):
    R, t = sensor_to_map(Tbm, Tsb)
    o = np.broadcast_to(np.asarray(orig_s, np.float64).reshape(-1, 3), dir_s.shape) @ R.T + t
    return o, np.asarray(dir_s, np.float64) @ R.T, R


def sim_params(range_min, range_max, opts):
    tfar_mode, min_mode, miss_fill = opts
    tfar = np.inf if tfar_mode else float(np.float32(range_max))
    return tfar, (float(np.float32(range_min)) if min_mode else None), miss_fill


def check_find(sc, out, Tbm, Tsb, orig_s, dir_s, range_min, range_max, opts=(0, 0, 0), ref=None, idx=None, what=""):
    """modelView-shaped output (points, normals, hits, face_ids, ranges) of rays dir_s (sensor frame) against the model.
    idx: the subset of rays to compare (None: all).  -> summary dict"""
    tfar, rmin, miss_fill = sim_params(range_min, range_max, opts)
    idx = np.arange(len(dir_s)) if idx is None else np.asarray(idx)
    os_ = np.broadcast_to(np.asarray(orig_s, np.float32).reshape(-1, 3), (len(dir_s), 3))[idx]
    ds = np.asarray(dir_s, np.float32)[idx]
    o, d, R = rays_of(Tbm, Tsb, os_, ds)
    if ref is None:
        ref = trace_model(sc, o, d, tfar, rmin)
    hits, faces = out["hits"][idx], out["face_ids"][idx].astype(np.int64)
    rng_, pts, nrm = out["ranges"][idx].astype(np.float64), out["points"][idx].astype(np.float64), out["normals"][idx].astype(np.float64)
    assert np.array_equal(hits == 1, faces != NOFACE) and np.isin(hits, (0, 1)).all(), what
    # the min_mode cut: the model's closest hit below range_min is a miss
    if rmin is not None:
        cut = np.isfinite(ref["t"]) & (ref["t"] < rmin)
        ref = dict(ref, t=np.where(cut, np.inf, ref["t"]), face=np.where(cut, NOFACE, ref["face"]))
    summ = check_hits(sc, ref, np.where(hits == 1, rng_, np.inf), faces, tfar, rmin, what)
    # misses: the exact encoding
    miss = hits == 0
    fill = 0.0 if miss_fill else np.nan
    assert (rng_[miss] == np.float64(np.float32(np.float32(range_max) + np.float32(1.0)))).all(), (what, "miss range", np.unique(rng_[miss])[:4])
    for a in (pts[miss], nrm[miss]):
        assert (np.isnan(a).all() if np.isnan(fill) else (a == 0).all() and not np.signbit(a).any()), (what, "miss fill", a[:2])
    # hits: point, normal
    h = np.flatnonzero(~miss)
    worst_p = worst_n = 0.0
    if len(h):
        f = faces[h]
        S = ref["no"][h] + rng_[h] * ref["nd"][h] + sc.E
        kap = sc.kappa[f]
        ng = sc.Ng[f] / sc.nNg[f][:, None] @ R                                       # float64 face normal in the sensor frame
        dsn = ds[h].astype(np.float64)
        ng = np.where((np.einsum("ij,ij->i", dsn, ng) > 0)[:, None], -ng, ng)
        nn = np.linalg.norm(nrm[h], axis=1)
        assert (np.abs(nn - 1) <= 8 * U).all(), (what, "normal not unit", nn[np.argmax(np.abs(nn - 1))])
        assert (np.einsum("ij,ij->i", dsn, nrm[h]) <= 0).all(), (what, "normal faces away from the sensor")
        ang = np.linalg.norm(np.cross(nrm[h], ng), axis=1) + np.maximum(0.0, -np.einsum("ij,ij->i", nrm[h], ng))
        nb = K_N * U * kap
        assert (ang <= nb).all(), (what, "normal", float((ang / nb).max()), h[np.argmax(ang / nb)])
        worst_n = float((ang / nb).max())
        a = h[ref["adm"][h]]
        if len(a):
            S_a = ref["no"][a] + ref["t"][a] * ref["nd"][a] + sc.E
            cosr = np.array([ref["cr"]["cos"][ref["bounds"][r]][ref["cr"]["face"][ref["bounds"][r]] == faces[r]][0] for r in a])
            tol = K_T * U * sc.kappa[faces[a]] * S_a / cosr
            want = os_[a].astype(np.float64) + ref["t"][a][:, None] * ds[a].astype(np.float64)
            dp = np.linalg.norm(pts[a] - want, axis=1)
            assert (dp <= tol + 2 * U * S_a).all(), (what, "point", float((dp / (tol + 2 * U * S_a)).max()))
            worst_p = float((dp / (tol + 2 * U * S_a)).max())
    summ.update(worst_p=worst_p, worst_n=worst_n, n=len(idx), hits=len(h))
    return summ, ref


def log(what, s, redrawn=None):
    extra = "" if redrawn is None else f" redrawn {redrawn}"
    print(f"{what}: rays {s.get('n', '?')} hits {s.get('hits', '?')} inadmissible kept {s['inadmissible']}{extra}; worst/bound t {s['worst_t']:.3f} "
          f"point {s.get('worst_p', 0):.3f} normal {s.get('worst_n', 0):.3f}; near-edge rays {s['near_edge']}, missed there {s['holes']}")


# =====================================================================================================================================
# inputs
# =====================================================================================================================================
def unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def random_dirs(n, rng):
    return unit(rng.normal(size=(n, 3))).astype(np.float32)


def pose(t=(0, 0, 0), q=None, rpy=(0, 0, 0)):
    from rmcl_b200 import synth
    T = synth.make_transform(t, rpy)
    if q is not None:
        T["R"] = np.asarray(unit(q), np.float32)
    return T


def near_180(axis, eps=1e-3):
    a = np.zeros(3)
    a[axis] = 1.0
    a = unit(a + np.array([0.01, -0.02, 0.015]))
    th = np.pi - eps
    return np.concatenate([a * np.sin(th / 2), [np.cos(th / 2)]])


TSB = dict(t=(0.2, -0.1, 0.3), rpy=(0.05, -0.03, 0.4))


def tsb():
    return pose(TSB["t"], rpy=TSB["rpy"])


def redraw(sc, make, n, seed, tfar=np.inf, rmin=None, tries=40):
    """make(k, rng) -> (o, d) float32 map-frame rays; draws n admissible rays -> (o, d, ref, redrawn)"""
    rng = np.random.default_rng(seed)
    o, d = make(n, rng)
    redrawn = 0
    for _ in range(tries):
        ref = trace_model(sc, o.astype(np.float64), d.astype(np.float64), tfar, rmin)
        bad = np.flatnonzero(~ref["adm"])
        if len(bad) == 0:
            return o, d, ref, redrawn
        redrawn += len(bad)
        o2, d2 = make(len(bad), rng)
        o[bad], d[bad] = o2, d2
    raise AssertionError(("could not draw admissible rays", sc.name, len(bad)))


# =====================================================================================================================================
# closest points
# =====================================================================================================================================
def closest_on_faces(sc, q, faces):
    """float64 closest point of q (k,3) on the triangles `faces` (k,) or on all (faces None: (k, F, 3))"""
    if faces is None:
        a, b, c, p = sc.v0[None], sc.v1[None], sc.v2[None], q[:, None, :]
    else:
        a, b, c, p = sc.v0[faces], sc.v1[faces], sc.v2[faces], q
    nrm = np.cross(b - a, c - a)
    nn = np.linalg.norm(nrm, axis=-1, keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        n_ = nrm / nn
        h = np.einsum("...k,...k->...", p - a, n_)
        x = p - h[..., None] * n_
        s0 = np.einsum("...k,...k->...", np.cross(b - a, x - a), n_)
        s1 = np.einsum("...k,...k->...", np.cross(c - b, x - b), n_)
        s2 = np.einsum("...k,...k->...", np.cross(a - c, x - c), n_)
    inside = (nn[..., 0] > 0) & (s0 >= 0) & (s1 >= 0) & (s2 >= 0)
    best = np.where(inside[..., None], x, np.nan)
    bd = np.where(inside, np.linalg.norm(p - x, axis=-1), np.inf)
    for u_, v_ in ((a, b), (b, c), (c, a)):
        e = v_ - u_
        ee = np.einsum("...k,...k->...", e, e)
        with np.errstate(divide="ignore", invalid="ignore"):
            w = np.clip(np.where(ee > 0, np.einsum("...k,...k->...", p - u_, e) / ee, 0.0), 0.0, 1.0)
        y = u_ + w[..., None] * e
        dy = np.linalg.norm(p - y, axis=-1)
        better = dy < bd
        best = np.where(better[..., None], y, best)
        bd = np.where(better, dy, bd)
    return best, bd


def cpc_model(sc, q, chunk=64):
    """-> (d64, face64, runner-up distance on a face that is not an exact duplicate of face64)"""
    n = len(q)
    d1, f1, d2 = np.full(n, np.inf), np.full(n, NOFACE, np.int64), np.full(n, np.inf)
    fin = np.isfinite(q).all(1)
    for a in range(0, n, chunk):
        rows = np.arange(a, min(n, a + chunk))
        rows = rows[fin[rows]]
        if len(rows) == 0:
            continue
        P, D = closest_on_faces(sc, q[rows], None)
        j = np.argmin(D, axis=1)
        r = np.arange(len(rows))
        d1[rows], f1[rows] = D[r, j], j
        other = sc.dup[None, :] != sc.dup[j][:, None]
        d2[rows] = np.where(other, D, np.inf).min(1)
    return d1, f1, d2


def check_cpc(sc, out, pts_s, Tbm, Tsb, max_dist, mask=None, skip_masked=False, what=""):
    n = len(pts_s)
    o, _, R = rays_of(Tbm, Tsb, np.zeros(3), np.zeros((1, 3)))
    with np.errstate(invalid="ignore"):
        q = np.asarray(pts_s, np.float64) @ R.T + o[0]
    d64, f64, d2 = cpc_model(sc, q)
    face, hits, dist = out["face_ids"].astype(np.int64), out["hits"], out["ranges"].astype(np.float64)
    P, Nr = out["points"].astype(np.float64), out["normals"].astype(np.float64)
    skipped = np.zeros(n, bool) if not skip_masked else ~(np.asarray(mask) > 0)
    miss = ~np.isfinite(q).all(1) | skipped
    # the miss encoding: range +inf, face NOFACE, hits 0, NaN point and normal
    assert (face[miss] == NOFACE).all() and (hits[miss] == 0).all() and np.isposinf(dist[miss]).all(), what
    assert np.isnan(P[miss]).all() and np.isnan(Nr[miss]).all(), what
    k = np.flatnonzero(~miss)
    assert (face[k] != NOFACE).all(), what
    S = np.linalg.norm(q[k], axis=1) + d64[k] + sc.E
    kc = np.where(sc.zero, 1.0, sc.kappa)
    tol = K_D * U * np.maximum(kc[face[k]], kc[f64[k]]) * S
    err = np.abs(dist[k] - d64[k])
    assert (err <= tol).all(), (what, "distance", float((err / tol).max()), k[np.argmax(err / tol)])
    # the point: float64 closest point on the reported face, in the sensor frame
    Pf, _ = closest_on_faces(sc, q[k], face[k])
    Ps = (Pf - o[0]) @ R
    ep = np.linalg.norm(P[k] - Ps, axis=1)
    assert (ep <= tol).all(), (what, "point", float((ep / tol).max()), k[np.argmax(ep / tol)])
    sep = d2[k] - d64[k] > 2 * tol
    assert (sc.dup[face[k][sep]] == sc.dup[f64[k][sep]]).all(), (what, "face", k[sep][sc.dup[face[k][sep]] != sc.dup[f64[k][sep]]][:5])
    k = k[~sc.zero[face[k]]]                                                         # a segment's closest point is real; its normal is not
    nref = (sc.Ng[face[k]] / sc.nNg[face[k]][:, None]) @ R
    ang = np.linalg.norm(np.cross(Nr[k], nref), axis=1) + np.maximum(0.0, -np.einsum("ij,ij->i", Nr[k], nref))
    nb = K_N * U * sc.kappa[face[k]]
    assert (ang <= nb).all(), (what, "normal", float((ang / nb).max()))
    k = np.flatnonzero(~miss)
    clear = np.abs(d64[k] - np.float32(max_dist)) > tol
    assert np.array_equal(hits[k][clear] == 1, d64[k][clear] <= np.float32(max_dist)), what
    s = dict(worst_d=float((err / tol).max()) if len(err) else 0.0, worst_p=float((ep / tol).max()) if len(ep) else 0.0,
             worst_n=float((ang / nb).max()) if len(ang) else 0.0, face_checked=int(sep.sum()), n=n)
    print(f"{what}: points {n} worst/bound distance {s['worst_d']:.3f} point {s['worst_p']:.3f} normal {s['worst_n']:.3f}; faces compared {s['face_checked']}")
    return s


def cpc_queries(sc, n, rng):
    """points on faces, on edges, on vertices, the centre, random interior points, 10^3 outside, NaN / inf"""
    ok = np.flatnonzero(~sc.zero)
    f = ok[rng.integers(0, len(ok), n)]
    w = rng.dirichlet((1, 1, 1), n)
    on_face = w[:, :1] * sc.v0[f] + w[:, 1:2] * sc.v1[f] + w[:, 2:] * sc.v2[f]
    s = rng.uniform(0, 1, (n, 1))
    on_edge = sc.v0[f] + s * sc.e1[f]
    on_vert = sc.v1[f]
    inner = rng.uniform(-0.8 * sc.E, 0.8 * sc.E, (n, 3))
    outer = unit(rng.normal(size=(n, 3))) * 1e3
    pick = rng.integers(0, 5, n)
    q = np.choose(pick[:, None], [on_face, on_edge, on_vert, inner, outer])
    q[0] = 0.0                                                                       # the centre (of the cube: equidistant from six walls)
    if n > 8:
        q[3] = np.nan
        q[5, 1] = np.inf
        q[7, 2] = -np.inf
    return q


# =====================================================================================================================================
# Umeyama
# =====================================================================================================================================
def rand_rot(rng):
    q = unit(rng.normal(size=4))
    return qmat(q)


def stats_record(Cm, dm, mm, n=100):
    from rmcl_b200 import synth
    s = np.zeros((), synth.CROSS_STATS_DTYPE)
    s["covariance"] = np.asarray(Cm, np.float32).T.reshape(9)                        # [c * 3 + r] = C[r, c]
    s["dataset_mean"], s["model_mean"], s["n_meas"] = np.asarray(dm, np.float32), np.asarray(mm, np.float32), n
    return s


def umeyama_model(s):
    """-> (R, t, |C|, g); R, t None for n_meas == 0"""
    if int(s["n_meas"]) == 0:
        return None, None, 0.0, 0.0
    Cm = np.asarray(s["covariance"], np.float64).reshape(3, 3).T
    Uu, sv, Vt = np.linalg.svd(Cm)
    sg = np.sign(np.linalg.det(Uu) * np.linalg.det(Vt)) or 1.0
    R = Uu @ np.diag([1.0, 1.0, sg]) @ Vt
    t = np.asarray(s["model_mean"], np.float64) - R @ np.asarray(s["dataset_mean"], np.float64)
    sdet = np.sign(np.linalg.det(Cm))
    g = min(sv[0] + sv[1], sv[0] + sdet * sv[2], sv[1] + sdet * sv[2])
    return R, t, sv[0], g


def umeyama_cases(rng):
    """-> list of (label, stats record)"""
    cases = []
    for k in range(20):
        sv = np.sort(rng.uniform(0.05, 1.0, 3))[::-1]
        cases.append(("random", rand_rot(rng) @ np.diag(sv) @ rand_rot(rng), rng.normal(size=3), rng.normal(size=3)))
    base = rand_rot(rng) @ np.diag([1.0, 0.6, 0.3]) @ rand_rot(rng)
    for e in range(-18, 19, 3):
        cases.append((f"scale 1e{e}", base * 10.0 ** e, rng.normal(size=3), rng.normal(size=3)))
    for e in (-20, -19, 19, 20):
        cases.append((f"scale 1e{e}", base * 10.0 ** e, rng.normal(size=3), rng.normal(size=3)))
    for r3 in (1e-2, 1e-4, 1e-7):
        for sg in (1, -1):
            for k in range(3):
                Ua, Vb = rand_rot(rng), rand_rot(rng)
                cases.append((f"s3 {sg * r3:g}", Ua @ np.diag([1.0, 0.5, sg * r3]) @ Vb.T, rng.normal(size=3), rng.normal(size=3)))
    Ua, Vb = rand_rot(rng), rand_rot(rng)
    cases.append(("rank 2", Ua @ np.diag([1.0, 0.4, 0.0]) @ Vb.T, rng.normal(size=3), rng.normal(size=3)))
    a, b = rng.normal(size=3), rng.normal(size=3)
    cases.append(("rank 1", np.outer(a, b), rng.normal(size=3), rng.normal(size=3)))
    for k in range(4):
        cases.append(("means 1e4", rand_rot(rng) @ np.diag(np.sort(rng.uniform(0.1, 1, 3))[::-1]) @ rand_rot(rng), rng.uniform(-1e4, 1e4, 3),
                      rng.uniform(-1e4, 1e4, 3)))
    # the ICP case: C = sum (M - mm)(D - dm)^T / n of a corridor-like scan and a slightly rotated copy: near-SPD, ill-conditioned
    P = np.concatenate([rng.uniform([-20, -1, 0], [20, 1, 3], (500, 3)), rng.uniform([-20, -1.05, 0], [20, -0.95, 3], (100, 3))])
    Rs = qmat(unit([0.001, -0.002, 0.01, 1.0]))
    M = P @ Rs.T + [0.02, -0.01, 0.005]
    cases.append(("icp corridor", (M - M.mean(0)).T @ (P - P.mean(0)) / len(P), P.mean(0), M.mean(0)))
    out = [(lab, stats_record(Cm, dm, mm)) for lab, Cm, dm, mm in cases]
    out.append(("n_meas 0", stats_record(base, rng.normal(size=3), rng.normal(size=3), n=0)))
    return out


def check_umeyama(out, cases, what=""):
    worst_r = worst_t = 0.0
    for (lab, s), T in zip(cases, out):
        R, t, nC, g = umeyama_model(s)
        if R is None:
            assert np.array_equal(T["R"], np.float32([0, 0, 0, 1])) and np.array_equal(T["t"], np.zeros(3, np.float32)), (what, lab)
            continue
        qd = np.asarray(T["R"], np.float64)
        assert abs(np.linalg.norm(qd) - 1) <= 8 * U, (what, lab, qd)
        if not g > 0:
            continue                                                                 # the rotation is not unique
        Rd = qmat(qd / np.linalg.norm(qd))
        E = Rd.T @ R
        ang = np.arctan2(np.linalg.norm([E[2, 1] - E[1, 2], E[0, 2] - E[2, 0], E[1, 0] - E[0, 1]]) / 2, (np.trace(E) - 1) / 2)
        rb = K_R * U * nC / g
        assert ang <= rb, (what, lab, "rotation", ang, rb)
        dm, mm = np.asarray(s["dataset_mean"], np.float64), np.asarray(s["model_mean"], np.float64)
        tb = rb * np.linalg.norm(dm) + 8 * U * (np.linalg.norm(mm) + np.linalg.norm(dm))
        et = np.linalg.norm(np.asarray(T["t"], np.float64) - t)
        assert et <= tb, (what, lab, "translation", et, tb)
        worst_r, worst_t = max(worst_r, ang / rb), max(worst_t, et / tb)
    print(f"{what}: cases {len(cases)} worst/bound rotation {worst_r:.3f} translation {worst_t:.3f}")
    return worst_r


# =====================================================================================================================================
# the host harness: ray_setup's B2_RAY_INTBOX flag
# =====================================================================================================================================
def intbox_flags(o, d, bmax):
    lines = "".join(" ".join(float(x).hex() for x in np.concatenate([a, b])) + "\n" for a, b in zip(o.astype(np.float32), d.astype(np.float32)))
    r = subprocess.run([native.nvcc_program("node_visit/node_visit.cu"), "flags"] + [float(x).hex() for x in np.asarray(bmax, np.float32)], input=lines,
                       capture_output=True, text=True, timeout=600, check=True)
    return np.array([int(x) for x in r.stdout.split()], np.int64)


def unflagged_ray(d, bmax, axis=0):
    """(origin coordinate, direction component) on `axis` with d > 1 for which ray_setup's far addend is exactly +0 with |idir| < 1: the
    ray takes the float reduction of the box test.  Emulates ray_setup's rounded float32 operations: idir = 1/d, oi = o idir,
    dl = (|oi| + B |idir|) 2^-20, ncf = dl - oi (zero only if o ~ B 2^-20; d is nudged until some o hits it exactly)."""
    f = np.float32
    B, k20, dk = f(bmax[axis]), f(2.0 ** -20), f(d[axis])
    assert dk > 1
    for _ in range(1000):
        idir = f(1) / dk
        o = f(float(B) * 2.0 ** -20 / (1 - 2.0 ** -20))
        last = None
        for _ in range(64):
            r = (abs(o * idir) + B * abs(idir)) * k20 - o * idir
            if r == 0:
                return o, dk
            s = r > 0
            if last is not None and s != last:
                break                                                                  # stepped over zero: try another d
            last = s
            o = np.nextafter(o, f(np.inf) if s else f(-np.inf))
        dk = np.nextafter(dk, f(np.inf))
    raise AssertionError("no unflagged origin found")


# =====================================================================================================================================
# tests
# =====================================================================================================================================
SMALL = ("cube", "sphere", "indoor", "degenerate")


def inside_rays(sc, spread=0.7):
    def make(k, rng):
        return rng.uniform(-spread, spread, (k, 3)).astype(np.float32) * np.float32(sc.E) * np.float32(0.9), random_dirs(k, rng)
    return make


def room_rays(lo, hi):
    def make(k, rng):
        return rng.uniform(lo, hi, (k, 3)).astype(np.float32), random_dirs(k, rng)
    return make


def grazing_rays(sc):
    """rays aimed at a random point of a random face with |cos| of the incidence uniform in [0.02, 0.2], from 0.5 to 5 m before it"""
    ok = np.flatnonzero(~sc.zero)

    def make(k, rng):
        f = ok[rng.integers(0, len(ok), k)]
        w = rng.dirichlet((2, 2, 2), k)
        p = w[:, :1] * sc.v0[f] + w[:, 1:2] * sc.v1[f] + w[:, 2:] * sc.v2[f]
        n = sc.Ng[f] / sc.nNg[f][:, None]
        t = unit(np.cross(n, rng.normal(size=(k, 3))))
        c = rng.uniform(0.02, 0.2, k)[:, None]
        d = unit(np.sqrt(1 - c * c) * t - c * n)
        return (p - d * rng.uniform(0.5, 5.0, (k, 1))).astype(np.float32), d.astype(np.float32)
    return make


def make_rays_for(sc):
    if sc.name == "indoor":
        main = room_rays((0.3, 0.3, 0.3), (11.7, 7.7, 2.7))
    else:
        main = inside_rays(sc, 0.85 if sc.name == "degenerate" else 0.75)
    graze = grazing_rays(sc)

    def make(k, rng):
        a, b = main(k, rng), graze(k, rng)
        g = rng.random(k) < 0.25
        return np.where(g[:, None], b[0], a[0]), np.where(g[:, None], b[1], a[1])
    return make


def test_f64_model_against_oracle(po):
    """The float64 model and its bounds against the oracle's FP32 restatement of the hit definition, on a machine without a GPU: rays in
    every small scene (intersect), the find with a non-trivial Tsb from inside and outside the map for every sim option (sensor-frame
    points, flipped normals, miss encoding), closest points, Umeyama.  Also shows the bounds are sharp: the worst errors are real fractions
    of them, and the admissible rays include low incidence angles."""
    from rmcl_b200 import synth
    for name in SMALL:
        sc = scene(name)
        osc = oracle_scene(po, name)
        o, d, ref, redrawn = redraw(sc, make_rays_for(sc), 3000, 1)
        t, f, ng, h = osc.intersect(o, d)
        s = check_hits(sc, ref, np.where(h == 1, t.astype(np.float64), np.inf), f, what=f"oracle intersect {name}")
        log(f"oracle intersect {name}", s, redrawn)
        cosr = np.array([ref["cr"]["cos"][ref["bounds"][r]][ref["cr"]["face"][ref["bounds"][r]] == ref["face"][r]][0] for r in np.flatnonzero(np.isfinite(ref["t"]))])
        assert (cosr < 0.15).sum() >= 20, (name, "low-incidence admissible rays", (cosr < 0.15).sum())
    # the find from inside (no flip needed in the cube) and outside (flip needed), Tsb non-trivial, every sim option
    sc = scene("cube")
    osc = oracle_scene(po, "cube")
    m = synth.SphericalModel(np.radians(-60.0), np.radians(120.0) / 23, 24, -np.pi, 2 * np.pi / 48, 48, 4.0, 12.0)
    o_s, d_s = po.model_rays(m)
    for Tbm in (pose((1.0, -0.5, 0.3), rpy=(0.1, 0.2, 0.3)), pose((15.0, 3.0, 2.0), rpy=(0.0, 0.1, 2.9))):
        for opts in [(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)]:
            out = osc.simulate(Tbm, tsb(), o_s, d_s, m.range_max, m.range_min, *opts)
            s, _ = check_find(sc, out, Tbm, tsb(), o_s, d_s, m.range_min, m.range_max, opts, what=f"oracle find {opts}")
            assert s["hits"] > 100
    log("oracle find (last)", s)
    # closest points
    for name in ("cube", "degenerate", "sphere"):
        sc = scene(name)
        q = cpc_queries(sc, 400, np.random.default_rng(3))
        Tbm = pose((0.3, -0.2, 0.1), rpy=(0.2, -0.1, 0.5))
        R, t = sensor_to_map(Tbm, tsb())
        with np.errstate(invalid="ignore"):
            ps = ((q - t) @ R).astype(np.float32)
        out = oracle_scene(po, name).cpc_find(Tbm, tsb(), ps, 1.0)
        out["ranges"] = out["dists"]
        check_cpc(sc, out, ps, Tbm, tsb(), 1.0, what=f"oracle closest points {name}")
    # Umeyama: the oracle's FP64 SVD of the float32 C
    cases = umeyama_cases(np.random.default_rng(5))
    check_umeyama([po.umeyama(s) for _, s in cases], cases, "oracle umeyama")


def test_intbox_flags_of_constructed_rays():
    """The rays test_intersect_edges builds to run the float box test (far addend exactly +0 with |idir| < 1) are unflagged by ray_setup,
    their unit-direction neighbours are flagged (host harness, the product's ray_setup)."""
    sc = scene("cube")
    o, d = intbox_rays(sc, 64, np.random.default_rng(9))
    fl = intbox_flags(o, d, sc.bmax)
    assert np.array_equal(fl, np.arange(64) % 2 == 0), fl


def intbox_rays(sc, n, rng):
    """n rays, even lanes flagged B2_RAY_INTBOX (unit directions), odd lanes not (|d_x| > 1, far addend +0)"""
    o = rng.uniform(-5, 5, (n, 3)).astype(np.float32)
    d = random_dirs(n, rng)
    for i in range(1, n, 2):
        dd = np.float32(rng.uniform(1.5, 3.0)) * d[i] / np.float32(max(abs(d[i, 0]), 1e-3))
        dd[0] = np.float32(abs(dd[0]))
        d[i] = dd.astype(np.float32)
        o[i, 0], d[i, 0] = unflagged_ray(d[i], sc.bmax, 0)
    return o, d


# ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_intersect_edges():
    """Map.intersect (k_intersect): axis-aligned directions with exact +-0 components, components around the 1e-18 clamp, non-unit
    directions (|d| = 1e-3, 1e3: t in units of |d|), tfar of 0, -0, negative, NaN, denormal, +inf and finite; NaN, inf and zero
    directions (misses); a warp interleaving rays with and without B2_RAY_INTBOX (flags confirmed by the host harness)."""
    for name in ("cube", "degenerate", "sphere"):
        sc = scene(name)
        gm = gpu_map(name)
        base = make_rays_for(sc)

        def axis_rays(k, rng):
            o, _ = base(k, rng)
            d = np.zeros((k, 3), np.float32)
            ax = rng.integers(0, 3, k)
            d[np.arange(k), ax] = rng.choice([-1.0, 1.0], k)
            d[rng.random((k, 3)) < 0.5] *= -1                                         # -0 components
            return o, d

        def clamp_rays(k, rng):
            o, d = base(k, rng)
            c = rng.integers(0, 3, k)
            d[np.arange(k), c] = rng.choice([1e-19, -1e-19, 1e-17, -1e-17, 1e-18, -1e-18], k).astype(np.float32)
            return o, d

        def scaled(s):
            def make(k, rng):
                o, d = base(k, rng)
                return o, (d * np.float32(s)).astype(np.float32)
            return make

        for label, make in (("axis", axis_rays), ("clamp", clamp_rays), ("|d| 1e-3", scaled(1e-3)), ("|d| 1e3", scaled(1e3)), ("random", base)):
            for tfar in (np.inf, 7.5):
                tf = tfar / 1e-3 if label == "|d| 1e-3" and np.isfinite(tfar) else (tfar / 1e3 if label == "|d| 1e3" and np.isfinite(tfar) else tfar)
                tf = float(np.float32(tf))
                o, d, ref, redrawn = redraw(sc, make, 700, hash((name, label)) % 1000, tf)
                t, f, ng, h = gm.intersect(o, d, tf)
                s = check_intersect(sc, ref, t, f, ng, h, tf, f"intersect {name} {label} tfar {tf}")
                log(f"intersect {name} {label} tfar {tf}", s, redrawn)
    # tfar edge values: no hit can have t <= 0, a denormal or NaN tfar
    sc = scene("cube")
    gm = gpu_map("cube")
    o, d, ref, _ = redraw(sc, make_rays_for(sc), 300, 77)
    for tf in (0.0, -0.0, -1.0, np.nan, float(np.float32(1e-40)), np.inf):
        t, f, ng, h = gm.intersect(o, d, tf)
        if np.isinf(tf):
            check_intersect(sc, ref, t, f, ng, h, tf, "tfar inf")
        else:
            assert (h == 0).all() and (f == NOFACE).all() and np.isposinf(t).all() and (ng == 0).all(), tf
    # NaN, inf and zero directions / origins: misses
    bad_o = np.array([[0, 0, 0], [np.nan, 0, 0], [0, np.inf, 0], [1, 2, 3], [1, 2, 3], [1, 2, 3], [1, 2, 3], [0, 0, -np.inf]], np.float32)
    bad_d = np.array([[0, 0, 0], [1, 0, 0], [0, 0, 1], [np.nan, 0, 1], [np.inf, 0, 0], [0, -np.inf, 1], [-0.0, 0, -0.0], [0, 0, 1]], np.float32)
    t, f, ng, h = gm.intersect(bad_o, bad_d)
    assert (h == 0).all() and (f == NOFACE).all() and np.isposinf(t).all() and (ng == 0).all(), (h, f, t)
    # one warp running both box-test instantiations, lane by lane
    for name in ("cube", "degenerate"):
        sc = scene(name)
        rng = np.random.default_rng(31)
        o, d = intbox_rays(sc, 256, rng)
        fl = intbox_flags(o, d, sc.bmax)
        assert np.array_equal(fl, np.arange(256) % 2 == 0), fl
        ref = trace_model(sc, o.astype(np.float64), d.astype(np.float64))
        t, f, ng, h = gpu_map(name).intersect(o, d)
        s = check_intersect(sc, ref, t, f, ng, h, np.inf, f"intbox mixed {name}")
        log(f"intbox mixed {name} (flags confirmed, {int((~ref['adm']).sum())} inadmissible kept)", s)


def check_intersect(sc, ref, t, f, ng, h, tfar, what):
    assert np.array_equal(h == 1, f != NOFACE), what
    miss = h == 0
    assert np.isposinf(t[miss]).all() and (ng[miss] == 0).all(), what
    s = check_hits(sc, ref, np.where(miss, np.inf, t.astype(np.float64)), f, tfar, None, what)
    k = np.flatnonzero(~miss)
    if len(k):
        fk = f[k].astype(np.int64)
        err = np.linalg.norm(ng[k].astype(np.float64) - sc.Ng[fk], axis=1)
        bnd = K_N * U * sc.l1[fk] * sc.l2[fk]
        assert (err <= bnd).all(), (what, "Ng", float((err / bnd).max()))
    s.update(n=len(t), hits=len(k))
    return s


# ----------------------------------------------------------------------------------------------------------------------------------
def rcc(kind, name, m, Tsb=None):
    import rmcl_b200
    cls = dict(spherical=rmcl_b200.RCCB200Spherical, pinhole=rmcl_b200.RCCB200Pinhole, o1dn=rmcl_b200.RCCB200O1Dn, ondn=rmcl_b200.RCCB200OnDn)[kind]
    h = cls(gpu_map(name))
    h.setTsb(tsb() if Tsb is None else Tsb)
    if m is not None:
        h.setModel(m)
    return h


def find_case(h, sc, Tbm, orig_s, range_min, range_max, opts=(0, 0, 0), idx=None, what="", Tsb=None):
    h.setSimOptions(*opts)
    h.find(Tbm)
    out = h.modelView()
    d_s = model_tables(h)
    s, _ = check_find(sc, out, Tbm, tsb() if Tsb is None else Tsb, orig_s, d_s, range_min, range_max, opts, idx=idx, what=what)
    log(what, s)
    return s, out


POSES = [
    ("identity", dict()),
    ("near 180 x", dict(t=(0.5, -0.3, 0.2), q=near_180(0))),
    ("near 180 y", dict(t=(-0.4, 0.6, -0.1), q=near_180(1))),
    ("near 180 z", dict(t=(0.2, 0.1, 0.7), q=near_180(2))),
    ("outside the map", dict(t=(14.0, -3.0, 2.5), rpy=(0.1, -0.05, 2.8))),
]


@pytest.mark.gpu
def test_find_sensor_models():
    """The find through modelView after find() for the spherical, pinhole, O1Dn (from a cloud with invalid points: zero directions) and
    OnDn (per-ray origins) models, at poses identity, near-180-degree rotations about each axis and outside the map's box, on every small
    scene; every setSimOptions combination on the cube (range limits placed so that hits fall below range_min and beyond range_max)."""
    from rmcl_b200 import synth
    import rmcl_b200
    sph = synth.SphericalModel(np.radians(-70.0), np.radians(140.0) / 15, 16, -np.pi, 2 * np.pi / 64, 64, 0.5, 60.0)
    pin = synth.PinholeModel(32, 24, 20.0, 20.0, 15.5, 11.5, 0.5, 60.0)
    for name in SMALL:
        sc = scene(name)
        centre = sc.V.astype(np.float64).mean(0) if name == "indoor" else np.zeros(3)
        for label, p in POSES:
            pp = dict(p)
            pp["t"] = tuple(np.asarray(pp.get("t", (0, 0, 0))) * (sc.E / 10.0) + centre)
            Tbm = pose(**pp)
            for kind, m in (("spherical", sph), ("pinhole", pin)):
                find_case(rcc(kind, name, m), sc, Tbm, np.zeros(3), m.range_min, m.range_max, what=f"{kind} {name} {label}")
        # O1Dn from an organised cloud with NaN points (zero directions), redrawn until every ray is admissible
        Tbm = pose(tuple(centre + [0.3, -0.2, 0.1]), rpy=(0.1, -0.2, 0.4))
        o_s = np.zeros(3)
        rng = np.random.default_rng(11)
        W, H = 24, 16
        dirs = random_dirs(W * H, rng)
        redrawn = 0
        for _ in range(40):
            o_m, d_m, _ = rays_of(Tbm, tsb(), np.zeros((len(dirs), 3)), dirs)
            ref = trace_model(sc, o_m, d_m, float(np.float32(50.0)))
            bad = np.flatnonzero(~ref["adm"])
            if len(bad) == 0:
                break
            redrawn += len(bad)
            dirs[bad] = random_dirs(len(bad), rng)
        assert len(bad) == 0
        pts = dirs.astype(np.float64) * rng.uniform(1.0, 5.0, (len(dirs), 1))
        nan = rng.random(len(dirs)) < 0.1
        pts[nan] = np.nan
        h = rcc("o1dn", name, None)
        h.setPointCloud(synth.pointcloud2(pts, W, H, seed=3), rmcl_b200.O1DnCloudFilter.defaults(0.3, 50.0))
        d_tab = model_tables(h)
        assert (d_tab[nan] == 0).all() and (np.abs(np.linalg.norm(d_tab[~nan], axis=1) - 1) < 1e-6).all()
        h.find(Tbm)
        out = h.modelView()
        assert (out["hits"][nan] == 0).all()
        s, _ = check_find(sc, out, Tbm, tsb(), o_s, d_tab, 0.3, 50.0, what=f"o1dn cloud {name}")
        assert s["inadmissible"] == 0
        log(f"o1dn cloud {name}", s, redrawn)
        # OnDn: per-ray origins
        n = 1000
        os_ = rng.uniform(-0.5, 0.5, (n, 3)).astype(np.float32)
        ds = random_dirs(n, rng)
        redrawn = 0
        for _ in range(40):
            o_m, d_m, _ = rays_of(Tbm, tsb(), os_, ds)
            ref = trace_model(sc, o_m, d_m, float(np.float32(60.0)))
            bad = np.flatnonzero(~ref["adm"])
            if len(bad) == 0:
                break
            redrawn += len(bad)
            os_[bad] = rng.uniform(-0.5, 0.5, (len(bad), 3))
            ds[bad] = random_dirs(len(bad), rng)
        assert len(bad) == 0
        m = synth.OnDnModel(50, 20, os_, ds, 0.5, 60.0)
        h = rcc("ondn", name, m)
        h.find(Tbm)
        s, _ = check_find(sc, h.modelView(), Tbm, tsb(), os_, model_tables(h), 0.5, 60.0, what=f"ondn {name}")
        assert s["inadmissible"] == 0
        log(f"ondn {name}", s, redrawn)
    # every sim option on the cube: range_min 4 and range_max 12 cut the 20 m cube's walls from inside
    sc = scene("cube")
    m = synth.SphericalModel(np.radians(-70.0), np.radians(140.0) / 15, 16, -np.pi, 2 * np.pi / 64, 64, 4.0, 12.0)
    h = rcc("spherical", "cube", m)
    for opts in [(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)]:
        for label, p in POSES[:2] + POSES[-1:]:
            find_case(h, sc, pose(**p), np.zeros(3), 4.0, 12.0, opts, what=f"sim options {opts} {label}")


@pytest.mark.gpu
def test_find_far_and_snapped_origins():
    """Origins 10^3 and 10^4 from the map (a narrow pinhole aimed at it: the bound grows with S), and origins snapped exactly onto vertex
    coordinates, which are also node planes (child boxes are the exact float AABBs of their triangles)."""
    from rmcl_b200 import synth
    for name in ("cube", "indoor"):
        sc = scene(name)
        c = sc.V.astype(np.float64).mean(0)
        for dist in (1e3, 1e4):
            half = 0.8 * sc.E
            fx = 16.0 * dist / half
            m = synth.PinholeModel(32, 32, fx, fx, 15.5, 15.5, 1.0, float(3 * dist))
            for yaw in (0.0, 2.0):
                tpos = c + dist * np.array([-np.cos(yaw), -np.sin(yaw), 0.05])
                Tbm = pose(tuple(tpos), rpy=(0.0, 0.05, yaw))
                find_case(rcc("pinhole", name, m, Tsb=pose()), sc, Tbm, np.zeros(3), m.range_min, m.range_max, what=f"far {dist:g} {name} yaw {yaw}",
                          Tsb=pose())
        # snapped origins: each coordinate a vertex coordinate inside the map
        vx = np.unique(sc.V[:, 0])
        vy = np.unique(sc.V[:, 1])
        vz = np.unique(sc.V[:, 2])
        m = synth.SphericalModel(np.radians(-80.0), np.radians(160.0) / 15, 16, -np.pi, 2 * np.pi / 64, 64, 0.1, 80.0)
        for k in range(3):
            p = (vx[len(vx) // 2 + k - 1], vy[len(vy) // 2 - k], vz[len(vz) // 2])
            find_case(rcc("spherical", name, m, Tsb=pose()), sc, pose(p), np.zeros(3), 0.1, 80.0, what=f"snapped {name} {p}", Tsb=pose())


def find_tickets(h):
    import rmcl_b200
    out = np.zeros(3, np.uint32)
    assert rmcl_b200.load_library().b2_rcc_debug_find_tickets(h._h, None, C.c_void_p(out.ctypes.data)) == 0
    return out


def tile_perm(h):
    import rmcl_b200
    n = C.c_uint32()
    assert rmcl_b200.load_library().b2_rcc_debug_tile_perm(h._h, None, 0, C.byref(n)) == 0
    return n.value


def sample_idx(n, rng, k=1500):
    """the rays of the first two and the last two tiles, and a random sample"""
    edge = np.concatenate([np.arange(min(n, 64)), np.arange(max(0, n - 64), n)])
    return np.unique(np.concatenate([edge, rng.choice(n, min(n, k), replace=False)]))


@pytest.mark.gpu
def test_find_launch_shapes():
    """Ray counts 1, 31, 32, 33; one 8x4 tile; rasters whose width / height are not multiples of 8 / 4 (raster order); tile counts just
    below and above the resident wave (read back from the launch's grid); more than 11 520 tiles (raster order, no schedule); a find after
    correctOnce on the same handle (runs with the tile schedule the ICP loop sorted).  Large cases compare the first and last tiles and a
    random sample with the model."""
    from rmcl_b200 import synth
    sc = scene("cube")
    Tbm = pose((0.7, -1.1, 0.4), rpy=(0.2, -0.1, 0.6))
    rng = np.random.default_rng(21)

    def sph(rows, cols, rmin=0.3, rmax=40.0):
        return synth.SphericalModel(np.radians(-75.0), np.radians(150.0) / max(rows - 1, 1), rows, -np.pi + 0.01, 2 * np.pi / cols, cols, rmin, rmax)

    for rows, cols in ((1, 1), (1, 31), (1, 32), (1, 33), (4, 8), (7, 12), (6, 16), (5, 13), (8, 24)):
        h = rcc("spherical", "cube", sph(rows, cols))
        find_case(h, sc, Tbm, np.zeros(3), 0.3, 40.0, what=f"raster {rows}x{cols}")
    # the resident wave: a large launch's grid is the wave (blocks of two warps, one tile each)
    big = PERM_MAX_TILES + 1
    h = rcc("spherical", "cube", sph(4, 8 * big))
    h.find(Tbm)
    assert tile_perm(h) == 0                                                          # beyond the schedule's tile count: raster order
    grid = int(find_tickets(h)[2])
    wave = grid * (FIND_BLOCK // 32)
    assert big > wave > 100, (grid, wave)
    find_case(h, sc, Tbm, np.zeros(3), 0.3, 40.0, idx=sample_idx(32 * big, rng), what=f"{big} tiles (wave {wave})")
    for n_tiles in (wave - 1, wave + 1):
        h = rcc("spherical", "cube", sph(4, 8 * n_tiles))
        find_case(h, sc, Tbm, np.zeros(3), 0.3, 40.0, idx=sample_idx(32 * n_tiles, rng), what=f"{n_tiles} tiles")
        assert int(find_tickets(h)[2]) == min(grid, -(-n_tiles // 2))
    # the tile schedule: a find after correctOnce on the same handle
    m = sph(32, 64)
    h = rcc("spherical", "cube", m)
    s0, out0 = find_case(h, sc, Tbm, np.zeros(3), m.range_min, m.range_max, what="before correctOnce")
    ranges = np.where(out0["hits"] == 1, out0["ranges"], np.float32(m.range_max + 1)).astype(np.float32)
    h.setParams(1.0, 0.15)
    h.correctOnce(synth.compose(Tbm, pose((0.02, -0.01, 0.0), rpy=(0, 0, 0.01))), pose(), 3, 0.0, ranges=ranges)
    assert tile_perm(h) == m.size // 32
    s1, out1 = find_case(h, sc, Tbm, np.zeros(3), m.range_min, m.range_max, what="after correctOnce (tile schedule)")
    for k in ("points", "normals", "hits", "face_ids", "ranges"):
        assert out0[k].tobytes() == out1[k].tobytes(), k


@pytest.mark.gpu
def test_find_large_map():
    """building:200000 seen by a C2-sized spherical scan (128 x 1024) from a pose inside the building: a random subset of 3000 rays and the
    first and last tiles against the model (faces culled by float64 group boxes padded by 10^-3 (1 + E), so no crossing is lost)."""
    from rmcl_b200 import synth
    sc = scene("building")
    m = synth.c2_sensor()
    Tbm = synth.compose(synth.building_gt_pose(), pose((0.13, -0.07, 0.0), rpy=(0.0, 0.0, 0.2)))
    h = rcc("spherical", "building", m, Tsb=synth.scenario_tsb())
    rng = np.random.default_rng(41)
    s, _ = find_case(h, sc, Tbm, np.zeros(3), m.range_min, m.range_max, idx=sample_idx(m.size, rng, 3000), what="building C2 subset",
                     Tsb=synth.scenario_tsb())
    assert s["hits"] > 2000


@pytest.mark.gpu
def test_cpc_find_edges():
    """Closest points (CPCB200.find, k_cpc_find): queries on faces, edges and vertices, the cube's centre, 10^3 outside the map, NaN / inf;
    point counts 1, 63, 64, 65, 64 k - 1, 64 k + 1; skip_masked off and on."""
    import rmcl_b200
    for name in ("cube", "degenerate", "sphere"):
        sc = scene(name)
        Tbm = pose((0.3, -0.2, 0.1), rpy=(0.2, -0.1, 0.5))
        R, t = sensor_to_map(Tbm, tsb())
        rng = np.random.default_rng(13)
        for n in (1, 63, 64, 65, 64 * 17 - 1, 64 * 17 + 1):
            q = cpc_queries(sc, n, rng)
            with np.errstate(invalid="ignore"):
                ps = ((q - t) @ R).astype(np.float32)
            mask = (rng.random(n) < 0.8).astype(np.uint8)
            for skip in (False, True):
                h = rmcl_b200.CPCB200(gpu_map(name))
                h.setTsb(tsb())
                h.setParams(1.0, 0.15)
                h.setDataset(ps, mask)
                h.setOptions(skip_masked=skip)
                h.find(Tbm)
                check_cpc(sc, h.modelView(), ps, Tbm, tsb(), 1.0, mask, skip, f"closest points {name} n {n} skip_masked {skip}")


@pytest.mark.gpu
def test_umeyama_device():
    """umeyama_transform (k_umeyama_batch, block 64) at batch sizes 1, 63, 64, 65 and on the whole case list: random rotations, C scaled
    from 10^-20 to 10^20 (the fro > 1e-30 cut-off, FTZ inputs, FP32 overflow of the Frobenius sum), s3 = +-1e-2, 1e-4, 1e-7 s1 on both
    sides of det C = 0, rank 2, rank 1, n_meas = 0, means of magnitude 10^4, the near-SPD ICP case."""
    import rmcl_b200
    cases = umeyama_cases(np.random.default_rng(5))
    stats = np.array([s for _, s in cases])
    check_umeyama(rmcl_b200.umeyama_transform(stats), cases, f"umeyama {len(cases)}")
    for n in (1, 63, 64, 65):
        idx = np.arange(n) % len(cases)
        sub = [cases[i] for i in idx]
        out = rmcl_b200.umeyama_transform(stats[idx])
        check_umeyama(out, sub, f"umeyama batch {n}")
    print(f"test file wall time so far {time.time() - _T0:.1f} s")
