"""The particle filter's sensor update (k_pf_update<CORR, MAP>) and its likelihood statistics (k_pf_residual_stats) at the edges of their launch
geometry, against a float64 restatement of the same operations.

The oracle restates the device's FP32 arithmetic op for op, so a mistake shared by both in the Gaussian evaluation stays invisible to it, and
it cannot see what exists only on the GPU: particles per block (ppb) and the partial last block, the lanes = beams / lanes = particles
mappings and the particle order of the sorted one, the direction sort of the beam table and its back-permutation into the shared tile, the
chunks of the two-stream host path, the grid-stride statistics.  Here a plain numpy float64 model (brute-force Moller-Trumbore and
point-to-triangle distance over a small non-convex scene, the Gaussian1D merge in the caller's beam order) checks every case, and the launch
shape the library reports (b2_pf_debug_launch_geometry) shows that each case hit the regime it was placed on.  Merge order is invisible to a
float64 model (the exact running mean does not depend on it), so every case is also compared with the oracle on the same caller order.

Admissible inputs instead of loose tolerances: a (particle, beam) pair whose float64 hit lies within EDGE_MARGIN of an edge of a triangle at or
before the closest hit (measured across the ray: the distance times |cos| of the incidence), or whose hit distance lies within EDGE_MARGIN of
range_min (again times |cos|), may legitimately change its answer under an FP32 rounding.  Each case redraws the particles owning such a pair
(where a few particles carry thousands of beams, the beams instead) and asserts that none remains.  Closest-point errors are continuous in the query point and need no margin.

Tolerances (float64 model vs FP32 device, u = 2^-24):
  n_meas    exact
  L (pair)  dL = max |dL/de| over [e - de, e + de] * de + (8 |arg| + 8) u L, where de = K_ERR u S |n| bounds the FP32 error of the error
            term (S = |origin| + max(t, range) + 1 in the map frame, |n| = |Ng| for ng_mode 0, 1 for ng_mode 1; closest points:
            S = |origin| + range + SCENE_EXTENT, |n| = 1) and arg = -e^2 / (2 sigma^2); penalty branches are exact up to the exp term
  mean      running merge bound next to the float64 merge: err_k <= w1 err_{k-1} + w2 dL_k + 4 u (|mean_{k-1}| + |mean_k| + |L_k|); it
            saturates near 10^4 u max L once the clamp holds n_meas at 10 000
  sigma     the same kind of bound through d1 = mean_{k-1} - mean_k and d2 = L_k - mean_k
Against the oracle (same FP32 formulas; the device's exp() and glibc's may differ in the last double bit before the rounding to float):
n_meas exact, mean and sigma within TOL_LIK * max(1, |value|), more than 99 % of the means bit-identical.
The CPU test at the top checks the model itself against the oracle, pair by pair and merged, within these bounds.
"""
import ctypes as C

import numpy as np
import pytest

U = 2.0 ** -24
K_ERR = 8.0
EDGE_MARGIN = 1e-4
TOL_LIK = 2e-6
SCENE_EXTENT = 20.0
MAX_N_MEAS = 10000
PF_BLOCK = 128                 # threads per k_pf_update block
B2_ERR_UNSUPPORTED = -5
CHUNKED_FROM = 32768           # b2_pf_sensor_update_host cuts the particles into 8 chunks from here on
AUTO_SORT_FROM = 4096          # mapping 3 considers the sorted mapping from here on
GEOM_KEYS = ("smem_optin", "map_req", "map", "kmap", "sorted", "ppb", "blocks", "smem", "n_chunks", "per", "n", "n_beams")

# dist_sigma, real_hit_sim_miss_error, real_miss_sim_hit_error, real_miss_sim_miss_error, range_min, range_max
PRM = (0.25, 0.3, 0.4, 0.2, 1.0, 40.0)
PRM_SHARP = (0.05,) + PRM[1:]
COMBOS = [(0, 0), (0, 1), (1, 0)]          # (correspondence type, ng_mode)


# =====================================================================================================================================
# scene: a 20 m cube (coarse walls and ceiling, a floor grid of unequal cells), one free-standing box inside
# =====================================================================================================================================
def _rect(origin, eu, ev, us, vs):
    """origin + s eu + t ev over the breakpoints us x vs (in [0, 1]), two triangles per cell"""
    o, eu, ev = (np.asarray(a, np.float64) for a in (origin, eu, ev))
    S, T = np.meshgrid(np.asarray(us, np.float64), np.asarray(vs, np.float64), indexing="xy")
    V = (o + S[..., None] * eu + T[..., None] * ev).reshape(-1, 3)
    nu = len(us)
    j, i = np.meshgrid(np.arange(len(vs) - 1), np.arange(nu - 1), indexing="ij")
    a = (j * nu + i).ravel()
    F = np.concatenate([np.stack([a, a + 1, a + nu + 1], 1), np.stack([a, a + nu + 1, a + nu], 1)])
    return V, F


def scene_mesh():
    g4, g2 = np.linspace(0, 1, 5), np.linspace(0, 1, 3)
    parts = [
        _rect((-10, -10, -10), (20, 0, 0), (0, 20, 0), np.linspace(0, 1, 9) ** 1.6, np.linspace(0, 1, 8) ** 0.7),   # floor, unequal cells
        _rect((-10, -10, 10), (0, 20, 0), (20, 0, 0), g4, g4),
        _rect((-10, -10, -10), (0, 0, 20), (20, 0, 0), g4, g4),
        _rect((-10, 10, -10), (20, 0, 0), (0, 0, 20), g4, g4),
        _rect((-10, -10, -10), (0, 20, 0), (0, 0, 20), g4, g4),
        _rect((10, -10, -10), (0, 0, 20), (0, 20, 0), g4, g4),
    ]
    lo, hi = np.array([2.0, -4.0, -7.0]), np.array([5.0, -1.0, -3.0])
    dx, dy, dz = hi - lo
    parts += [_rect(lo, (dx, 0, 0), (0, dy, 0), g2, g2), _rect((lo[0], lo[1], hi[2]), (dx, 0, 0), (0, dy, 0), g2, g2),
              _rect(lo, (dx, 0, 0), (0, 0, dz), g2, g2), _rect((lo[0], hi[1], lo[2]), (dx, 0, 0), (0, 0, dz), g2, g2),
              _rect(lo, (0, dy, 0), (0, 0, dz), g2, g2), _rect((hi[0], lo[1], lo[2]), (0, dy, 0), (0, 0, dz), g2, g2)]
    vs, fs, off = [], [], 0
    for V, F in parts:
        vs.append(V)
        fs.append(F + off)
        off += len(V)
    return np.concatenate(vs).astype(np.float32), np.concatenate(fs).astype(np.uint32)


_S = {}


def scene():
    if "V" not in _S:
        V, F = scene_mesh()
        v = V.astype(np.float64)
        v0, v1, v2 = v[F[:, 0]], v[F[:, 1]], v[F[:, 2]]
        e1, e2 = v1 - v0, v2 - v0
        Ng = np.cross(e1, e2)
        nn = np.linalg.norm(Ng, axis=1)
        _S.update(V=V, F=F, v0=v0, v1=v1, v2=v2, e1=e1, e2=e2, Ng=Ng, nNg=nn, l0=np.linalg.norm(v2 - v1, axis=1), l1=np.linalg.norm(e2, axis=1),
                  l2=np.linalg.norm(e1, axis=1))
    return _S


def oracle_pf(po):
    if "osc" not in _S:
        s = scene()
        _S["osc"] = po.Scene(s["V"], s["F"])
    return _S["osc"]


def gpu_scene():
    import rmcl_b200
    if "map" not in _S:
        s = scene()
        _S["map"] = rmcl_b200.Map(s["V"], s["F"], device=0)
    return _S["map"]


# =====================================================================================================================================
# float64 reference: evaluate_rcc / evaluate_cpc / sensorUpdate up to `eval` (PCDSensorUpdaterEmbree.cpp:18-95, 197-224), the Gaussian1D
# merge with its MAX_N_MEAS clamp, compute_stats (resampling.cu:41-92)
# =====================================================================================================================================
def qmul(a, b):
    ax, ay, az, aw = np.moveaxis(a, -1, 0)
    bx, by, bz, bw = np.moveaxis(b, -1, 0)
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], -1)


def qrot(q, v):
    """q v q* (the Hamilton form of the transform's rotation, on the stored quaternion as it is)"""
    p = np.concatenate([v, np.zeros(v.shape[:-1] + (1,))], -1)
    return qmul(qmul(q, p), q * np.array([-1.0, -1.0, -1.0, 1.0]))[..., :3]


def rays_in_map(P, Tsb, B):
    """T_sm = pose * Tsb; beam origins and directions in the map frame: (n, nb, 3) each"""
    qp, tp = P["R"].astype(np.float64), P["t"].astype(np.float64)
    qs, ts = np.asarray(Tsb["R"], np.float64), np.asarray(Tsb["t"], np.float64)
    q = qmul(qp, np.broadcast_to(qs, qp.shape))
    t = qrot(qp, np.broadcast_to(ts, tp.shape)) + tp
    qb = np.broadcast_to(q[:, None, :], (len(P), len(B), 4))
    o = qrot(qb, np.broadcast_to(B["orig"].astype(np.float64), (len(P), len(B), 3))) + t[:, None, :]
    d = qrot(qb, np.broadcast_to(B["dir"].astype(np.float64), (len(P), len(B), 3)))
    return o, d


def trace(o, d, range_min, chunk=1024):
    """brute-force closest hit (t > 0) over all triangles -> t (inf: none), face, |cos| of the incidence, ambiguous flag"""
    s = scene()
    m = len(o)
    tb, fb, cb, amb = np.full(m, np.inf), np.zeros(m, np.int64), np.ones(m), np.zeros(m, bool)
    e1, e2, v0, Ng, nNg = s["e1"], s["e2"], s["v0"], s["Ng"], s["nNg"]
    for a in range(0, m, chunk):
        oo, dd = o[a:a + chunk, None, :], d[a:a + chunk, None, :]
        pv = np.cross(dd, e2)
        det = np.einsum("rtk,tk->rt", pv, e1)
        with np.errstate(divide="ignore", invalid="ignore"):
            tv = oo - v0
            Uu = np.einsum("rtk,rtk->rt", tv, pv) / det
            qv = np.cross(tv, e1)
            Vv = np.einsum("rtk,rtk->rt", np.broadcast_to(dd, qv.shape), qv) / det
            t = np.einsum("tk,rtk->rt", e2, qv) / det
            W = 1.0 - Uu - Vv
            ed = np.minimum(np.minimum(W * nNg / s["l0"], Uu * nNg / s["l1"]), Vv * nNg / s["l2"])     # signed distance to the nearest edge
            cos = np.abs(np.einsum("rtk,tk->rt", np.broadcast_to(dd, (dd.shape[0], len(Ng), 3)), Ng)) / (nNg * np.linalg.norm(dd, axis=-1))
        ok = np.isfinite(t) & (t > 0) & (ed >= 0)
        tt = np.where(ok, t, np.inf)
        f = np.argmin(tt, axis=1)                                                          # ties: smallest face id
        r = np.arange(len(f))
        best = tt[r, f]
        near = np.isfinite(t) & (t > 0) & (t <= best[:, None] * (1 + 1e-6) + EDGE_MARGIN) & (np.abs(ed) * cos < EDGE_MARGIN)
        c = cos[r, f]
        amb[a:a + chunk] = near.any(1) | (np.isfinite(best) & (np.abs(best - range_min) * c < EDGE_MARGIN))
        tb[a:a + chunk], fb[a:a + chunk], cb[a:a + chunk] = best, f, c
    return tb, fb, cb, amb


def point_mesh_distance(q, chunk=1024):
    """float64 distance of each point to the nearest triangle (plane distance inside, nearest edge segment outside)"""
    s = scene()
    v0, v1, v2, Ng, nNg = s["v0"], s["v1"], s["v2"], s["Ng"], s["nNg"]
    nrm = Ng / nNg[:, None]
    out = np.empty(len(q))

    def seg(p, a, b):
        ab = b - a
        w = np.clip(np.einsum("rtk,tk->rt", p - a, ab) / np.einsum("tk,tk->t", ab, ab), 0.0, 1.0)
        return np.linalg.norm(p - (a + w[..., None] * ab), axis=-1)

    for a in range(0, len(q), chunk):
        p = q[a:a + chunk, None, :]
        h = np.einsum("rtk,tk->rt", p - v0, nrm)
        x = p - h[..., None] * nrm
        c0 = np.einsum("rtk,tk->rt", np.cross(v1 - v0, x - v0), nrm)
        c1 = np.einsum("rtk,tk->rt", np.cross(v2 - v1, x - v1), nrm)
        c2 = np.einsum("rtk,tk->rt", np.cross(v0 - v2, x - v2), nrm)
        inside = ((c0 >= 0) & (c1 >= 0) & (c2 >= 0)) | ((c0 <= 0) & (c1 <= 0) & (c2 <= 0))
        dist = np.where(inside, np.abs(h), np.minimum(np.minimum(seg(p, v0, v1), seg(p, v1, v2)), seg(p, v2, v0)))
        out[a:a + chunk] = dist.min(1)
    return out


def evaluate(P, Tsb, B, prm, corr, ng_mode):
    """per (particle, beam): L (float64), its FP32 error bound dL, ambiguous flags, and the count of pairs with 0 < t <= range_min"""
    sigma, rhsm, rmsh, rmsm, rmin, rmax = (np.float64(np.float32(x)) for x in prm)
    o, d = rays_in_map(P, Tsb, B)
    n, nb = len(P), len(B)
    o, d = o.reshape(-1, 3), d.reshape(-1, 3)
    r = np.broadcast_to(B["range"].astype(np.float64), (n, nb)).reshape(-1)
    amb = np.zeros(n * nb, bool)
    short = 0
    if corr == 1:
        qp = o + d * r[:, None]
        e = point_mesh_distance(qp)
        de = K_ERR * U * (np.linalg.norm(o, axis=1) + r + SCENE_EXTENT)
    else:
        s = scene()
        t, f, _, amb = trace(o, d, rmin)
        real = (np.float32(rmin) <= B["range"]) & (B["range"] <= np.float32(rmax))
        real = np.broadcast_to(real, (n, nb)).reshape(-1)
        sim = np.isfinite(t) & (t > rmin)
        short = int((np.isfinite(t) & (t > 0) & (t <= rmin)).sum())
        Ng = s["Ng"][f]
        nn = s["nNg"][f]
        if ng_mode == 1:
            Ng, nn = Ng / nn[:, None], np.ones_like(nn)
        tt = np.where(np.isfinite(t), t, 0.0)
        err = np.abs(np.einsum("rk,rk->r", (o + d * tt[:, None]) - (o + d * r[:, None]), Ng))
        e = np.where(sim, np.where(real, err, rmsh), np.where(real, rhsm, rmsm))
        de = np.where(sim & real, K_ERR * U * (np.linalg.norm(o, axis=1) + np.maximum(tt, r) + 1.0) * nn, 0.0)
    arg = -e * e / (2 * sigma * sigma)
    L = np.exp(arg) / np.sqrt(2 * np.pi * sigma * sigma)
    lo = np.maximum(e - de, 0.0)
    slope = (e + de) / (sigma * sigma) * np.exp(-lo * lo / (2 * sigma * sigma)) / np.sqrt(2 * np.pi * sigma * sigma)
    dL = slope * de + (8 * np.abs(arg) + 8) * U * L
    return dict(L=L.reshape(n, nb), dL=dL.reshape(n, nb), amb=amb.reshape(n, nb), short=short)


def merge(A0, L, dL):
    """Gaussian1D += {L_k, 0, 1} over the beams in the caller's order with the per-add clamp, float64, and the FP32 bounds"""
    lk = A0["likelihood"]
    mean, sig, nm = lk["mean"].astype(np.float64), lk["sigma"].astype(np.float64), lk["n_meas"].astype(np.int64)
    em, es = np.zeros(len(A0)), np.zeros(len(A0))
    for k in range(L.shape[1]):
        Lk, dk = L[:, k], dL[:, k]
        n1 = nm + 1
        w1, w2 = nm / n1, 1.0 / n1
        m2 = mean * w1 + Lk * w2
        d1, d2 = mean - m2, Lk - m2
        s2 = sig * w1 + (d1 * d1 * w1 + d2 * d2 * w2)
        em2 = w1 * em + w2 * dk + 4 * U * (np.abs(mean) + np.abs(m2) + np.abs(Lk))
        dd1 = em + em2 + 2 * U * np.abs(d1)
        dd2 = dk + em2 + 2 * U * np.abs(d2)
        es = w1 * es + w1 * (2 * np.abs(d1) * dd1 + dd1 * dd1) + w2 * (2 * np.abs(d2) * dd2 + dd2 * dd2) + 8 * U * (s2 + sig * w1 + d1 * d1 * w1 + d2 * d2 * w2)
        mean, sig, em, nm = m2, s2, em2, np.minimum(n1, MAX_N_MEAS)
    return dict(mean=mean, sigma=sig, n_meas=nm, em=em, es=es)


def model(P, A0, Tsb, B, prm, corr, ng_mode):
    ev = evaluate(P, Tsb, B, prm, corr, ng_mode)
    out = merge(A0, ev["L"], ev["dL"])
    out.update(amb=ev["amb"], short=ev["short"], L=ev["L"])
    return out


def take(ref, idx):
    """the model's per-particle results for particles repeated by index"""
    return {k: (v[idx] if isinstance(v, np.ndarray) else v) for k, v in ref.items()}


def stats_f64(A):
    L = A["likelihood"]["mean"].astype(np.float64)
    return float(L.sum()), float(max(0.0, L.max())) if len(L) else 0.0


# =====================================================================================================================================
# inputs
# =====================================================================================================================================
def tsb():
    from rmcl_b200 import synth
    return synth.make_transform((0.2, -0.05, 0.5), (0.02, -0.03, 0.17))


SCAN_POSE = dict(t=(0.95, -2.4, -5.5), yaw=0.3)     # sensor ~0.8 m in front of the box: some beams end closer than range_min


def beams(n, seed, penalties=True, dup=0):
    """n beams seen from the scan pose: random directions (sensor frame), small origins on a third of them, ranges = float64 hit distance
    + N(0, 0.03); a few out of [range_min, range_max] (real misses); `dup` of them repeat earlier directions (direction-sort ties)"""
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    B = np.zeros(n, synth.RANGE_MEAS_DTYPE)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    if dup:
        d[n - dup:] = d[rng.integers(0, n - dup, dup)]
    B["dir"] = d.astype(np.float32)
    B["orig"][: n // 3] = rng.uniform(-0.05, 0.05, (n // 3, 3)).astype(np.float32)
    P0 = scan_particles(1)
    o, dm = rays_in_map(P0, tsb(), B)
    t, _, _, _ = trace(o[0], dm[0], PRM[4])
    B["range"] = (np.where(np.isfinite(t), t, 5.0) + rng.normal(0, 0.03, n)).astype(np.float32)
    if penalties and n >= 8:
        B["range"][rng.choice(n, max(1, n // 40), replace=False)] = np.float32(0.5)
        B["range"][rng.choice(n, max(1, n // 40), replace=False)] = np.float32(60.0)
        B["range"][0] = np.float32(PRM[4])                              # exactly on range_min / range_max: exact float32 comparisons
        B["range"][1] = np.float32(PRM[5])
    B["cov"][:, [0, 4, 8]] = 0.1
    return B


def scan_particles(n, seed=0, spread=0.0, yaw_spread=0.0):
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    P = synth.transforms(n)
    P["t"] = (np.asarray(SCAN_POSE["t"]) + rng.uniform(-spread, spread, (n, 3))).astype(np.float32)
    yaw = SCAN_POSE["yaw"] + rng.uniform(-yaw_spread, yaw_spread, n)
    P["R"][:, 2] = np.sin(yaw / 2).astype(np.float32)
    P["R"][:, 3] = np.cos(yaw / 2).astype(np.float32)
    return P


def admissible(P, B, seed, spread, yaw_spread, corr=0):
    """redraw every particle that owns an ambiguous pair until none is left"""
    if corr == 1:
        return P
    rng = np.random.default_rng(seed + 1000)
    for _ in range(50):
        o, d = rays_in_map(P, tsb(), B)
        _, _, _, amb = trace(o.reshape(-1, 3), d.reshape(-1, 3), PRM[4])
        bad = np.flatnonzero(amb.reshape(len(P), len(B)).any(1))
        if len(bad) == 0:
            return P
        P[bad] = scan_particles(len(bad), int(rng.integers(1 << 30)), spread, yaw_spread)
    raise AssertionError("could not draw admissible particles")


def admissible_beams(P, B, seed):
    """for a few particles with thousands of beams (where nearly every particle owns some ambiguous pair): redraw the beams instead"""
    rng = np.random.default_rng(seed + 2000)
    B = B.copy()
    for _ in range(50):
        o, d = rays_in_map(P, tsb(), B)
        _, _, _, amb = trace(o.reshape(-1, 3), d.reshape(-1, 3), PRM[4])
        bad = np.flatnonzero(amb.reshape(len(P), len(B)).any(0))
        if len(bad) == 0:
            return B
        B[bad] = beams(len(bad), int(rng.integers(1 << 30)), penalties=False)
    raise AssertionError("could not draw admissible beams")


def attrs(n, n_meas=0, mean=1.0):
    from rmcl_b200 import synth
    A = np.zeros(n, synth.PARTICLE_ATTR_DTYPE)
    A["likelihood"]["mean"] = mean
    A["likelihood"]["n_meas"] = n_meas
    A["state_sigma"] = 0.1
    return A


def params(prm, corr, ng_mode, oracle=None):
    import rmcl_b200
    cls = oracle.PFParams if oracle is not None else rmcl_b200.PFParams
    return cls(*prm, ng_mode, corr)


# =====================================================================================================================================
# comparisons
# =====================================================================================================================================
def assert_model(out, ref, what=""):
    """device (or oracle) attrs vs the float64 model and its bounds"""
    assert not ref["amb"].any(), (what, "ambiguous pairs left in the case's inputs")
    lk = out["likelihood"]
    assert np.array_equal(lk["n_meas"].astype(np.int64), ref["n_meas"]), what
    dm = np.abs(lk["mean"].astype(np.float64) - ref["mean"])
    ds = np.abs(lk["sigma"].astype(np.float64) - ref["sigma"])
    assert (dm <= ref["em"]).all(), (what, "mean", float((dm / ref["em"]).max()), int(np.argmax(dm - ref["em"])))
    assert (ds <= ref["es"]).all(), (what, "sigma", float((ds / ref["es"]).max()), int(np.argmax(ds - ref["es"])))


def assert_oracle(out, ref, what=""):
    a, b = out["likelihood"], ref["likelihood"]
    assert np.array_equal(a["n_meas"], b["n_meas"]), what
    for k in ("mean", "sigma"):
        x, y = a[k].astype(np.float64), b[k].astype(np.float64)
        assert (np.abs(x - y) <= TOL_LIK * np.maximum(1.0, np.abs(y))).all(), (what, k, float(np.abs(x - y).max()))
    assert np.mean(a["mean"] == b["mean"]) > 0.99, (what, float(np.mean(a["mean"] == b["mean"])))
    assert np.array_equal(out["state_sigma"], ref["state_sigma"]), what


def geometry(up):
    import rmcl_b200
    out = np.zeros(len(GEOM_KEYS), np.uint32)
    assert rmcl_b200.load_library().b2_pf_debug_launch_geometry(up._h, C.c_void_p(out.ctypes.data)) == 0
    return dict(zip(GEOM_KEYS, map(int, out)))


def expected_ppb(n_beams, smem_optin):
    """pf_prepare_beams: min(smem_optin / (4 n_beams), 64, ceil(8 * 128 / n_beams)), at least 1"""
    return max(1, min(smem_optin // (4 * n_beams), 64, -(-8 * PF_BLOCK // n_beams)))


def log(what, g):
    print(f"{what}: ppb {g['ppb']} map {g['map_req']}->{g['map']} kernel MAP {g['kmap']} sorted {g['sorted']} blocks {g['blocks']} smem {g['smem']} "
          f"chunks {g['n_chunks']} per {g['per']} (n {g['n']}, beams {g['n_beams']})")


def to_dev(P, A):
    import torch
    return (torch.from_numpy(P.view(np.float32).reshape(-1, 8).copy()).cuda(), torch.from_numpy(A.view(np.float32).reshape(-1, 9).copy()).cuda())


def from_dev(Ad):
    import torch
    from rmcl_b200 import synth
    torch.cuda.synchronize()
    return Ad.cpu().numpy().view(synth.PARTICLE_ATTR_DTYPE).reshape(-1)


def update_dev(up, P, A, B, prm):
    Pd, Ad = to_dev(P, A)
    up.update(Pd, Ad, tsb(), B, prm)
    return from_dev(Ad)


def updater(mapping=None):
    import rmcl_b200
    up = rmcl_b200.PCDSensorUpdaterB200(gpu_scene())
    if mapping is not None:
        up.setMapping(mapping)
    return up


def smem_optin():
    up = updater(0)
    P, A = scan_particles(1), attrs(1)
    B = beams(1, 1)
    update_dev(up, P, A, B, params(PRM, 0, 0))
    return geometry(up)["smem_optin"]


def check_case(po, up, P, A, B, prm, corr, ng_mode, what, device=True, f64=True, oracle=True):
    """run the update (device-resident or host arrays), compare with the float64 model and the oracle; -> (attrs, launch shape)"""
    p = params(prm, corr, ng_mode)
    out = update_dev(up, P, A, B, p) if device else up.update(P, A, tsb(), B, p)
    g = geometry(up)
    log(what, g)
    if f64:
        assert_model(out, model(P, A, tsb(), B, prm, corr, ng_mode), what)
    if oracle:
        assert_oracle(out, oracle_pf(po).pf_update(P, A, tsb(), B, params(prm, corr, ng_mode, po)), what)
    return out, g


# =====================================================================================================================================
# tests
# =====================================================================================================================================
@pytest.mark.parametrize("corr,ng_mode", COMBOS)
def test_f64_model_against_oracle(po, corr, ng_mode):
    """The float64 model itself, against the oracle's FP32 restatement on the same scene: pair by pair (one beam per call, so the merged mean
    is the evaluation) within dL, and merged over 180 beams within the merge bounds, at both dist_sigma values; the statistics within
    their FP32 summation bound.  Runs without a GPU, so the yardstick of the GPU tests below is checked rather than assumed."""
    osc = oracle_pf(po)
    B = beams(180, 3)
    for prm, spread in ((PRM, 0.3), (PRM_SHARP, 0.1)):
        P = admissible(scan_particles(200, 5, spread, 0.05), B, 5, spread, 0.05, corr)
        A = attrs(200)
        ev = evaluate(P, tsb(), B, prm, corr, ng_mode)
        assert not ev["amb"].any()
        if corr == 0:
            assert ev["short"] > 0                                             # pairs with 0 < t <= range_min exist (the sim-miss branch)
        for k in range(0, 180, 9):
            o = osc.pf_update(P, A, tsb(), B[k:k + 1], params(prm, corr, ng_mode, po))["likelihood"]["mean"].astype(np.float64)
            assert (np.abs(o - ev["L"][:, k]) <= ev["dL"][:, k] + TOL_LIK * np.maximum(1.0, ev["L"][:, k])).all(), (prm, k)
        ref = merge(A, ev["L"], ev["dL"])
        ref.update(amb=ev["amb"])
        assert_model(osc.pf_update(P, A, tsb(), B, params(prm, corr, ng_mode, po)), ref, f"merged {prm[0]}")
        # sensitivity of the comparison: the merged mean varies between particles far more than the tolerance
        assert ref["mean"].std() >= 100 * ref["em"].max(), (ref["mean"].std(), ref["em"].max())
    # the clamp crossed in the middle of the merge
    A = attrs(200, 9990, 0.7)
    P = admissible(scan_particles(200, 6, 0.3, 0.05), B, 6, 0.3, 0.05, corr)
    assert_model(osc.pf_update(P, A, tsb(), B, params(PRM, corr, ng_mode, po)), model(P, A, tsb(), B, PRM, corr, ng_mode), "clamp")
    # statistics: float64 sum against the oracle's FP32 tree sum
    rng = np.random.default_rng(2)
    A = attrs(100_000)
    A["likelihood"]["mean"] = rng.uniform(0, 1.6, len(A)).astype(np.float32)
    s, m = po.pf_likelihood_stats(A)
    sr, mr = stats_f64(A)
    assert m == mr and abs(s - sr) <= (len(A) / 512 + 12) * U * sr


@pytest.mark.gpu
@pytest.mark.parametrize("corr,ng_mode", COMBOS)
def test_pf_beam_count_regimes(po, corr, ng_mode):
    """Beam counts on every boundary of particles-per-block (1, 16 | 17, 512 | 513, 1024 | 1025), the C3 count (180), the last count at which
    the lanes = particles mapping fits in shared memory and one more (it falls back to lanes = beams), the last count the update accepts and
    one more (refused with B2_ERR_UNSUPPORTED, attrs untouched, no pending CUDA error).  Mappings 0 and 1, results bit-identical."""
    import rmcl_b200
    optin = smem_optin()
    t_map1, t_refuse = optin // (4 * 32), optin // 4
    counts = [1, 16, 17, 180, 512, 513, 1024, 1025, t_map1, t_map1 + 1, t_refuse]
    ups = [updater(0), updater(1)]
    for i, nb in enumerate(counts):
        B = beams(nb, 100 + i)
        ppb = expected_ppb(nb, optin)
        n = 2 * ppb + 1 if nb < 4096 else 3
        if nb <= 1024:
            P = admissible(scan_particles(n, 200 + i, 0.3, 0.05), B, 200 + i, 0.3, 0.05, corr)
        else:
            P = scan_particles(n, 200 + i, 0.3, 0.05)
            B = B if corr == 1 else admissible_beams(P, B, 100 + i)
        A = attrs(n)
        outs = []
        for mode, up in enumerate(ups):
            out, g = check_case(po, up, P, A, B, PRM, corr, ng_mode, f"beams {nb} mapping {mode}", oracle=nb < 4096 or corr == 0)
            assert g["smem_optin"] == optin and g["n_beams"] == nb
            kmap = 1 if mode == 1 and nb <= t_map1 else 0
            want_ppb = 32 if kmap else (ppb if mode == 0 else max(1, optin // (4 * nb)))
            assert (g["kmap"], g["ppb"], g["blocks"], g["smem"]) == (kmap, want_ppb, -(-n // want_ppb), 4 * nb * want_ppb), (nb, mode, g)
            outs.append(out)
        assert outs[0].tobytes() == outs[1].tobytes(), nb
    # one beam more than shared memory holds for one particle: refused, nothing changed, no CUDA error left behind
    B = beams(t_refuse + 1, 99)
    P, A = scan_particles(3), attrs(3)
    for up in ups:
        Pd, Ad = to_dev(P, A)
        with pytest.raises(rmcl_b200.B2Error) as e:
            up.update(Pd, Ad, tsb(), B, params(PRM, corr, ng_mode))
        assert e.value.code == B2_ERR_UNSUPPORTED
        assert from_dev(Ad).tobytes() == A.tobytes()
        with pytest.raises(rmcl_b200.B2Error):
            up.update(P, A, tsb(), B, params(PRM, corr, ng_mode))
        assert rmcl_b200.load_library().b2_peek_cuda_error().decode() == ""
        # and the handle still works
        check_case(po, up, P, A, beams(180, 3), PRM, corr, ng_mode, "after the refusal", f64=False)


@pytest.mark.gpu
@pytest.mark.parametrize("corr,ng_mode", COMBOS)
def test_pf_particle_count_edges(po, corr, ng_mode):
    """Particle counts around one block (1, ppb - 1, ppb, ppb + 1), around a warp (31, 32, 33: one lanes = particles block) and a large count
    with a partial last block, in both mappings; the large cloud repeats a smaller admissible set, so the float64 model runs on its distinct
    particles.  A case with dist_sigma 0.05 and particles spread around the scan pose shows the comparison is sensitive."""
    optin = smem_optin()
    B = beams(180, 7)
    ppb = expected_ppb(180, optin)
    base = admissible(scan_particles(400, 11, 0.3, 0.05), B, 11, 0.3, 0.05, corr)
    ref_base = model(base, attrs(len(base)), tsb(), B, PRM, corr, ng_mode)
    ups = [updater(0), updater(1)]
    large = 20 * 1024 + 7
    assert large % ppb and large % 32
    for n in sorted({1, ppb - 1, ppb, ppb + 1, 31, 32, 33, large}):
        idx = np.arange(n) % len(base) if n <= len(base) else np.random.default_rng(n).integers(0, len(base), n)
        P, A = base[idx], attrs(n)
        for mode, up in enumerate(ups):
            p = params(PRM, corr, ng_mode)
            out = update_dev(up, P, A, B, p)
            g = geometry(up)
            log(f"n {n} mapping {mode}", g)
            want = 32 if mode else ppb
            assert g["n"] == n and g["ppb"] == want and g["blocks"] == -(-n // want)
            assert_model(out, take(ref_base, idx), f"n {n} mapping {mode}")
            assert_oracle(out, oracle_pf(po).pf_update(P, A, tsb(), B, params(PRM, corr, ng_mode, po)), f"n {n}")
    # sensitivity: sharp Gaussian, particles a few centimetres around the scan pose
    P = admissible(scan_particles(300, 12, 0.1, 0.03), B, 12, 0.1, 0.03, corr)
    A = attrs(len(P))
    for mode, up in enumerate(ups):
        out, _ = check_case(po, up, P, A, B, PRM_SHARP, corr, ng_mode, f"sharp mapping {mode}")
    ref = model(P, A, tsb(), B, PRM_SHARP, corr, ng_mode)
    assert ref["mean"].std() >= 100 * ref["em"].max(), (ref["mean"].std(), ref["em"].max())


@pytest.mark.gpu
@pytest.mark.parametrize("corr,ng_mode", COMBOS)
def test_pf_mappings_and_auto(po, corr, ng_mode):
    """Mappings 0, 1, 2 (sorted particles) and 3 (auto) on a spread cloud and a converged one (near-identical poses, repeated sort keys,
    exact duplicates): bit-identical to each other, against the float64 model and the oracle.  Auto mode at 4095 and 4096 particles: below
    the threshold it stays on lanes = beams; from it on the second update runs the sorted mapping."""
    B = beams(180, 9)
    rng = np.random.default_rng(3)
    base = admissible(scan_particles(1000, 21, 0.3, 0.05), B, 21, 0.3, 0.05, corr)
    si = rng.permutation(np.arange(5000) % len(base))
    spread = base[si]
    uniq = admissible(scan_particles(300, 22, 0.002, 0.001), B, 22, 0.002, 0.001, corr)
    ci = rng.integers(0, len(uniq), 5000)
    conv = uniq[ci]
    for name, P in (("spread", spread), ("converged", conv)):
        A = attrs(len(P))
        outs = []
        for mode in (0, 1, 2, 3):
            up = updater(mode)
            for rep in range(2 if mode == 3 else 1):
                out, g = check_case(po, up, P, A, B, PRM, corr, ng_mode, f"{name} mapping {mode}.{rep}", f64=False, oracle=mode == 0)
                assert g["map_req"] == mode and g["sorted"] == int(g["map"] == 2) and g["kmap"] == int(g["map"] != 0)
                outs.append(out)
        for o in outs[1:]:
            assert o.tobytes() == outs[0].tobytes(), name
        if name == "converged":
            assert_model(outs[0], take(model(uniq, attrs(len(uniq)), tsb(), B, PRM, corr, ng_mode), ci), name)
        else:
            assert_model(outs[0], take(model(base, attrs(len(base)), tsb(), B, PRM, corr, ng_mode), si), name)
    # auto mode around its particle-count threshold
    for n, chosen in ((AUTO_SORT_FROM - 1, (0, 0)), (AUTO_SORT_FROM, (0, 2))):       # (from the third update on the choice follows timing)
        up = updater(3)
        P, A = spread[:n], attrs(n)
        ref = None
        for k, want in enumerate(chosen):
            out = update_dev(up, P, A, B, params(PRM, corr, ng_mode))
            g = geometry(up)
            log(f"auto n {n} update {k}", g)
            assert up.mapping() == (3, want) and g["map"] == want and g["sorted"] == int(want == 2)
            ref = out if ref is None else ref
            assert out.tobytes() == ref.tobytes()


@pytest.mark.gpu
def test_pf_host_path_chunks(po):
    """b2_pf_sensor_update_host below and at the start of the chunked two-stream path (32767, 32768, 32769) and at a large count that is not a
    multiple of 8 ppb: chunk sizes in whole blocks, pageable and pinned arrays, in place and not, byte for byte equal to the device-resident
    call; the float64 model at every chunk boundary, the oracle on all particles."""
    import torch
    optin = smem_optin()
    B = beams(180, 13)
    ppb = expected_ppb(180, optin)
    base = admissible(scan_particles(300, 31, 0.3, 0.05), B, 31, 0.3, 0.05)
    big = 100_003
    assert big % (8 * ppb)
    up_h, up_d = updater(0), updater(0)
    for n in (CHUNKED_FROM - 1, CHUNKED_FROM, CHUNKED_FROM + 1, big):
        idx = np.random.default_rng(n).integers(0, len(base), n)
        P, A = base[idx], attrs(n)
        A["likelihood"]["mean"] = np.random.default_rng(1).uniform(0.5, 1.5, n).astype(np.float32)
        A["likelihood"]["n_meas"] = np.arange(n) % 3
        dev = update_dev(up_d, P, A, B, params(PRM, 0, 0))
        out = up_h.update(P, A, tsb(), B, params(PRM, 0, 0))
        g = geometry(up_h)
        log(f"host n {n}", g)
        chunks = 8 if n >= CHUNKED_FROM else 1
        per = -(-(-(-n // chunks)) // ppb) * ppb
        assert (g["n_chunks"], g["per"], g["ppb"], g["blocks"]) == (chunks, per, ppb, -(-n // ppb)), g
        assert out.tobytes() == dev.tobytes(), n
        Ph = torch.from_numpy(P.view(np.uint8).copy()).pin_memory().numpy().view(P.dtype).reshape(-1)
        Ah = torch.from_numpy(A.view(np.uint8).copy()).pin_memory().numpy().view(A.dtype).reshape(-1)
        assert up_h.update(Ph, Ah, tsb(), B, params(PRM, 0, 0), inplace=True) is Ah and Ah.tobytes() == dev.tobytes()
        Ap = A.copy()
        assert up_h.update(P, Ap, tsb(), B, params(PRM, 0, 0), inplace=True) is Ap and Ap.tobytes() == dev.tobytes()
        assert up_h.update(Ph, A, tsb(), B, params(PRM, 0, 0)).tobytes() == dev.tobytes()
        # float64 model around every chunk boundary and at the end
        cut = sorted({j for c in range(chunks + 1) for j in range(c * per - 3, c * per + 3) if 0 <= j < n} | set(range(n - 5, n)))
        sub = np.asarray(cut)
        ref = model(P[sub], A[sub], tsb(), B, PRM, 0, 0)
        assert_model(out[sub], ref, f"host n {n}")
        if n < big:
            assert_oracle(out, oracle_pf(po).pf_update(P, A, tsb(), B, params(PRM, 0, 0, po)), f"host n {n}")


@pytest.mark.gpu
@pytest.mark.parametrize("corr,ng_mode", COMBOS)
def test_pf_n_meas_clamp(po, corr, ng_mode):
    """n_meas starting at 0, 9 990 (the MAX_N_MEAS clamp is crossed in the middle of the merge) and 10 000: against the float64 model and
    the oracle, and a second update equals one update with the beams concatenated, byte for byte."""
    B1, B2 = beams(180, 41), beams(180, 42)
    B = np.concatenate([B1, B2])
    P = admissible(scan_particles(300, 43, 0.3, 0.05), B, 43, 0.3, 0.05, corr)
    for ups in ((updater(0),), (updater(1),)):
        up = ups[0]
        for start in (0, 9990, 10000):
            A = attrs(len(P), start, 0.7)
            A["likelihood"]["sigma"] = 0.05
            one, _ = check_case(po, up, P, A, B1, PRM, corr, ng_mode, f"n_meas {start}")
            two, _ = check_case(po, up, P, one, B2, PRM, corr, ng_mode, f"n_meas {start} second")
            both, _ = check_case(po, up, P, A, B, PRM, corr, ng_mode, f"n_meas {start} concatenated")
            assert two.tobytes() == both.tobytes(), start
            assert (both["likelihood"]["n_meas"] == min(start + 360, MAX_N_MEAS)).all()


def dir_sort_key(B):
    """the beam table's sort key (api.cu dir_sort_key): Morton code of the direction on a 1024^3 lattice"""
    def q(v):
        return np.clip(((v * np.float32(0.5) + np.float32(0.5)) * np.float32(1023.0)).astype(np.int64), 0, 1023).astype(np.uint64)

    def spread(x):
        x = x & 0x3ff
        for s, m in ((16, 0x30000ff), (8, 0x300f00f), (4, 0x30c30c3), (2, 0x9249249)):
            x = (x | (x << np.uint64(s))) & np.uint64(m)
        return x
    d = B["dir"]
    return spread(q(d[:, 0])) | (spread(q(d[:, 1])) << np.uint64(1)) | (spread(q(d[:, 2])) << np.uint64(2))


@pytest.mark.gpu
@pytest.mark.parametrize("corr,ng_mode", COMBOS)
def test_pf_beam_order(po, corr, ng_mode):
    """The caller's beams in an order far from their direction sort, with repeated directions (sort-key ties): the merge follows the caller's
    order (oracle on the same order: n_meas exact, TOL_LIK, > 99 % bit-identical), the float64 model agrees within the merge bound, and the
    same beams in sorted order differ from it, if at all, only within the FP32 merge bound."""
    B = beams(512, 51, dup=64)
    key = dir_sort_key(B)
    srt = np.argsort(key, kind="stable")
    far = B[srt[::-1]]                                                    # reversed direction sort
    assert len(np.unique(key)) < len(key)
    P = admissible(scan_particles(257, 52, 0.3, 0.05), B, 52, 0.3, 0.05, corr)
    A = attrs(len(P))
    for mode in (0, 1):
        up = updater(mode)
        a, _ = check_case(po, up, P, A, far, PRM, corr, ng_mode, f"reversed mapping {mode}")
        b, _ = check_case(po, up, P, A, B[srt], PRM, corr, ng_mode, f"sorted mapping {mode}")
        ra = model(P, A, tsb(), far, PRM, corr, ng_mode)
        rb = model(P, A, tsb(), B[srt], PRM, corr, ng_mode)
        d = np.abs(a["likelihood"]["mean"].astype(np.float64) - b["likelihood"]["mean"])
        assert (d <= ra["em"] + rb["em"]).all() and np.array_equal(a["likelihood"]["n_meas"], b["likelihood"]["n_meas"])


@pytest.mark.gpu
def test_pf_likelihood_stats_edges():
    """likelihoodStats (k_pf_residual_stats) on each side of one block, of a last-block combine that strides (more blocks than a warp has lanes), of the
    grid cap 4 n_sm and far beyond it (grid-stride): float64 sum within 2e-6 relative, max exact; back-to-back calls of different sizes on
    one handle (the ticket is reset by each call's last block)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cap = 4 * sms * 256
    up = updater()
    rng = np.random.default_rng(7)
    A = attrs(1_000_003)
    A["likelihood"]["mean"] = rng.uniform(0, 0.2, len(A)).astype(np.float32)
    A["likelihood"]["mean"][rng.integers(0, len(A), 50)] = 0.0
    _, Ad = to_dev(scan_particles(1), A)
    sizes = [0, 1, 255, 256, 257, 65536, 65537, cap - 1, cap, cap + 1, len(A)]
    for n in sizes + sizes[::-1] + [65537, 1, cap + 1]:
        s, m = up.likelihoodStats(Ad[:n])
        sr, mr = stats_f64(A[:n])
        assert m == np.float32(mr) and abs(s - sr) <= 2e-6 * sr, (n, s, sr, m, mr)
        print(f"stats n {n}: blocks {min(4 * sms, -(-n // 256))}")
    # the max where only one particle carries it, in the last partial block
    A2 = A[: cap + 1].copy()
    A2["likelihood"]["mean"][-1] = 0.5
    _, Ad2 = to_dev(scan_particles(1), A2)
    assert up.likelihoodStats(Ad2)[1] == np.float32(0.5)


def scratch_call(up, op, Pd, Ad):
    """one particle-filter call of test_pf_shared_scratch_calls -> what it returned and wrote, as numpy arrays"""
    import torch
    import rmcl_b200
    n = Pd.shape[0]
    if op == "stats":
        return [np.array(up.likelihoodStats(Ad), np.float32)]
    if op == "estimate":
        return [up.estimateStats(Pd, Ad, max_induction_particles=n)]
    if op == "recovery":
        up.recoveryReset()
        return [up.recoveryObserve(Ad, want_state=True)]
    if op == "clusters":
        labels = torch.zeros(n, dtype=torch.int32, device=Pd.device)
        res, recs = up.estimateClusters(Pd, Ad, labels=labels)
        return [res, recs, labels.cpu().numpy()]
    Pn, An = torch.zeros_like(Pd), torch.zeros_like(Ad)
    if op == "residual":
        res = up.resampleResidual(Pd, Ad, Pn, An, seed=5, step=1)
    else:
        kld = rmcl_b200.KLDConfig.defaults()
        kld.n_min = min(kld.n_min, n)                                      # n_min <= n_max = n
        res = up.resampleKLD(Pd, Ad, Pn, An, kld, seed=5, step=2)
    return [res, Pn.cpu().numpy(), An.cpu().numpy()]


@pytest.mark.gpu
def test_pf_shared_scratch_calls():
    """likelihoodStats, estimateStats, resampleResidual, resampleKLD, estimateClusters and recoveryReset + recoveryObserve share one handle's
    block partials, tickets and records: on one handle, in a seeded shuffled order at 1, 257, 4 n_sm 256 + 1 and 1 000 003 particles, each
    call equals byte for byte the same call on a fresh handle.  likelihoodStats is the float32 of resampleResidual's weight_sum and weight_max
    on the same set: every caller reads one pass of the set's weight statistics."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(17)
    ops = ["stats", "estimate", "residual", "kld", "clusters", "recovery"]
    shared = updater()
    for n in (1, 257, 4 * sms * 256 + 1, 1_000_003):
        P = scan_particles(n, n % 1000, 0.5, 0.3)
        A = attrs(n)
        A["likelihood"]["mean"] = rng.uniform(0, 0.2, n).astype(np.float32)
        A["likelihood"]["mean"][rng.integers(0, n, max(1, n // 100))] = 0.0
        A["likelihood"]["mean"][0] = 0.1
        Pd, Ad = to_dev(P, A)
        got = {}
        for op in (ops[i] for i in rng.permutation(len(ops))):
            got[op] = scratch_call(shared, op, Pd, Ad)
            want = scratch_call(updater(), op, Pd, Ad)
            assert [a.tobytes() for a in got[op]] == [b.tobytes() for b in want], (n, op)
        r = got["residual"][0]
        assert got["stats"][0].tobytes() == np.array([r["weight_sum"], r["weight_max"]], np.float32).tobytes(), (n, got["stats"][0], r)
        assert r["n_particles"] > 0 and got["clusters"][0]["n_records"] >= 1, n
