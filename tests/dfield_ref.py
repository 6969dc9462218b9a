"""TEST INFRASTRUCTURE ONLY: references for the distance field (b2_dfield_*, b2_pf_sensor_update_field, rmcl_b200.DistanceField).

* ProductField: the product's df_* functions, pf_eval_field / pf_merge and the bounded closest point (rmcl_b200/csrc/kernels.cuh, trace.cuh)
  compiled for the CPU over the product's host-built BVH (dfield_ref/dfield_emul.cu): the grid, the build, the lookup and the update.
* RefField: a node's value restated over the oracle's closest point (dfield_ref/dfield_ref.c), brute force or through the oracle's BVH.
* node_points / lookup64 / update64: numpy restatements -- the nodes' positions in float32 ops, the trilinear lookup in float64 over the
  stored nodes, the sensor update in float64.
Both libraries are built on first use by native.py."""
import ctypes as C

import numpy as np

import native
import pyemul

NOBRICK = 0xFFFFFFFF
_ref = None
_emul = None


def _ref_lib():
    global _ref
    if _ref is None:
        _ref = native.restatement("dfield_ref/dfield_ref.c")
        _ref.orc_scene_create.restype = C.c_void_p
        _ref.orc_scene_destroy.argtypes = [C.c_void_p]
    return _ref


def _emul_lib():
    global _emul
    if _emul is None:
        _emul = native.emulator()
        _emul.emul_df_build.restype = C.c_int64
        _emul.emul_df_grid.restype = C.c_int
    return _emul


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _mesh(V, F):
    return np.ascontiguousarray(V, np.float32).reshape(-1, 3), np.ascontiguousarray(F, np.uint32).reshape(-1, 3)


def default_box(V, trunc):
    """the map's AABB grown by trunc, in float32 ops (b2_dfield_create with null bounds)"""
    V = np.asarray(V, np.float32).reshape(-1, 3)
    t = np.float32(trunc)
    return V.min(0) - t, V.max(0) + t


class Grid:
    """a field's grid: lo, hi (float32), h, trunc, dims (x, y, z nodes), bdims (x, y, z bricks), inv_h"""

    def __init__(self, lo, hi, h, trunc):
        self.lo, self.hi = np.asarray(lo, np.float32).reshape(3).copy(), np.asarray(hi, np.float32).reshape(3).copy()
        self.h, self.trunc = float(np.float32(h)), float(np.float32(trunc))
        dims = np.zeros(6, np.uint32)
        inv = C.c_float()
        nb = C.c_uint64()
        why = C.create_string_buffer(256)
        rc = _emul_lib().emul_df_grid(_p(self.lo), _p(self.hi), C.c_float(self.h), C.c_float(self.trunc), _p(dims), C.byref(inv), C.byref(nb), why, 256)
        self.refused = why.value.decode() if rc else None
        self.dims, self.bdims, self.inv_h, self.n_bricks = tuple(int(x) for x in dims[:3]), tuple(int(x) for x in dims[3:]), inv.value, nb.value

    def args(self):
        return _p(self.lo), _p(self.hi), C.c_float(self.h), C.c_float(self.trunc)


def node_points(g, ids):
    """float32 positions (len(ids), 9, 9, 9, 3) of the nodes of the bricks with linear ids, indexed [z, y, x]: add(origin, mul((float)i, h))"""
    ids = np.asarray(ids, np.int64)
    bx, by, _ = g.bdims
    bi, bj, bk = ids % bx, ids // bx % by, ids // bx // by
    l = np.arange(9)
    h = np.float32(g.h)
    X = g.lo[0] + (8 * bi[:, None] + l[None, :]).astype(np.float32) * h
    Y = g.lo[1] + (8 * bj[:, None] + l[None, :]).astype(np.float32) * h
    Z = g.lo[2] + (8 * bk[:, None] + l[None, :]).astype(np.float32) * h
    n = len(ids)
    P = np.empty((n, 9, 9, 9, 3), np.float32)
    P[..., 0] = X[:, None, None, :]
    P[..., 1] = Y[:, None, :, None]
    P[..., 2] = Z[:, :, None, None]
    return P


def brick_centres(g):
    """float32 centre node (8b + 4) of every brick, in linear order: node_points(g, ids)[:, 4, 4, 4] without its other 728 nodes"""
    ids = np.arange(g.n_bricks, dtype=np.int64)
    bx, by, _ = g.bdims
    b = np.stack([ids % bx, ids // bx % by, ids // bx // by], 1)
    return g.lo + (8 * b + 4).astype(np.float32) * np.float32(g.h)


def lookup64(g, index, bricks, pts):
    """the lookup restated: g = (p - origin) * inv_h in float32 ops, cell and t as the product picks them, trilinear (x, y, z) in float64"""
    pts = np.asarray(pts, np.float32).reshape(-1, 3)
    out = np.full(len(pts), g.trunc, np.float64)
    fin = np.isfinite(pts).all(1)
    out[~fin] = np.inf
    with np.errstate(over="ignore", invalid="ignore"):
        G = (pts - g.lo) * np.float32(g.inv_h)
    dims = np.array(g.dims)
    inside = fin & (G >= 0).all(1) & (G <= (dims - 1).astype(np.float32)).all(1)
    Gi = G[inside]
    c = np.minimum(np.floor(Gi).astype(np.int64), dims - 2)
    t = (Gi - c.astype(np.float32)).astype(np.float64)
    b = c >> 3
    slot = index[b[:, 2], b[:, 1], b[:, 0]].astype(np.int64)
    l = c & 7
    v = np.full(len(Gi), g.trunc, np.float64)
    ok = slot != NOBRICK
    s, lx, ly, lz, tt = slot[ok], l[ok, 0], l[ok, 1], l[ok, 2], t[ok]
    B = bricks.astype(np.float64)

    def at(dz, dy, dx):
        return B[s, lz + dz, ly + dy, lx + dx]
    tx, ty, tz = tt[:, 0], tt[:, 1], tt[:, 2]
    c00 = at(0, 0, 0) * (1 - tx) + at(0, 0, 1) * tx
    c10 = at(0, 1, 0) * (1 - tx) + at(0, 1, 1) * tx
    c01 = at(1, 0, 0) * (1 - tx) + at(1, 0, 1) * tx
    c11 = at(1, 1, 0) * (1 - tx) + at(1, 1, 1) * tx
    v[ok] = (c00 * (1 - ty) + c10 * ty) * (1 - tz) + (c01 * (1 - ty) + c11 * ty) * tz
    out[inside] = v
    return out


def _qmul(a, b):
    ax, ay, az, aw = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bx, by, bz, bw = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], -1)


def _qrot(q, v):
    u, w = q[..., :3], q[..., 3:4]
    t = 2.0 * np.cross(u, v)
    return v + w * t + np.cross(u, t)


def beam_points64(poses, Tsb, beams):
    """(n, n_beams, 3) float64 beam end points orig_m + dir_m * range with Tsm = pose * Tsb"""
    R = poses["R"].astype(np.float64)
    t = poses["t"].astype(np.float64)
    sR, st = np.asarray(Tsb["R"], np.float64).reshape(4), np.asarray(Tsb["t"], np.float64).reshape(3)
    Rm = _qmul(R, np.broadcast_to(sR, R.shape))
    tm = t + _qrot(R, np.broadcast_to(st, t.shape))
    o = beams["orig"].astype(np.float64)
    d = beams["dir"].astype(np.float64)
    r = beams["range"].astype(np.float64)
    Rb = Rm[:, None, :]
    om = tm[:, None, :] + _qrot(np.broadcast_to(Rb, (len(R), len(o), 4)), np.broadcast_to(o, (len(R), len(o), 3)))
    dm = _qrot(np.broadcast_to(Rb, (len(R), len(o), 4)), np.broadcast_to(d, (len(R), len(o), 3)))
    return om + dm * r[None, :, None]


def merge64(attrs, ev):
    """Gaussian1D merge of evaluations ev (n, n_beams) in beam order, float64, with the MAX_N_MEAS clamp: -> (mean, sigma, n_meas)"""
    mean = attrs["likelihood"]["mean"].astype(np.float64).copy()
    sig = attrs["likelihood"]["sigma"].astype(np.float64).copy()
    nm = attrs["likelihood"]["n_meas"].astype(np.int64).copy()
    for b in range(ev.shape[1]):
        n = nm + 1
        w1, w2 = nm / n, 1.0 / n
        m = mean * w1 + ev[:, b] * w2
        sig = sig * w1 + (mean - m) ** 2 * w1 + (ev[:, b] - m) ** 2 * w2
        mean = m
        nm = np.minimum(n, 10000)
    return mean, sig, nm


def evaluate64(err, dist_sigma):
    sq = float(np.float32(dist_sigma) * np.float32(dist_sigma))
    return np.exp(-(err * err) / sq / 2.0) / np.sqrt(2.0 * sq * np.pi)


class ProductField(pyemul.Scene):
    """the product's distance-field functions on the CPU"""

    def build(self, g):
        """-> (index uint32 (bz, by, bx), bricks float32 (n, 9, 9, 9))"""
        bx, by, bz = g.bdims
        index = np.empty((bz, by, bx), np.uint32)
        cap = g.n_bricks
        bricks = np.empty((cap, 9, 9, 9), np.float32)
        n = _emul_lib().emul_df_build(self._h, *g.args(), _p(index), _p(bricks), C.c_uint64(cap))
        assert n >= 0
        return index, bricks[:n].copy()

    def closest(self, pts, bounded=False, trunc=0.0):
        """-> (d2, face) of the product's closest point, bounded at trunc (limit from fl(trunc^2)) or not"""
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
        d2, face = np.empty(len(pts), np.float32), np.empty(len(pts), np.uint32)
        t = np.float32(trunc)
        _emul_lib().emul_df_closest(self._h, _p(pts), C.c_uint32(len(pts)), C.c_int(int(bounded)), C.c_float(float(t * t)), _p(d2), _p(face))
        return d2, face


def lookup(g, index, bricks, pts):
    """the product's df_lookup on the CPU"""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    out = np.empty(len(pts), np.float32)
    bricks = np.ascontiguousarray(bricks, np.float32)
    _emul_lib().emul_df_lookup(*g.args(), _p(np.ascontiguousarray(index)), _p(bricks) if bricks.size else None, _p(pts), C.c_uint32(len(pts)), _p(out))
    return out


def pf_update(g, index, bricks, poses, attrs, Tsb, beams, prm):
    """the product's field update (pf_eval_field + pf_merge) on the CPU: -> updated copy of attrs"""
    A = np.array(attrs, copy=True)
    P = np.ascontiguousarray(poses)
    B = np.ascontiguousarray(beams)
    Tsb = np.ascontiguousarray(Tsb)
    bricks = np.ascontiguousarray(bricks, np.float32)
    _emul_lib().emul_df_pf_update(*g.args(), _p(np.ascontiguousarray(index)), _p(bricks) if bricks.size else None, _p(P), _p(A), C.c_uint32(len(P)), _p(Tsb),
                                  _p(B) if len(B) else None, C.c_uint32(len(B)), C.byref(prm))
    return A


class RefField:
    """the node rule over the oracle's closest point"""

    def __init__(self, V, F):
        self.V, self.F = _mesh(V, F)
        self._s = _ref_lib().orc_scene_create(_p(self.V), C.c_uint32(len(self.V)), _p(self.F), C.c_uint32(len(self.F)))
        assert self._s

    def __del__(self):
        if getattr(self, "_s", None):
            _ref_lib().orc_scene_destroy(self._s)

    def values(self, pts, trunc, brute=False):
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
        out = np.empty(len(pts), np.float32)
        _ref_lib().orc_df_values(C.c_void_p(self._s), _p(pts), C.c_uint32(len(pts)), C.c_float(trunc), C.c_int(int(brute)), _p(out))
        return out

    def dist(self, pts, brute=False):
        pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
        out = np.empty(len(pts), np.float32)
        _ref_lib().orc_df_dist(C.c_void_p(self._s), _p(pts), C.c_uint32(len(pts)), C.c_int(int(brute)), _p(out))
        return out

    def lower_bound(self, pts, depth=2):
        """float64 lower bound of the distance from each point to the mesh: the distance to the nearest of 2^depth boxes that together hold
        every face (faces split at the median centroid along the longest axis of their box, depth times)"""
        T = self.V[self.F].astype(np.float64)
        groups = [np.arange(len(T))]
        for _ in range(depth):
            nxt = []
            for g in groups:
                if len(g) < 2:
                    nxt.append(g)
                    continue
                c = T[g].mean(1)
                ax = int(np.argmax(c.max(0) - c.min(0)))
                o = g[np.argsort(c[:, ax], kind="stable")]
                nxt += [o[: len(o) // 2], o[len(o) // 2:]]
            groups = nxt
        lo = np.array([T[g].min((0, 1)) for g in groups])
        hi = np.array([T[g].max((0, 1)) for g in groups])
        pts = np.asarray(pts, np.float64).reshape(-1, 3)
        out = np.full(len(pts), np.inf)
        for l, h in zip(lo, hi):
            d2 = np.zeros(len(pts))
            for k in range(3):
                e = np.maximum(l[k] - pts[:, k], pts[:, k] - h[k])
                np.maximum(e, 0.0, out=e)
                d2 += e * e
            np.minimum(out, d2, out=out)
        return np.sqrt(out)
