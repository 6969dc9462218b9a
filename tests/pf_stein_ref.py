"""TEST INFRASTRUCTURE ONLY: references for the Stein variational step (b2_pf_stein_update, PCDSensorUpdaterB200.steinUpdate).

* The product's functions (rmcl_b200/csrc/kernels.cuh, b2_math.cuh) compiled for the CPU (pf_stein_ref/stein_emul.cu): exp_f and the library
  forms, df_lookup_grad, the draws of J, the score, the bandwidth, the pair sums, the move and the whole call, in the device's order.
* float64 numpy restatements of SURVEY appendix L: philox (Random123's Philox4x32-10), the draws of J, the chart, the score from a field
  given as (index, bricks), the bandwidth and the pair sums.
The library is built on first use into the per-user temporary directory of chain_ref."""
import ctypes as C
import os

import numpy as np

import dfield_ref as DR
from chain_ref import _build

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_CSRC = os.path.join(_ROOT, "rmcl_b200", "csrc")
TAG = 8
_emul = None


def lib():
    global _emul
    if _emul is None:
        src = os.path.join(_HERE, "pf_stein_ref", "stein_emul.cu")
        deps = [src] + [os.path.join(_CSRC, f) for f in ("kernels.cuh", "icp_loop.cuh", "trace.cuh", "b2_math.cuh", "bvh8.h", "bvh_build.cpp")] + \
               [os.path.join(_ROOT, "include", "rmcl_b200.h")]
        nvcc = os.environ.get("NVCC", "nvcc")
        _emul = _build("stein_emul", deps, [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-fmad=false",
                                            "-Xcompiler", "-fPIC,-fopenmp,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared", src,
                                            os.path.join(_CSRC, "bvh_build.cpp"), "-lgomp"])
        _emul.emul_stein_scene.restype = C.c_void_p
        _emul.emul_stein_scene_free.argtypes = [C.c_void_p]
    return _emul


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


class SteinConfig(C.Structure):
    _fields_ = [("iterations", C.c_uint32), ("n_ref", C.c_uint32), ("step_t", C.c_float), ("step_r", C.c_float), ("min_bandwidth_t", C.c_float),
                ("min_bandwidth_r", C.c_float), ("w_rand", C.c_float), ("pad", C.c_float)]


class SteinResult(C.Structure):
    _fields_ = [("bandwidth", C.c_float * 3), ("n_ref", C.c_uint32), ("n_blocked", C.c_uint32), ("rms_step_t", C.c_float), ("rms_step_r", C.c_float),
                ("pad", C.c_float)]


def exp_f(x):
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(x)
    lib().emul_exp_f(_p(x), C.c_uint64(x.size), _p(out))
    return out


def lib_f(which, a, b=None):
    """0: (float) atan2(a, b) in FP64; 1: (float) sin(a); 2: (float) cos(a)"""
    a = np.ascontiguousarray(a, np.float32)
    b = a if b is None else np.ascontiguousarray(b, np.float32)
    out = np.empty_like(a)
    lib().emul_lib_f(C.c_int(which), _p(a), _p(b), C.c_uint64(a.size), _p(out))
    return out


def lookup_grad(g, index, bricks, pts):
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    val, grad = np.empty(len(pts), np.float32), np.empty((len(pts), 3), np.float32)
    bricks = np.ascontiguousarray(bricks, np.float32)
    lib().emul_df_lookup_grad(*g.args(), _p(np.ascontiguousarray(index)), _p(bricks) if bricks.size else None, _p(pts), C.c_uint32(len(pts)), _p(val), _p(grad))
    return val, grad


def ref_index(m, n, n_ref, seed, step, it):
    out = np.empty(m, np.uint32)
    lib().emul_stein_ref_index(C.c_uint32(m), C.c_uint32(n), C.c_uint32(n_ref), C.c_uint64(seed), C.c_uint32(step), C.c_uint32(it), _p(out))
    return out


def chart(poses):
    P = np.ascontiguousarray(poses)
    out = np.empty((len(P), 3), np.float32)
    lib().emul_chart(_p(P), C.c_uint32(len(P)), _p(out))
    return out


def n_refs(n, n_ref):
    return n if n_ref == 0 or n_ref >= n else n_ref


def score(g, index, bricks, poses, n_ref, seed, step, it, Tsb, beams, dist_sigma, w_rand):
    """the product's k_pf_stein_score: -> snapshot (m, 6) float32 (x, y, psi, gx, gy, gpsi)"""
    P, B, T = np.ascontiguousarray(poses), np.ascontiguousarray(beams), np.ascontiguousarray(Tsb)
    m = n_refs(len(P), n_ref)
    snap = np.empty((m, 6), np.float32)
    bricks = np.ascontiguousarray(bricks, np.float32)
    lib().emul_stein_score(*g.args(), _p(np.ascontiguousarray(index)), _p(bricks) if bricks.size else None, _p(P), C.c_uint32(len(P)), C.c_uint32(m),
                           C.c_uint32(n_ref), C.c_uint64(seed), C.c_uint32(step), C.c_uint32(it), _p(T), _p(B) if len(B) else None, C.c_uint32(len(B)),
                           C.c_float(dist_sigma), C.c_float(w_rand), _p(snap))
    return snap


def bandwidth(poses, m, floor_t, floor_r):
    """the product's k_pf_stein_bandwidth: -> (h (3,) float32, sums (7,) float64)"""
    P = np.ascontiguousarray(poses)
    h, tot = np.empty(3, np.float32), np.empty(7, np.float64)
    lib().emul_stein_bandwidth(_p(P), C.c_uint32(len(P)), C.c_uint32(m), C.c_float(floor_t), C.c_float(floor_r), _p(h), _p(tot))
    return h, tot


def pairs(ci, snap, h):
    """the product's pair sums: -> acc (n, 3) float32"""
    ci = np.ascontiguousarray(ci, np.float32).reshape(-1, 3)
    snap = np.ascontiguousarray(snap, np.float32).reshape(-1, 6)
    h = np.ascontiguousarray(h, np.float32)
    acc = np.empty_like(ci)
    lib().emul_stein_pairs(_p(ci), C.c_uint32(len(ci)), _p(snap), C.c_uint32(len(snap)), _p(h), _p(acc))
    return acc


class Scene:
    """the product's host-built BVH of a mesh (the walls of the move)"""

    def __init__(self, V, F):
        self.V, self.F = DR._mesh(V, F)
        self._s = lib().emul_stein_scene(_p(self.V), C.c_uint32(len(self.V)), _p(self.F), C.c_uint32(len(self.F)))
        assert self._s

    def __del__(self):
        if getattr(self, "_s", None):
            lib().emul_stein_scene_free(self._s)

    def move(self, poses, snap, it, step_t, step_r, v, h, rec):
        """the product's k_pf_stein_move: poses and v (n, 3) float32 in place, rec (SteinResult) updated"""
        snap = np.ascontiguousarray(snap, np.float32)
        h = np.ascontiguousarray(h, np.float32)
        lib().emul_stein_move(C.c_void_p(self._s), _p(poses), C.c_uint32(len(poses)), _p(snap), C.c_uint32(len(snap)), C.c_uint32(it), C.c_float(step_t),
                              C.c_float(step_r), _p(v), _p(h), C.byref(rec))

    def update(self, g, index, bricks, poses, Tsb, beams, dist_sigma, cfg, seed, step):
        """the whole call on a copy of poses: -> (poses, SteinResult)"""
        P = np.array(poses, copy=True)
        B, T = np.ascontiguousarray(beams), np.ascontiguousarray(Tsb)
        bricks = np.ascontiguousarray(bricks, np.float32)
        rec = SteinResult()
        lib().emul_stein_update(C.c_void_p(self._s), *g.args(), _p(np.ascontiguousarray(index)), _p(bricks) if bricks.size else None, _p(P),
                                C.c_uint32(len(P)), _p(T), _p(B) if len(B) else None, C.c_uint32(len(B)), C.c_float(dist_sigma), C.byref(cfg),
                                C.c_uint64(seed), C.c_uint32(step), C.byref(rec))
        return P, rec


# ---------------------------------------------------------------- float64 restatements -----------------------------------------------
def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11) on uint32 arrays: -> four uint32 arrays"""
    M = np.uint64(0xFFFFFFFF)
    c = [np.asarray(x, np.uint64) & M for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0) & M, np.uint64(k1) & M
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & M, p1 & M, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & M, p0 & M]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M, (k1 + np.uint64(0xBB67AE85)) & M
    return [x.astype(np.uint32) for x in c]


def ref_index64(m, n, n_ref, seed, step, it):
    if n_ref == 0 or n_ref >= n:
        return np.arange(m, dtype=np.uint32)
    r = np.arange(m, dtype=np.uint64)
    w = philox(r, np.full(m, TAG), np.full(m, step), np.full(m, it), seed & 0xFFFFFFFF, seed >> 32)[0]
    return (w % np.uint32(n)).astype(np.uint32)


def chart64(poses):
    q = poses["R"].astype(np.float64)
    x, y, z, w = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    with np.errstate(invalid="ignore"):
        psi = np.where(np.isfinite(q).all(1), np.arctan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z)), np.nan)
    return np.stack([poses["t"][:, 0].astype(np.float64), poses["t"][:, 1].astype(np.float64), psi], 1)


def wrap64(a):
    return a - 2 * np.pi * np.rint(a / (2 * np.pi))


def lookup_grad64(g, index, bricks, pts):
    """the trilinear interpolant's value and gradient in float64 over the stored nodes, cell and t as the product picks them"""
    pts = np.asarray(pts, np.float32).reshape(-1, 3)
    val = DR.lookup64(g, index, bricks, pts)
    grad = np.zeros((len(pts), 3))
    fin = np.isfinite(pts).all(1)
    with np.errstate(over="ignore", invalid="ignore"):
        G = (pts - g.lo) * np.float32(g.inv_h)
    dims = np.array(g.dims)
    inside = fin & (G >= 0).all(1) & (G <= (dims - 1).astype(np.float32)).all(1)
    Gi = G[inside]
    c = np.minimum(np.floor(Gi).astype(np.int64), dims - 2)
    t = (Gi - c.astype(np.float32)).astype(np.float64)
    b = c >> 3
    slot = index[b[:, 2], b[:, 1], b[:, 0]].astype(np.int64)
    ok = slot != DR.NOBRICK
    l = (c & 7)[ok]
    s, tt = slot[ok], t[ok]
    B = np.asarray(bricks, np.float64)
    n = np.empty((len(s), 2, 2, 2))
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                n[:, dz, dy, dx] = B[s, l[:, 2] + dz, l[:, 1] + dy, l[:, 0] + dx]
    tx, ty, tz = tt[:, 0], tt[:, 1], tt[:, 2]
    wx = np.stack([1 - tx, tx], 1)
    wy = np.stack([1 - ty, ty], 1)
    wz = np.stack([1 - tz, tz], 1)
    dw = np.array([-1.0, 1.0])
    gx = np.einsum("izyx,iz,iy,x->i", n, wz, wy, dw)
    gy = np.einsum("izyx,iz,y,ix->i", n, wz, dw, wx)
    gz = np.einsum("izyx,z,iy,ix->i", n, dw, wy, wx)
    gi = np.zeros((len(Gi), 3))
    gi[ok] = np.stack([gx, gy, gz], 1) * float(np.float32(g.inv_h))
    grad[inside] = gi
    return val, grad


def score64(g, index, bricks, poses, idx, Tsb, beams, dist_sigma, w_rand):
    """the score of the particles idx in float64: -> (m, 3); NaN rows where the chart or score is not finite"""
    P = poses[idx]
    pts = DR.beam_points64(P, Tsb, beams)
    m, nb = len(P), len(beams)
    out = np.zeros((m, 3))
    if nb:
        e, gr = lookup_grad64(g, index, bricks, pts.reshape(-1, 3))
        e, gr = e.reshape(m, nb), gr.reshape(m, nb, 3)
        s2 = float(np.float32(dist_sigma)) ** 2
        w = float(np.float32(w_rand))
        with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
            G = np.exp(-e * e / (2 * s2))
            num = (1 - w) * G
            a = np.where(np.isfinite(e), -(e / s2) * np.where(num > 0, num / (num + w), 0.0), 0.0)
            gr = np.where(np.isfinite(e)[..., None], gr, 0.0)
        t = P["t"].astype(np.float64)
        rel = pts - t[:, None, :]
        out[:, 0] = (a * gr[..., 0]).sum(1)
        out[:, 1] = (a * gr[..., 1]).sum(1)
        out[:, 2] = (a * (rel[..., 0] * gr[..., 1] - rel[..., 1] * gr[..., 0])).sum(1)
    c = chart64(P)
    bad = ~(np.isfinite(c).all(1) & np.isfinite(out).all(1))
    out[bad] = np.nan
    return out


def bandwidth64(poses, m, floor_t, floor_r):
    c = chart64(poses)
    c = c[np.isfinite(c).all(1)]
    if len(c) == 0:
        return np.array([floor_t, floor_t, floor_r], np.float64)
    R = np.hypot(np.cos(c[:, 2]).mean(), np.sin(c[:, 2]).mean())
    s = np.array([c[:, 0].std(), c[:, 1].std(), np.sqrt(2 * max(1 - R, 0.0))])
    return np.maximum(s * float(m) ** (-1 / 7), [floor_t, floor_t, floor_r])


def pairs64(ci, snap, h):
    """sum over the valid references of k (g + Delta / h^2), float64: -> (n, 3)"""
    ci = np.asarray(ci, np.float64)
    sn = np.asarray(snap, np.float64)
    sn = sn[np.isfinite(sn[:, 0])]
    h = np.asarray(h, np.float64)
    D = ci[:, None, :] - sn[None, :, :3]
    D[..., 2] = wrap64(D[..., 2])
    U = D / h ** 2
    k = np.exp(-0.5 * (D * U).sum(2))
    return np.einsum("ij,ijd->id", k, sn[None, :, 3:] + U)
