"""TEST INFRASTRUCTURE ONLY: the branch-and-bound search's functions (rmcl_b200/csrc/kernels.cuh) compiled for the CPU
(pf_search_bnb_ref/bnb_emul.cu, the emulator library plus the pyramid build and the bound): the pyramid of a field, the bounds of the
nodes of a tree level and the exact scores of the candidates.  Built on first use with native.py's recipes."""
import ctypes as C
import os

import numpy as np

import dfield_ref as D
import native

_emul = None


def _lib():
    global _emul
    if _emul is None:
        _emul = C.CDLL(native._build("bnb_emul", native._NVCC, native._NVCC_FLAGS +
                                     ["-Xcompiler", "-fPIC,-fopenmp,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared"],
                                     [os.path.join(native.TESTS, "pf_search_bnb_ref", "bnb_emul.cu"),
                                      os.path.join(native.ROOT, "rmcl_b200", "csrc", "bvh_build.cpp")], ["-lgomp"], ".so"))
        _emul.emul_scene_create.restype = C.c_void_p
        _emul.emul_bnb_pyramid.restype = C.c_uint32
        _emul.emul_bnb_eval.restype = None
        _emul.emul_bnb_select.restype = C.c_uint32
        _emul.emul_bnb_query.restype = C.c_float
    return _emul


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


class Field:
    """a mesh, its product field built on the CPU (dfield_ref.ProductField) over the box [lo, hi], and a scene for the surface rule"""

    def __init__(self, V, F, h, trunc, lo=None, hi=None):
        self.V, self.F = np.ascontiguousarray(V, np.float32).reshape(-1, 3), np.ascontiguousarray(F, np.uint32).reshape(-1, 3)
        if lo is None:
            lo, hi = D.default_box(self.V, trunc)
        self.g = D.Grid(lo, hi, h, trunc)
        self.index, self.bricks = D.ProductField(self.V, self.F).build(self.g)
        err = C.c_char_p()
        self._s = _lib().emul_scene_create(_p(self.V), C.c_uint32(len(self.V)), _p(self.F), C.c_uint32(len(self.F)), C.byref(err))
        assert self._s

    def _bricks(self):
        return self.bricks if len(self.bricks) else np.zeros((1, 9, 9, 9), np.float32)

    def pyramid(self):
        """-> (fine2 (n, 64), fine4 (n, 8), [dense level L (z, y, x)])"""
        n = len(self.bricks)
        fine2, fine4 = np.zeros((max(n, 1), 64), np.float32), np.zeros((max(n, 1), 8), np.float32)
        bx, by, bz = self.g.bdims
        dense = np.zeros(2 * bx * by * bz + 64, np.float32)
        off = np.zeros(24, np.uint64)
        nd = _lib().emul_bnb_pyramid(*self.g.args(), _p(self.index), _p(self._bricks()), C.c_uint64(n), _p(fine2), _p(fine4), _p(dense), _p(off))
        levels = []
        for L in range(nd):
            d = [((b - 1) >> L) + 1 for b in (bx, by, bz)]
            levels.append(dense[int(off[L]):int(off[L]) + d[0] * d[1] * d[2]].reshape(d[2], d[1], d[0]))
        return fine2[:n], fine4[:n], levels

    def query(self, lo, hi):
        """the pyramid's min over the cells lo .. hi (x, y, z each) through the product's pyr_query"""
        clo, chi = np.ascontiguousarray(lo, np.uint32), np.ascontiguousarray(hi, np.uint32)
        return _lib().emul_bnb_query(*self.g.args(), _p(self.index), _p(self._bricks()), C.c_uint64(len(self.bricks)), _p(clo), _p(chi))

    def eval(self, Tsb, beams, prm, cfg, surface, level):
        """level >= 1: the bounds of the level's nodes, (K, nby, nbx); level 0: the candidates' exact scores, (K, ny, nx)"""
        nbx, nby = (cfg.nx + (1 << level) - 1) >> level, (cfg.ny + (1 << level) - 1) >> level
        out = np.zeros((cfg.n_yaw, nby, nbx), np.float32)
        B = np.ascontiguousarray(beams)
        _lib().emul_bnb_eval(C.c_void_p(self._s), *self.g.args(), _p(self.index), _p(self._bricks()), C.c_uint64(len(self.bricks)), _p(np.ascontiguousarray(Tsb)),
                             _p(B) if len(B) else None, C.c_uint32(len(B)), C.byref(prm), C.byref(cfg), None if surface is None else C.byref(surface),
                             C.c_uint32(level), _p(out))
        return out


def select(Lc, Ls, cfg):
    """one pass's peaks over L (sorted by c), their ranking and separation, by the product's functions -> (kept c, kept scores, n_peaks)"""
    Lc, Ls = np.ascontiguousarray(Lc, np.uint64), np.ascontiguousarray(Ls, np.float32)
    kc, ks, npk = np.zeros(64, np.uint64), np.zeros(64, np.float32), C.c_uint64()
    n = _lib().emul_bnb_select(_p(Lc) if len(Lc) else None, _p(Ls) if len(Ls) else None, C.c_uint64(len(Lc)), C.byref(cfg), _p(kc), _p(ks), C.byref(npk))
    return kc[:n], ks[:n], int(npk.value)


def search(S, bounds, cfg, n_beams, dist_sigma, min_ratio):
    """a restatement of the threshold passes (SURVEY N5) over a field's exact scores S (K, ny, nx) and the bounds of each tree level l >= 1
    (bounds[l], (K, nby, nbx)): a pass keeps the children of nodes with bound >= t, L = its leaves with score >= t, then select().
    -> (kept c, kept scores, best, tau, passes, L sets of every pass)"""
    K, ny, nx = S.shape
    depth = max(0, int(np.ceil(np.log2(max(nx, ny))))) if max(nx, ny) > 1 else 0
    sq = np.float32(dist_sigma) * np.float32(dist_sigma)
    denom = np.sqrt(float(np.float32(2.0) * sq) * np.pi)
    U = np.float32(1.0 / denom) if n_beams else np.float32(0.0)
    flat = S.reshape(-1)
    passes = []

    def one(t):
        alive = np.ones((K, 1, 1), bool)
        for lv in range(depth, 0, -1):
            b = bounds[lv]
            up = np.repeat(np.repeat(alive, 2, 1), 2, 2)[:, :b.shape[1], :b.shape[2]] if lv < depth else alive
            alive = up & (b >= t)
        leaves = np.repeat(np.repeat(alive, 2, 1), 2, 2)[:, :ny, :nx] if depth else alive
        Lc = np.flatnonzero(leaves.reshape(-1) & (flat >= t)).astype(np.uint64)
        passes.append((t, Lc))
        kc, ks, _ = select(Lc, flat[Lc.astype(np.int64)], cfg)
        return Lc, kc, ks

    best = tau = np.float32(-1.0)
    kc = ks = np.zeros(0)
    for q in range(1, 9):
        t = np.float32(U * np.float32((8 - q) / 8.0))
        Lc, kc, ks = one(t)
        if not len(Lc):
            continue
        best = np.float32(flat[Lc.astype(np.int64)].max())
        tau = np.float32(np.float32(min_ratio) * best)
        last, qb = t, 0
        while len(kc) < cfg.max_records and last > tau:
            qb += 1
            while np.float32(best * np.float32((8 - qb) / 8.0)) >= last:
                qb += 1
            tb = max(tau, np.float32(best * np.float32((8 - qb) / 8.0)))
            _, kc, ks = one(tb)
            last = tb
        break
    keep = ks >= tau if best >= 0 else np.zeros(len(ks), bool)
    return kc[keep], ks[keep], best, tau, passes
