"""TEST INFRASTRUCTURE ONLY: one rank's session of the sharded Stein steps (b2_pf_stein_slice_*, SURVEY L14) on the CPU, through the
product's functions compiled for the host (pf_stein_sharded_ref/stein_slice_emul.cu: the emulator library plus the slice score and move).

Session.score and Session.move run a rank's launches: the score of its range of J, then the bandwidth over the whole set and the move of
its slice.  The whole-set reference they are compared against is pf_stein_ref.Scene.update, the emulated b2_pf_stein_update.  The library
is built on first use with native.py's emulator recipe."""
import ctypes as C
import functools
import os

import numpy as np

import native
import pf_stein_ref as S


@functools.cache
def lib():
    L = C.CDLL(native._build("stein_slice_emul", native._NVCC, native._NVCC_FLAGS +
                             ["-Xcompiler", "-fPIC,-fopenmp,-ffp-contract=off,-mavx2,-mfma,-fvisibility=hidden", "-shared"],
                             [os.path.join(native.TESTS, "pf_stein_sharded_ref", "stein_slice_emul.cu"),
                              os.path.join(native.ROOT, "rmcl_b200", "csrc", "bvh_build.cpp")], ["-lgomp"], ".so"))
    L.emul_scene_create.restype = C.c_void_p
    return L


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


class SteinSliceResult(C.Structure):
    _fields_ = [("bandwidth", C.c_float * 3), ("n_ref", C.c_uint32), ("n_blocked", C.c_uint32), ("n_steps", C.c_uint32), ("sum_step_t2", C.c_double),
                ("sum_step_r2", C.c_double)]


class Walls:
    """the product's host-built BVH of a mesh in this library (the walls of the move)"""

    def __init__(self, verts, faces):
        self.verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
        self.faces = np.ascontiguousarray(faces, np.uint32).reshape(-1, 3)
        err = C.c_char_p()
        h = lib().emul_scene_create(_p(self.verts), C.c_uint32(len(self.verts)), _p(self.faces), C.c_uint32(len(self.faces)), C.byref(err))
        if not h:
            raise RuntimeError("emul BVH build failed: " + err.value.decode())
        self._h = C.c_void_p(h)

    def __del__(self):
        try:
            lib().emul_scene_destroy(self._h)
        except Exception:
            pass


class Session:
    """one rank's b2_pf_stein_slice_* session: score(P_all, it) -> (j_count, 6) snapshot rows; move(P_all, snap_all, it, out) runs the
    whole-set bandwidth, then moves poses first + i into out[i]; result() -> the record dict"""

    def __init__(self, walls, g, index, bricks, n_all, first, n_local, j_first, j_count, Tsb, beams, dist_sigma, cfg, seed, step):
        self.walls, self.g, self.index = walls, g, np.ascontiguousarray(index)
        self.bricks = np.ascontiguousarray(bricks, np.float32)
        self.B, self.T = np.ascontiguousarray(beams), np.ascontiguousarray(Tsb)
        self.n_all, self.first, self.n_local, self.j_first, self.j_count = n_all, first, n_local, j_first, j_count
        self.m = S.n_refs(n_all, cfg.n_ref)
        self.dist_sigma, self.cfg, self.seed, self.step = dist_sigma, cfg, seed, step
        self.v = np.zeros((n_local, 3), np.float32)
        self.rec = SteinSliceResult()

    def score(self, P_all, it):
        snap = np.empty((self.j_count, 6), np.float32)
        if self.j_count:
            lib().emul_stein_slice_score(*self.g.args(), _p(self.index), _p(self.bricks) if self.bricks.size else None, _p(P_all), C.c_uint32(self.n_all),
                                         C.c_uint32(self.j_first), C.c_uint32(self.j_count), C.c_uint32(self.cfg.n_ref), C.c_uint64(self.seed),
                                         C.c_uint32(self.step), C.c_uint32(it), _p(self.T), _p(self.B) if len(self.B) else None, C.c_uint32(len(self.B)),
                                         C.c_float(self.dist_sigma), C.c_float(self.cfg.w_rand), _p(snap))
        return snap

    def move(self, P_all, snap_all, it, out):
        h, _ = S.bandwidth(P_all, self.m, self.cfg.min_bandwidth_t, self.cfg.min_bandwidth_r)
        self.rec.bandwidth[:] = h.tolist()
        self.rec.n_ref = self.m
        snap_all = np.ascontiguousarray(snap_all, np.float32)
        lib().emul_stein_slice_move(self.walls._h, _p(P_all), C.c_uint32(self.first), C.c_uint32(self.n_local), _p(snap_all), C.c_uint32(self.m),
                                    C.c_uint32(it), C.c_float(self.cfg.step_t), C.c_float(self.cfg.step_r), _p(self.v), _p(h), _p(out), C.byref(self.rec))

    def result(self):
        r = self.rec
        return {"bandwidth": tuple(np.array(r.bandwidth, np.float32).tolist()), "n_ref": r.n_ref, "n_blocked": r.n_blocked, "n_steps": r.n_steps,
                "sum_step_t2": r.sum_step_t2, "sum_step_r2": r.sum_step_r2}
