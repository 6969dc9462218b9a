"""ctypes binding of the emulator library (tests/emul/emul.cu, built by tests/native.py) -- TEST HARNESS ONLY (CPU run of the product's
host+device traversal code)."""
from __future__ import annotations

import ctypes as C

import numpy as np

import native
from rmcl_b200.synth import CROSS_STATS_DTYPE as CROSS_STATS, TRANSFORM_DTYPE as TRANSFORM


class _EmulTf(C.Structure):
    _fields_ = [("v", C.c_float * 7), ("stamp", C.c_uint32)]


class _EmulSensor(C.Structure):
    _fields_ = [("n", C.c_uint32), ("n_origs", C.c_uint32), ("origs", C.c_void_p), ("dirs", C.c_void_p), ("dpts", C.c_void_p), ("dmask", C.c_void_p),
                ("Tbo", _EmulTf), ("Tsb", _EmulTf), ("range_max", C.c_float), ("max_dist", C.c_float), ("pad0", C.c_float), ("pad1", C.c_float),
                ("merge_weight", C.c_double)]


class PFParams(C.Structure):
    _fields_ = [("dist_sigma", C.c_float), ("real_hit_sim_miss_error", C.c_float), ("real_miss_sim_hit_error", C.c_float),
                ("real_miss_sim_miss_error", C.c_float), ("range_min", C.c_float), ("range_max", C.c_float), ("ng_mode", C.c_int),
                ("correspondence_type", C.c_int)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = native.emulator()
        _lib.emul_scene_create.restype = C.c_void_p
    return _lib


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


class Scene:
    """the product's host-built BVH of a mesh"""

    def __init__(self, verts, faces):
        self.verts = _f32(verts).reshape(-1, 3)
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

    def info(self):
        a, b, c, d = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_float()
        lib().emul_scene_info(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d))
        return dict(n_nodes=a.value, n_tris=b.value, max_depth=c.value, sah=d.value)

    def export_blob(self):
        """the host-built tree as Map.export_blob lays it out (numpy uint8)"""
        inf = self.info()
        buf = np.zeros(64 + 224 * inf["n_nodes"] + 48 * inf["n_tris"], np.uint8)
        lib().emul_export(self._h, C.c_uint32(len(self.faces)), C.c_uint32(len(self.verts)), _p(buf))
        return buf

    def intersect(self, origs, dirs, tfar=np.inf, per_ray=False):
        origs, dirs = _f32(origs).reshape(-1, 3), _f32(dirs).reshape(-1, 3)
        n = len(origs)
        t, f, ng, h = np.empty(n, np.float32), np.empty(n, np.uint32), np.empty((n, 3), np.float32), np.empty(n, np.uint8)
        mn, mt = C.c_double(), C.c_double()
        pn = np.zeros(n, np.uint32) if per_ray else None
        pt = np.zeros(n, np.uint32) if per_ray else None
        lib().emul_intersect(self._h, _p(origs), _p(dirs), C.c_uint32(n), C.c_float(tfar), _p(t), _p(f), _p(ng), _p(h), C.byref(mn), C.byref(mt), _p(pn), _p(pt))
        if per_ray:
            return t, f, ng, h, (mn.value, mt.value), pn, pt
        return t, f, ng, h, (mn.value, mt.value)

    def find(self, Tbm, Tsb, origs_s, dirs_s, range_max, range_min=0.0, sim_opts=0):
        origs_s, dirs_s = _f32(origs_s).reshape(-1, 3), _f32(dirs_s).reshape(-1, 3)
        n = len(dirs_s)
        out = dict(points=np.empty((n, 3), np.float32), normals=np.empty((n, 3), np.float32), hits=np.empty(n, np.uint8),
                   face_ids=np.empty(n, np.uint32), ranges=np.empty(n, np.float32))
        Tbm, Tsb = np.ascontiguousarray(Tbm), np.ascontiguousarray(Tsb)
        lib().emul_find_opt(self._h, _p(Tbm), _p(Tsb), C.c_uint32(n), _p(origs_s), C.c_uint32(len(origs_s)), _p(dirs_s), C.c_float(range_min), C.c_float(range_max),
                            C.c_uint32(sim_opts), _p(out["points"]), _p(out["normals"]), _p(out["hits"]), _p(out["face_ids"]), _p(out["ranges"]))
        return out

    def cpc_find(self, Tbm, Tsb, dataset_pts, max_dist):
        dp = _f32(dataset_pts).reshape(-1, 3)
        n = len(dp)
        out = dict(points=np.empty((n, 3), np.float32), normals=np.empty((n, 3), np.float32), hits=np.empty(n, np.uint8),
                   face_ids=np.empty(n, np.uint32), dists=np.empty(n, np.float32))
        Tbm, Tsb = np.ascontiguousarray(Tbm), np.ascontiguousarray(Tsb)
        mn, mt = C.c_double(), C.c_double()
        pn, pt = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        lib().emul_cpc_find(self._h, _p(Tbm), _p(Tsb), C.c_uint32(n), _p(dp), C.c_float(max_dist), _p(out["points"]), _p(out["normals"]), _p(out["hits"]),
                            _p(out["face_ids"]), _p(out["dists"]), C.byref(mn), C.byref(mt), _p(pn), _p(pt))
        out["work"] = (mn.value, mt.value)
        out["per_query"] = (pn, pt)
        return out

    def correct_once(self, origs_s, dirs_s, range_max, dpts, dmask, Tom, Tbo, Tsb, iterations, max_dist, fast_tail=False):
        origs_s, dirs_s = _f32(origs_s).reshape(-1, 3), _f32(dirs_s).reshape(-1, 3)
        dpts, dmask = _f32(dpts), np.ascontiguousarray(dmask, np.uint8)
        Tn, Td, Cm = np.zeros((), TRANSFORM), np.zeros((), TRANSFORM), np.zeros((), CROSS_STATS)
        Tom, Tbo, Tsb = np.ascontiguousarray(Tom), np.ascontiguousarray(Tbo), np.ascontiguousarray(Tsb)
        lib().emul_correct_once(self._h, C.c_uint32(len(dirs_s)), _p(origs_s), C.c_uint32(len(origs_s)), _p(dirs_s), C.c_float(range_max), _p(dpts), _p(dmask),
                                _p(Tom), _p(Tbo), _p(Tsb), C.c_uint32(iterations), C.c_float(max_dist), _p(Tn), _p(Td), _p(Cm), C.c_int(int(fast_tail)))
        return Tn, Td, Cm

    def micp_multi(self, sensors, Tom, iterations=5):
        """the fused loop of the product (icp_tail, weighted multi-sensor merge) on the CPU; sensors: list of dicts like pyoracle.micp_correct_once_multi
        (ray-casting sensors only; `max_dist` is the effective gate)"""
        arr = (_EmulSensor * len(sensors))()
        keep = []
        for k, sd in enumerate(sensors):
            dp, dm = _f32(sd["dataset_points"]).reshape(-1, 3), np.ascontiguousarray(sd["dataset_mask"], np.uint8)
            o, d = _f32(sd["origs"]).reshape(-1, 3), _f32(sd["dirs"]).reshape(-1, 3)
            keep += [dp, dm, o, d]
            a = arr[k]
            a.n, a.n_origs, a.origs, a.dirs, a.dpts, a.dmask = len(d), len(o), o.ctypes.data, d.ctypes.data, dp.ctypes.data, dm.ctypes.data
            C.memmove(C.byref(a, _EmulSensor.Tbo.offset), np.ascontiguousarray(sd["Tbo"]).ctypes.data, 32)
            C.memmove(C.byref(a, _EmulSensor.Tsb.offset), np.ascontiguousarray(sd["Tsb"]).ctypes.data, 32)
            a.range_max, a.max_dist, a.merge_weight = sd["range_max"], sd.get("max_dist", 1.0), sd.get("weight", 1.0)
        Tn, Td, Cm = np.zeros((), TRANSFORM), np.zeros((), TRANSFORM), np.zeros((), CROSS_STATS)
        Tom = np.ascontiguousarray(Tom)
        lib().emul_micp_multi(self._h, C.c_uint32(len(sensors)), arr, _p(Tom), C.c_uint32(iterations), _p(Tn), _p(Td), _p(Cm))
        return Tn, Td, Cm

    def refit(self, verts, faces):
        verts, faces = _f32(verts).reshape(-1, 3), np.ascontiguousarray(faces, np.uint32).reshape(-1, 3)
        lib().emul_refit.restype = C.c_int
        rc = lib().emul_refit(self._h, _p(verts), C.c_uint32(len(verts)), _p(faces))
        assert rc == 0, "tree layout: a child index is not larger than its parent's"

    def pf_motion(self, poses, attrs, T, forget_rate, collide):
        poses, attrs = np.ascontiguousarray(poses).copy(), np.ascontiguousarray(attrs).copy()
        T = np.ascontiguousarray(T)
        lib().emul_pf_motion(self._h, C.c_uint32(len(poses)), _p(poses), _p(attrs), _p(T), C.c_double(forget_rate), C.c_int(int(collide)))
        return poses, attrs

    def pf_update(self, poses, attrs, Tsb, beams, params):
        poses = np.ascontiguousarray(poses)
        attrs = np.ascontiguousarray(attrs).copy()
        beams = np.ascontiguousarray(beams)
        Tsb = np.ascontiguousarray(Tsb)
        prm = PFParams(params.dist_sigma, params.real_hit_sim_miss_error, params.real_miss_sim_hit_error, params.real_miss_sim_miss_error,
                       params.range_min, params.range_max, params.ng_mode, getattr(params, "correspondence_type", 0))
        lib().emul_pf_update(self._h, C.c_uint32(len(poses)), _p(poses), _p(attrs), _p(Tsb), C.c_uint32(len(beams)), _p(beams), C.byref(prm))
        return attrs


def segment(origs_s, dirs_s, range_min, range_max, ranges_real, ranges_sim, normals_sim, min_scan, min_map):
    origs_s, dirs_s = _f32(origs_s).reshape(-1, 3), _f32(dirs_s).reshape(-1, 3)
    n = len(dirs_s)
    rr, rs, ns_ = _f32(ranges_real).reshape(-1), _f32(ranges_sim).reshape(-1), _f32(normals_sim).reshape(-1, 3)
    a, b, lab = np.zeros((n, 3), np.float32), np.zeros((n, 3), np.float32), np.zeros(n, np.uint8)
    na, nb = C.c_uint32(), C.c_uint32()
    lib().emul_segment(C.c_uint32(n), _p(origs_s), C.c_uint32(len(origs_s)), _p(dirs_s), C.c_float(range_min), C.c_float(range_max), _p(rr), _p(rs), _p(ns_),
                       C.c_float(min_scan), C.c_float(min_map), _p(a), C.byref(na), _p(b), C.byref(nb), _p(lab))
    return a[: na.value].copy(), b[: nb.value].copy(), lab


def gladiator(poses, attrs, first, n_local, cfg, seed, step):
    poses, attrs = np.ascontiguousarray(poses), np.ascontiguousarray(attrs)
    Pn, An = np.zeros(n_local, poses.dtype), np.zeros(n_local, attrs.dtype)
    raw, nrm = np.zeros(n_local, np.uint32), np.zeros((n_local, 6), np.float32)
    lib().emul_gladiator(C.c_uint32(len(poses)), _p(poses), _p(attrs), C.c_uint32(first), C.c_uint32(n_local), C.byref(cfg), C.c_uint64(seed), C.c_uint32(step),
                         _p(Pn), _p(An), _p(raw), _p(nrm))
    return Pn, An, raw, nrm


def cross_statistics(Tpre, dpts, dmask, mpts, mnrm, mmask, max_dist):
    out = np.zeros((), CROSS_STATS)
    dpts, mpts, mnrm = _f32(dpts), _f32(mpts), _f32(mnrm)
    dmask, mmask = np.ascontiguousarray(dmask, np.uint8), np.ascontiguousarray(mmask, np.uint8)
    Tpre = np.ascontiguousarray(Tpre)
    lib().emul_cross_statistics(_p(Tpre), C.c_uint32(len(dmask)), _p(dpts), _p(dmask), _p(mpts), _p(mnrm), _p(mmask), C.c_float(max_dist), _p(out))
    return out


def umeyama(stats):
    stats = np.ascontiguousarray(stats)
    out = np.zeros((), TRANSFORM)
    lib().emul_umeyama(_p(stats), _p(out))
    return out
