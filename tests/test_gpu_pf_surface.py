"""The surface constraint on the device (b2_pf_project_to_surface, PCDSensorUpdaterB200.projectToSurface, k_pf_surface).

* The device matches the product's pf_surface_one compiled for the host (tests/pf_surface_ref/, itself byte-identical to the C restatement
  on the CPU, tests/test_pf_surface.py) bit for bit: every CPU case, and n in {1, 127, 129, 100 003, 1 000 000} on synth.terrain and on
  building:1000000.
* Refusals launch nothing and leave both buffers as they were; two slices concatenate to the whole result.
* A deterministic drive up the ramp tracks its height and pitch; a whole init -> motion -> project -> sensor update -> Gladiator -> project
  -> estimateStats cycle tracks the true z and pitch."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import gpu_map, mesh
from pf_surface_ref import ProductScene
from test_pf_surface import (CFG_IDS, CONFIGS, PLANE_BOUND, TERRAIN_TRIS, _cfg, _lattice_cases, _marked, _mezzanine_cases, _on_plane,
                             _plane, _random_cases, _special_cases, _stairs_cases)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RAMP_SLOPE = math.atan2(3.0, 17.0)

_MAPS = {}


def _map(name):
    """device map and host-compiled product scene of 'terrain' (TERRAIN_TRIS), 'plane' or a conftest mesh name"""
    import rmcl_b200
    from rmcl_b200 import synth
    if name not in _MAPS:
        if name == "terrain":
            V, F = synth.terrain(TERRAIN_TRIS)
        elif name == "plane":
            V, F = _plane()
        else:
            V, F = mesh(name)
        gm = gpu_map(name) if name not in ("terrain", "plane") else rmcl_b200.Map(V, F, device=0)
        _MAPS[name] = (gm, ProductScene(V, F), (V, F))
    return _MAPS[name]


def _to_dev(P, A):
    import torch
    tp = torch.from_numpy(np.ascontiguousarray(P).view(np.float32).reshape(-1, 8).copy()).cuda()
    ta = torch.from_numpy(np.ascontiguousarray(A).view(np.float32).reshape(-1, 9).copy()).cuda()
    return tp, ta


def _to_np(tp, ta):
    from rmcl_b200.synth import PARTICLE_ATTR_DTYPE, TRANSFORM_DTYPE
    return tp.cpu().numpy().view(TRANSFORM_DTYPE).reshape(-1).copy(), ta.cpu().numpy().view(PARTICLE_ATTR_DTYPE).reshape(-1).copy()


def _device(name, P, A, cfg):
    import rmcl_b200
    import torch
    gm = _map(name)[0]
    up = rmcl_b200.PCDSensorUpdaterB200(gm)
    tp, ta = _to_dev(P, A)
    up.projectToSurface(tp, ta, cfg)
    torch.cuda.synchronize()
    return _to_np(tp, ta)


def _same(name, P, A, cfg):
    Pd, Ad = _device(name, P, A, cfg)
    Ph, Ah = _map(name)[1].project(P, A, cfg)
    assert Pd.tobytes() == Ph.tobytes()
    assert Ad.tobytes() == Ah.tobytes()
    return Pd, Ad


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
@pytest.mark.parametrize("case", ["random", "lattice", "mezzanine", "stairs", "special"])
def test_device_matches_host_on_terrain_cases(case, cfg):
    P, A = {"random": lambda: _random_cases(1), "lattice": lambda: _lattice_cases(2), "mezzanine": lambda: _mezzanine_cases(5),
            "stairs": lambda: _stairs_cases(4), "special": _special_cases}[case]()
    _same("terrain", P, A, cfg)
    _same("terrain", P, A, _cfg(probe_above=3.5, probe_below=1.0, base_height=cfg.base_height, align=cfg.align))


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_device_matches_host_on_plane(cfg):
    P, A = _on_plane(10)
    Pd, Ad = _same("plane", P, A, cfg)
    assert not _marked(Ad).any()
    for ms in (math.atan(math.hypot(0.25, 0.125)) + 1e-4, math.atan(math.hypot(0.25, 0.125)) - 1e-4):
        _same("plane", P, A, _cfg(max_slope=ms, align=cfg.align, base_height=cfg.base_height))


def _spread(n, lo, hi, seed):
    """n particles uniform in the box lo..hi with any heading and small tilts"""
    from rmcl_b200.synth import PARTICLE_ATTR_DTYPE, TRANSFORM_DTYPE
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(lo, hi, (n, 3))
    rpy = np.stack([rng.normal(0, 0.1, n), rng.normal(0, 0.1, n), rng.uniform(-math.pi, math.pi, n)], 1)
    P, A = np.zeros(n, TRANSFORM_DTYPE), np.zeros(n, PARTICLE_ATTR_DTYPE)
    P["t"] = xyz.astype(np.float32)
    P["stamp"] = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    A["likelihood"]["mean"] = rng.uniform(0.1, 1.0, n)
    A["likelihood"]["n_meas"] = rng.integers(0, 5000, n)
    A["state_sigma"] = rng.uniform(0.0, 1.0, (n, 6))
    cr, sr, cp, sp, cy, sy = (f(rpy[:, k] / 2) for k in range(3) for f in (np.cos, np.sin))
    P["R"] = np.stack([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy], 1).astype(np.float32)
    return P, A


@pytest.mark.parametrize("n", [1, 127, 129, 100_003, 1_000_000])
@pytest.mark.parametrize("name", ["terrain", "building:1000000"])
def test_device_matches_host_sizes(name, n):
    V = _map(name)[2][0]
    lo, hi = V.min(0).astype(np.float64) - [1.0, 1.0, 0.5], V.max(0).astype(np.float64) + [1.0, 1.0, 0.5]
    P, A = _spread(n, lo, hi, seed=n)
    for cfg in (_cfg(align=1), _cfg(base_height=0.3, align=0)):
        _same(name, P, A, cfg)


def test_refusals_launch_nothing():
    import rmcl_b200
    import torch
    from rmcl_b200.api import _chk, _devptr
    gm = _map("terrain")[0]
    up = rmcl_b200.PCDSensorUpdaterB200(gm)
    P, A = _random_cases(3)
    tp, ta = _to_dev(P, A)
    torch.cuda.synchronize()
    before = (tp.cpu().numpy().tobytes(), ta.cpu().numpy().tobytes())
    nan, inf = float("nan"), float("inf")
    bad = [_cfg(probe_above=nan), _cfg(probe_below=inf), _cfg(base_height=nan), _cfg(max_slope=nan), _cfg(probe_above=-0.1),
           _cfg(probe_below=-1.0), _cfg(probe_above=0.0, probe_below=0.0), _cfg(base_height=-0.01), _cfg(max_slope=-0.1), _cfg(max_slope=1.6),
           _cfg(align=2), _cfg(align=-1)]
    lib = rmcl_b200.load_library()
    k0 = rmcl_b200.kernel_launch_count()
    for cfg in bad:
        with pytest.raises(rmcl_b200.B2Error):
            up.projectToSurface(tp, ta, cfg)
    n = C.c_uint32(len(P))
    good = _cfg()
    for args in ((None, _devptr(tp), _devptr(ta), n, C.byref(good)), (up._h, None, _devptr(ta), n, C.byref(good)),
                 (up._h, _devptr(tp), None, n, C.byref(good)), (up._h, _devptr(tp), _devptr(ta), n, None)):
        with pytest.raises(rmcl_b200.B2Error):
            _chk(lib.b2_pf_project_to_surface(*args))
    # n == 0 is no work, with or without buffers; pi/2 as a float is accepted
    _chk(lib.b2_pf_project_to_surface(up._h, None, None, C.c_uint32(0), C.byref(good)))
    assert rmcl_b200.kernel_launch_count() == k0
    torch.cuda.synchronize()
    assert (tp.cpu().numpy().tobytes(), ta.cpu().numpy().tobytes()) == before
    up.projectToSurface(tp, ta, _cfg(max_slope=float(np.float32(math.pi / 2))))
    assert rmcl_b200.kernel_launch_count() == k0 + 1


def test_two_slices_concatenate_to_the_whole():
    import rmcl_b200
    import torch
    P, A = _random_cases(21)
    cfg = _cfg(base_height=0.2)
    whole = _device("terrain", P, A, cfg)
    up = rmcl_b200.PCDSensorUpdaterB200(_map("terrain")[0])
    tp, ta = _to_dev(P, A)
    k = 1111
    up.projectToSurface(tp[:k], ta[:k], cfg)
    up.projectToSurface(tp[k:], ta[k:], cfg)
    torch.cuda.synchronize()
    Ps, As = _to_np(tp, ta)
    assert Ps.tobytes() == whole[0].tobytes() and As.tobytes() == whole[1].tobytes()


def _ramp_height(x):
    from rmcl_b200 import synth
    r = synth.TERRAIN_RAMP
    return np.clip((np.asarray(x, np.float64) - r["x0"]) * r["rise"] / r["run"], 0.0, r["rise"])


def _pitch(R):
    """REP-103 pitch (rotation about y, nose up negative) of x y z w quaternions"""
    q = np.asarray(R, np.float64)
    return np.arcsin(np.clip(2.0 * (q[:, 3] * q[:, 1] - q[:, 2] * q[:, 0]), -1.0, 1.0))


FOOT = (3.0, 2.0)                     # 1 m before the ramp, on its centre line
FOOT_COV = np.diag([0.04, 0.09, 0.0, 0.0, 0.0, 0.0])


def test_ramp_drive():
    """initSamples at the foot of the ramp (x, y spread only), then 30 steps of body-frame odometry (0.2, 0, 0), each followed by
    projectToSurface(align 1).  Bound: every projection puts the particle on the surface afresh, so z carries the error of one projection,
    PLANE_BOUND (16 ulp at 16 m; the ramp stays below 21 m); its z-axis is the ramp's normal within 1e-6 rad (the plane test's bound), so
    with heading 0 its pitch is -atan(3/17) within 1e-6 rad.  Without the projection the same drive ends 0.5 to 1.2 m under the ramp (its x
    then lies between 7.5 and 10 m, where the ramp is 0.6 to 1.1 m high)."""
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    up = rmcl_b200.PCDSensorUpdaterB200(_map("terrain")[0])
    n = 20000
    pose = synth.make_transform((FOOT[0], FOOT[1], 0.0))
    step = synth.make_transform((0.2, 0.0, 0.0))
    runs = []
    for project in (True, False):
        tp, ta = torch.empty((n, 8), dtype=torch.float32, device="cuda"), torch.empty((n, 9), dtype=torch.float32, device="cuda")
        up.initSamples(tp, ta, pose, FOOT_COV, seed=5)
        for _ in range(30):
            up.motionUpdate(tp, ta, step, 0.0)
            if project:
                up.projectToSurface(tp, ta, _cfg(align=1))
        torch.cuda.synchronize()
        runs.append(_to_np(tp, ta))
    (P, A), (Q, _) = runs
    assert not _marked(A).any()
    x = P["t"][:, 0].astype(np.float64)
    assert x.min() > synth.TERRAIN_RAMP["x0"] + 2.0                                   # every particle is well up the ramp
    assert np.abs(P["t"][:, 2] - _ramp_height(x)).max() <= PLANE_BOUND
    assert np.abs(_pitch(P["R"]) + RAMP_SLOPE).max() <= 1e-6
    under = _ramp_height(Q["t"][:, 0]) - Q["t"][:, 2].astype(np.float64)
    assert np.all(Q["t"][:, 2] == 0.0) and under.min() >= 0.5 and under.max() <= 1.2


def _true_path(steps):
    """float64 model of the drive of FOOT: flat to the ramp's foot, then along it; -> (x, z, pitch) after each step"""
    x, p, out = FOOT[0], 0.0, []
    for _ in range(steps):
        x += 0.2 * math.cos(p)
        z = float(_ramp_height(x))
        p = -RAMP_SLOPE if x > 4.0 else 0.0
        out.append((x, z, p))
    return out


def test_full_cycle_tracks_the_ramp():
    """init -> 30 x (motion, project, sensor update with beams from the oracle's scans of synth.terrain at the true pose, Gladiator
    resampling, project, estimateStats).
    Bound, from the geometry and the particle spread: every particle sits on the surface (projected after every move), and the ramp is
    linear in x, so the weighted mean height differs from the true one by 3/17 of the mean's along-track error, plus PLANE_BOUND.  The
    initial spread is 0.2 m in x; Gladiator only copies particles and adds 0.03 m of noise per step, so after 30 steps the cloud lies within
    3 (0.2 + 0.03 sqrt(30)) = 1.1 m of its start and the mean's error is below 1.1 m: z within 0.2 m, against the 0.9 m the ramp rises in this
    run.  Once every particle is past the foot (x > 4), each has the ramp's pitch within 1e-6 rad apart from the 0.01 rad yaw noise, which
    changes the REP-103 pitch of a tilted body by at most slope * yaw^2 / 2 (yaw within 0.1 rad): the estimate's pitch within 2e-3 rad."""
    import rmcl_b200
    import torch
    from oracle import pyoracle as po
    from rmcl_b200 import synth
    gm, _, (V, F) = _map("terrain")
    osc = po.Scene(V, F)
    up = rmcl_b200.PCDSensorUpdaterB200(gm)
    Tsb = synth.scenario_tsb()
    m = synth.SphericalModel(np.radians(-30.0), np.radians(60.0) / 15, 16, -np.pi, 2 * np.pi / 128, 128, 0.3, 60.0)
    o, d = po.model_rays(m)
    prm = rmcl_b200.PFParams.defaults()
    glad = rmcl_b200.GladiatorConfig.defaults()
    n = 20000
    tp, ta = torch.empty((n, 8), dtype=torch.float32, device="cuda"), torch.empty((n, 9), dtype=torch.float32, device="cuda")
    up.initSamples(tp, ta, synth.make_transform((FOOT[0], FOOT[1], 0.0)), FOOT_COV, seed=9)
    step = synth.make_transform((0.2, 0.0, 0.0))
    rise, checked = 0.0, 0
    for k, (x, z, p) in enumerate(_true_path(30)):
        up.motionUpdate(tp, ta, step, 0.0)
        up.projectToSurface(tp, ta)
        Tgt = synth.make_transform((x, FOOT[1], z), (0.0, p, 0.0))
        scan = osc.simulate(Tgt, Tsb, o, d, m.range_max)
        up.update(tp, ta, Tsb, synth.pf_beams(scan["points"], 64, seed=k), prm)
        Pn, An = torch.empty_like(tp), torch.empty_like(ta)
        up.resample(tp, ta, Pn, An, glad, seed=9, step=k)
        tp, ta = Pn, An
        up.projectToSurface(tp, ta)
        est = up.estimateStats(tp, ta, max_induction_particles=n)
        assert abs(float(est["position"][2]) - z) <= 0.2 + PLANE_BOUND, (k, est["position"], z)
        P, _ = _to_np(tp, ta)
        if P["t"][:, 0].min() > 4.0:
            q = np.asarray(est["orientation"], np.float64).reshape(1, 4)
            assert abs(float(_pitch(q)[0]) - p) <= 2e-3, (k, q, p)
            checked += 1
        rise = z
    assert rise > 0.8 and checked >= 10


def test_cpp_classes_match_python(tmp_path):
    """tests/pf_surface_cpp/pf_surface_cpp.cpp, compiled here against include/rmcl_b200/rcc_b200.hpp, projects device particles through
    PCDSensorUpdaterB200::projectToSurface: byte for byte what the Python path gives"""
    import rmcl_b200
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "pf_surface_cpp")
    lib_dir = os.path.dirname(rmcl_b200.lib_path())
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(cuda, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "pf_surface_cpp", "pf_surface_cpp.cpp"), "-L" + lib_dir, "-lrmcl_b200",
                           "-L" + os.path.join(cuda, "lib64"), "-lcudart", "-Wl,-rpath," + lib_dir])
    _, _, (V, F) = _map("terrain")
    P, A = _random_cases(31)
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(np.array([len(V), len(F), len(P)], np.uint32).tobytes())
        for a in (V, F, P, A):
            f.write(np.ascontiguousarray(a).tobytes())
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "REFUSED" in r.stdout and "max_slope" in r.stdout
    P1, A1 = _device("terrain", P, A, rmcl_b200.SurfaceConfig.defaults())
    P2, A2 = _device("terrain", P1, A1, _cfg(align=0, base_height=0.25))
    assert np.fromfile(out, np.uint8).tobytes() == b"".join(a.tobytes() for a in (P1, A1, P2, A2))
