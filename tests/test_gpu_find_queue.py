"""k_rcc_find runs as one resident wave whose warps take 8x4-ray tiles from a per-handle ticket counter.  Every tile must be traced exactly
once whatever the scan's size, the tile order, the number of poses, the counter's value (it wraps around 2^32) or a second handle on another
stream; the model buffers must equal the oracle byte for byte."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("hits", "face_ids", "ranges", "points", "normals")
_SCENES = {}


def _scene(name):
    """(gpu map, oracle scene) of a synthetic mesh, built once per module"""
    import rmcl_b200
    from rmcl_b200 import synth
    from oracle import pyoracle
    if name not in _SCENES:
        kind, n = name.split(":")
        V, F = synth.building(int(n)) if kind == "building" else synth.indoor(int(n))
        _SCENES[name] = (rmcl_b200.Map(V, F, device=0), pyoracle.Scene(V, F))
    return _SCENES[name]


def _lib():
    import rmcl_b200
    return rmcl_b200.load_library()


def _case(case):
    """(scene, model, handle class, pose) of one scan shape"""
    import rmcl_b200
    from rmcl_b200 import synth
    rng = np.random.default_rng(2)
    if case == "C2":
        return "building:1000000", synth.c2_sensor(), rmcl_b200.RCCB200Spherical, synth.building_gt_pose()
    if case == "C4":
        return "indoor:500000", synth.c4_sensor(), rmcl_b200.RCCB200Pinhole, synth.indoor_gt_pose()
    if case == "raster":      # 12 288 tiles: above what the loop sorts, traced in raster order
        return "building:200000", synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 383, 384, -np.pi, 2 * np.pi / 1024, 1024, 0.5, 120.0), \
            rmcl_b200.RCCB200Spherical, synth.building_gt_pose()
    w, h = {"odd": (37, 13), "tiny": (5, 3)}[case]        # 481 rays (last tile partial), 15 rays (less than one warp)
    dirs = rng.normal(size=(w * h, 3)).astype(np.float32)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    return "indoor:20000", synth.O1DnModel(w, h, np.array([0.1, 0.0, 0.05], np.float32), dirs, 0.1, 20.0), rmcl_b200.RCCB200O1Dn, synth.indoor_gt_pose()


def _handle(case):
    from rmcl_b200 import synth
    from oracle import pyoracle
    name, m, cls, Tbm = _case(case)
    gmap, osc = _scene(name)
    h = cls(gmap)
    h.setTsb(synth.scenario_tsb()); h.setModel(m); h.setParams(1.0, 0.15)
    o, d = pyoracle.model_rays(m)
    return h, m, Tbm, osc.simulate(Tbm, synth.scenario_tsb(), o, d, m.range_max)


def _tickets(h, set_to=None):
    out = (C.c_uint * 3)()
    v = C.c_uint(set_to) if set_to is not None else None
    assert _lib().b2_rcc_debug_find_tickets(h._h, C.byref(v) if v is not None else None, out) == 0
    return int(out[0]), int(out[1]), int(out[2])


def _same_as(h, ref):
    mv = h.modelView()
    for k in KEYS:
        assert mv[k].tobytes() == ref[k].tobytes(), k


def _find_checked(h, Tbm, n_tiles):
    """one find: it consumed exactly n_tiles tickets and the host's count follows the device counter"""
    before, host_before, _ = _tickets(h)
    assert before == host_before
    h.find(Tbm)
    after, host_after, grid = _tickets(h)
    assert after == host_after and after == (before + n_tiles) % (1 << 32)
    assert 1 <= grid <= (n_tiles + 1) // 2


@pytest.mark.parametrize("case", ["C2", "C4", "odd", "tiny", "raster"])
def test_every_tile_once(case):
    import torch
    h, m, Tbm, ref = _handle(case)
    n_tiles = (m.size + 31) // 32
    stamps = torch.zeros(2 * n_tiles, dtype=torch.int64, device="cuda")
    assert _lib().b2_rcc_debug_find_warp_times(h._h, C.c_void_p(stamps.data_ptr())) == 0
    try:
        _find_checked(h, Tbm, n_tiles)
        t = stamps.cpu().numpy().reshape(-1, 2)
    finally:
        assert _lib().b2_rcc_debug_find_warp_times(h._h, None) == 0
    assert (t[:, 0] > 0).all() and (t[:, 1] >= t[:, 0]).all()          # every tile was started and finished
    _same_as(h, ref)
    # the tile durations: one per tile when the schedule is on (whole tiles, at most 11 520), each rewritten by every launch
    n = C.c_uint32(0)
    cost = np.zeros(n_tiles, np.uint32)
    assert _lib().b2_rcc_debug_tile_cost(h._h, C.c_void_p(cost.ctypes.data), C.c_uint32(n_tiles), C.byref(n), 1) == 0
    sched = m.size % 32 == 0 and 2 <= n_tiles <= 11520
    assert n.value == (n_tiles if sched else 0)
    for _ in range(2):
        _find_checked(h, Tbm, n_tiles)
        _same_as(h, ref)
        if sched:
            cost[:] = 0
            assert _lib().b2_rcc_debug_tile_cost(h._h, C.c_void_p(cost.ctypes.data), C.c_uint32(n_tiles), C.byref(n), 1) == 0
            assert (cost != 0xFFFFFFFF).all()


def test_multi_pose_find_keeps_the_queue():
    """the multi-pose find (unfused v1 benchmark) takes its tickets from the same counter: a find behind it still traces every tile"""
    from rmcl_b200 import synth
    h, m, Tbm, ref = _handle("raster")
    h.setRanges(ref["ranges"])
    n_tiles = (m.size + 31) // 32
    poses = np.stack([synth.compose(Tbm, synth.make_transform((0.01 * k, 0.0, 0.0))) for k in range(3)]).view(synth.TRANSFORM_DTYPE).reshape(-1)
    before, _, _ = _tickets(h)
    h.benchmark(poses, 2)
    after, host, _ = _tickets(h)
    tiles3 = (3 * m.size + 31) // 32
    assert after == host and after == (before + 2 * tiles3) % (1 << 32)
    _find_checked(h, Tbm, n_tiles)
    _same_as(h, ref)


def test_ticket_wrap():
    """1 000 consecutive finds on one handle with the counter started just below 2^32"""
    h, m, Tbm, ref = _handle("C2")
    n_tiles = m.size // 32
    start = (1 << 32) - 3 * n_tiles
    _tickets(h, start)
    crossed = False
    for k in range(1000):
        before = _tickets(h)[0] if k < 8 else None
        h.find(Tbm)
        if k < 8:
            after = _tickets(h)[0]
            crossed = crossed or after < before
            _same_as(h, ref)
        elif k % 97 == 0 or k == 999:
            _same_as(h, ref)
    assert crossed
    after, host, _ = _tickets(h)
    assert after == host and after == (start + 1000 * n_tiles) % (1 << 32)


def test_two_handles_two_streams():
    import torch
    from rmcl_b200 import synth
    (h1, m1, T1, r1), (h2, m2, T2, r2) = _handle("C2"), _handle("raster")
    T2b = synth.compose(T2, synth.make_transform((0.3, -0.2, 0.0), (0.0, 0.0, 0.4)))
    from oracle import pyoracle
    o2, d2 = pyoracle.model_rays(m2)
    r2 = _scene("building:200000")[1].simulate(T2b, synth.scenario_tsb(), o2, d2, m2.range_max)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    h1.setStream(s1.cuda_stream); h2.setStream(s2.cuda_stream)
    for _ in range(20):
        h1.find(T1); h2.find(T2b)
    torch.cuda.synchronize()
    _same_as(h1, r1); _same_as(h2, r2)
    for h in (h1, h2):
        dev, host, _ = _tickets(h)
        assert dev == host


_PDL_SCRIPT = r"""
import hashlib, numpy as np, rmcl_b200
from rmcl_b200 import synth
V, F = synth.building(1_000_000)
h = rmcl_b200.RCCB200Spherical(rmcl_b200.Map(V, F, device=0))
m = synth.c2_sensor()
h.setTsb(synth.scenario_tsb()); h.setModel(m); h.setParams(1.0, 0.15)
Tgt = synth.building_gt_pose()
h.find(Tgt)
h.setRanges(synth.noisy_ranges(h.modelView()["ranges"], m.range_max))
Tom, I = synth.compose(Tgt, synth.scenario_pose_offset()), synth.make_transform()
dig = hashlib.sha256()
for _ in range(4):
    for x in h.correctOnce(Tom, I, 5, 0.0):
        dig.update(np.ascontiguousarray(x).tobytes())
    mv = h.modelView()
    for k in sorted(mv):
        dig.update(np.ascontiguousarray(mv[k]).tobytes())
print(dig.hexdigest())
"""


def test_correct_once_same_with_and_without_early_launch():
    """B2_PDL is read once per process: each setting runs in its own interpreter"""
    out = {}
    for pdl in ("0", "1"):
        env = dict(os.environ, B2_PDL=pdl, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
        r = subprocess.run([sys.executable, "-s", "-c", _PDL_SCRIPT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        out[pdl] = r.stdout.strip().splitlines()[-1]
    assert out["0"] == out["1"]
