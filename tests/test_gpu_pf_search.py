"""GPU tests of the global search (b2_pf_global_search, PCDSensorUpdaterB200.globalSearch).

  * scores: every entry of the likelihood map equals b2_pf_sensor_update_field on the materialised candidate, from attributes {0, 0, 0}, bit
    for bit; with surface the candidates are materialised by projectToSurface, and those it marks score -1.
  * records: the counts and records equal the C restatement (tests/pf_search_ref.py) applied to the device's score array; a record's pose
    is its materialised candidate.
  * repeatability over calls, handles and two streams; localisation on building:1000000; the symmetric poses of a cube room; no side effects
    on a later sensor update."""
import math

import numpy as np
import pytest

import pf_search_ref as R
from conftest import gpu_map

pytestmark = pytest.mark.gpu

_FIELDS = {}


def _field(name, h=0.05):
    import rmcl_b200
    if (name, h) not in _FIELDS:
        gmap = gpu_map(name)
        _FIELDS[(name, h)] = (gmap, rmcl_b200.DistanceField(gmap, h, 1.0))
    return _FIELDS[(name, h)]


def _beams(k, seed=3):
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    B = np.zeros(k, synth.RANGE_MEAS_DTYPE)
    a = rng.uniform(-np.pi, np.pi, k)
    el = rng.uniform(-0.3, 0.3, k)
    B["dir"] = np.stack([np.cos(a) * np.cos(el), np.sin(a) * np.cos(el), np.sin(el)], 1).astype(np.float32)
    B["range"] = rng.uniform(0.5, 8.0, k).astype(np.float32)
    B["orig"] = [0.05, 0.0, 0.2]
    return B


def _cfg(x0, y0, z0, step, nx, ny, K, max_records=16, sep_xy=0.0, sep_yaw=0.0):
    import rmcl_b200
    return rmcl_b200.SearchConfig(x0, y0, z0, step, nx, ny, K, max_records, sep_xy, sep_yaw)


def _params(sigma=0.2):
    import rmcl_b200
    p = rmcl_b200.PFParams.defaults()
    p.dist_sigma = sigma
    return p


def _tensor(a, width):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.float32).reshape(-1, width).copy()).cuda()


def _field_update(up, f, P, Tsb, B, prm):
    """likelihood.mean of b2_pf_sensor_update_field on poses P from {0, 0, 0}"""
    import torch
    from rmcl_b200 import synth
    up.setDistanceField(f)
    A = torch.zeros((len(P), 9), dtype=torch.float32, device="cuda")
    up.update(_tensor(P, 8), A, Tsb, B, prm)
    return A.cpu().numpy().reshape(-1).view(synth.PARTICLE_ATTR_DTYPE)["likelihood"]["mean"]


def _search(up, f, Tsb, B, cfg, surface=None, prm=None):
    import torch
    n = cfg.nx * cfg.ny * cfg.n_yaw
    S = torch.empty(n, dtype=torch.float32, device="cuda")
    res, recs = up.globalSearch(f, Tsb, B, cfg, surface, prm or _params(), S)
    return res, recs, S.cpu().numpy()


GRIDS = [  # name, cfg, surface, beams
    ("building:1000000", (30.0, 20.0, 0.5, 0.25, 7, 5, 3), None, 1),
    ("building:1000000", (0.1, 0.1, 0.5, 0.25, 40, 30, 36), None, 180),
    ("building:1000000", (0.1, 0.1, 0.5, 0.25, 40, 30, 36), None, 0),
    ("building:1000000", (-1.0, -1.0, 0.3, 0.5, 125, 85, 72), "align0", 180),
    ("building:1000000", (20.0, 10.0, 0.3, 0.1, 100, 100, 100), None, 180),       # 10^6 candidates
    ("indoor:500000", (0.0, 0.0, 0.4, 0.2, 60, 40, 24), "align1", 180),
    ("indoor:500000", (0.0, 0.0, 0.4, 0.2, 60, 40, 24), "align1", 1),
    ("indoor:500000", (0.0, 0.0, 0.4, 0.2, 60, 40, 24), "align1", 0),
]


def _surface(kind):
    import rmcl_b200
    if kind is None:
        return None
    s = rmcl_b200.SurfaceConfig.defaults()
    s.align = 1 if kind == "align1" else 0
    s.base_height = 0.5
    return s


@pytest.mark.parametrize("name,grid,surf,n_beams", GRIDS)
def test_scores_equal_the_field_update_and_records_the_restatement(name, grid, surf, n_beams):
    import rmcl_b200
    from rmcl_b200 import synth
    gmap, f = _field(name)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    cfg = _cfg(*grid, max_records=64, sep_xy=1.0, sep_yaw=math.radians(30))
    B, Tsb, prm = _beams(n_beams), synth.scenario_tsb(), _params()
    surface = _surface(surf)
    res, recs, S = _search(up, f, Tsb, B, cfg, surface, prm)
    P = R.poses(cfg)
    valid = np.ones(len(P), bool)
    if surface is not None:
        import torch
        Pd, Ad = _tensor(P, 8), torch.zeros((len(P), 9), dtype=torch.float32, device="cuda")
        up.projectToSurface(Pd, Ad, surface)
        P = Pd.cpu().numpy().reshape(-1).view(synth.TRANSFORM_DTYPE)
        valid = Ad.cpu().numpy()[:, 2] == 0.0                     # the mark: n_meas 10000
    want = np.full(len(P), -1.0, np.float32)
    want[valid] = _field_update(up, f, P[valid], Tsb, B, prm)
    bad = np.flatnonzero(S.view(np.uint32) != want.view(np.uint32))
    assert len(bad) == 0, f"{len(bad)} scores differ, first {bad[:5]}: {S[bad[:5]]} vs {want[bad[:5]]}"
    hres, kept = R.host_result(S, cfg)
    assert res == hres
    assert np.array_equal(recs["i"] + cfg.nx * (recs["j"] + cfg.ny * recs["k"]), kept)
    assert recs["score"].tobytes() == S[kept].tobytes()
    assert recs["pose"].tobytes() == P[kept].tobytes()
    print(f"{name} {grid} {surf} {n_beams} beams: {res}, best {recs['score'][:3]}")


def test_repeats_over_calls_handles_and_streams():
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    gmap, f = _field("building:1000000")
    cfg = _cfg(0.1, 0.1, 0.5, 0.25, 80, 60, 72, max_records=16, sep_xy=1.0, sep_yaw=0.5)
    B, Tsb = _beams(180), synth.scenario_tsb()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    ups = [rmcl_b200.PCDSensorUpdaterB200(gmap) for _ in streams]
    outs = []
    for up, s in zip(ups, streams):
        up.setStream(s.cuda_stream)
        for _ in range(2):
            res, recs, S = _search(up, f, Tsb, B, cfg, _surface("align1"))
            outs.append((res, recs.tobytes(), S.tobytes()))
    assert all(o == outs[0] for o in outs[1:])


def _scan(gmap, Tgt, n_beams=180):
    import rmcl_b200
    from rmcl_b200 import synth
    Tsb = synth.scenario_tsb()
    h = rmcl_b200.RCCB200Spherical(gmap)
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(m); h.find(Tgt)
    return Tsb, synth.pf_beams(h.modelView()["points"], n_beams)


def _yaw(T):
    return 2 * math.atan2(float(T["R"][2]), float(T["R"][3]))


def _wrap(a):
    return (a + math.pi) % (2 * math.pi) - math.pi


@pytest.mark.parametrize("surf", [None, "align0"])
def test_record_zero_is_at_the_true_pose_on_the_building(surf):
    """The building is the same after a half turn about its centre, and its 5 m bays, each with a door in the middle of every wall, repeat:
    from most poses a scan sees one bay, which fits every bay equally well (at synth.building_gt_pose the top score is shared by bays 5 m
    apart).  So the pose stands where two lines of doors cross, and its beams reach the outer walls both ways; the grid covers the half
    x < 30 m that holds the pose and not its twin, and passes through the pose."""
    import rmcl_b200
    from rmcl_b200 import synth
    gmap, f = _field("building:1000000")
    Tgt = synth.make_transform((2.5, 22.5, 0.5), (0.0, 0.0, math.radians(30.0)))
    Tsb, B = _scan(gmap, Tgt, 2000)
    step, K = 0.25, 72
    cfg = rmcl_b200.SearchConfig.defaults((0.25, 0.25), (29.9, 39.9), 0.5, step)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    res, recs = up.globalSearch(f, Tsb, B, cfg, _surface(surf), _params())
    r0 = recs[0]
    d = math.hypot(float(r0["pose"]["t"][0]) - float(Tgt["t"][0]), float(r0["pose"]["t"][1]) - float(Tgt["t"][1]))
    dy = abs(_wrap(_yaw(r0["pose"]) - _yaw(Tgt)))
    print(f"{surf}: {res}; record 0 at {r0['pose']['t']} yaw {math.degrees(_yaw(r0['pose'])):.1f}, score {r0['score']:.4f}; "
          f"next {recs['score'][1:4]} at {recs['pose']['t'][1:4].tolist()}; error {d:.3f} m {math.degrees(dy):.2f} deg")
    assert d <= step / math.sqrt(2) + 1e-6 and dy <= math.pi / K + 1e-9


def test_a_square_room_gives_its_four_symmetric_poses():
    import rmcl_b200
    from rmcl_b200 import synth
    gmap, f = _field("cube29", 0.1)
    Tgt = synth.make_transform((0.0, 0.0, -9.0), (0.0, 0.0, math.radians(20.0)))
    Tsb, B = _scan(gmap, Tgt)
    cfg = _cfg(-2.0, -2.0, -9.0, 0.25, 17, 17, 72, max_records=8, sep_xy=1.0, sep_yaw=math.radians(30))
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    res, recs = up.globalSearch(f, Tsb, B, cfg, None, _params())
    print(res, recs["score"], recs["i"], recs["j"], recs["k"])
    top = recs[:4]
    yaws = sorted(round(math.degrees(_wrap(_yaw(r["pose"]) - _yaw(Tgt)))) % 360 for r in top)
    assert yaws == [0, 90, 180, 270]
    assert np.abs(top["pose"]["t"][:, :2]).max() <= 0.25 / math.sqrt(2) + 1e-6
    assert top["score"].min() >= 0.99 * top["score"].max()
    assert len(recs) == 4 or recs["score"][4] < 0.9 * top["score"].min()


def test_a_search_leaves_a_later_sensor_update_as_it_was():
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    gmap, f = _field("building:1000000")
    rng = np.random.default_rng(1)
    P = synth.transforms(50_000)
    P["t"] = np.stack([rng.uniform(1, 59, 50_000), rng.uniform(1, 39, 50_000), np.full(50_000, 0.5)], 1).astype(np.float32)
    B, Tsb = _beams(180), synth.scenario_tsb()
    outs = []
    for search in (False, True):
        up = rmcl_b200.PCDSensorUpdaterB200(gmap)
        Pd, Ad = _tensor(P, 8), torch.zeros((50_000, 9), dtype=torch.float32, device="cuda")
        Ad[:, 2] = 3.0
        if search:
            _search(up, f, Tsb, _beams(64, seed=9), _cfg(0.1, 0.1, 0.5, 0.5, 100, 60, 36), _surface("align1"))
        up.setDistanceField(f)
        up.update(Pd, Ad, Tsb, B, _params())
        torch.cuda.synchronize()
        outs.append((Pd.cpu().numpy().tobytes(), Ad.cpu().numpy().tobytes()))
    assert outs[0] == outs[1]


def test_refusals_launch_nothing_on_a_handle():
    import rmcl_b200
    from rmcl_b200 import synth
    gmap, f = _field("cube29", 0.1)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    n0 = rmcl_b200.kernel_launch_count()
    for cfg in (_cfg(0, 0, 0, 0.25, 0, 4, 4), _cfg(0, 0, 0, -1.0, 4, 4, 4), _cfg(0, 0, 0, 0.25, 4, 4, 32769), _cfg(0, 0, 0, 0.25, 4, 4, 4, max_records=65)):
        with pytest.raises(rmcl_b200.B2Error):
            up.globalSearch(f, synth.scenario_tsb(), _beams(4), cfg)
    assert rmcl_b200.kernel_launch_count() == n0
