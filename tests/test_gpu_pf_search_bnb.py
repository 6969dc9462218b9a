"""GPU tests of the branch-and-bound global search (b2_pf_global_search_bnb, PCDSensorUpdaterB200.globalSearchBnB).

  * records: on every grid, the records equal b2_pf_global_search's records whose score is >= min_ratio * s*, byte for byte, with the same
    n_records at min_ratio 0; s* is the exhaustive search's best score.
  * above 2^30 candidates: a 200 x 200 x 32768 grid on building:1000000, checked against two exhaustive searches over x-tiles of it.
  * repeatability over calls, handles and two streams; no side effect on a later sensor update; refusals launch nothing."""
import math

import numpy as np
import pytest

import pf_search_ref as R
from conftest import gpu_map

pytestmark = pytest.mark.gpu

_FIELDS = {}
_TERRAIN = {}


class G:
    """the helpers of these tests: fields, beams, configs and scans"""

    @staticmethod
    def _field(name, h=0.05):
        import rmcl_b200
        if (name, h) not in _FIELDS:
            gmap = gpu_map(name)
            _FIELDS[(name, h)] = (gmap, rmcl_b200.DistanceField(gmap, h, 1.0))
        return _FIELDS[(name, h)]

    @staticmethod
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

    @staticmethod
    def _cfg(x0, y0, z0, step, nx, ny, K, max_records=16, sep_xy=0.0, sep_yaw=0.0):
        import rmcl_b200
        return rmcl_b200.SearchConfig(x0, y0, z0, step, nx, ny, K, max_records, sep_xy, sep_yaw)

    @staticmethod
    def _params(sigma=0.2):
        import rmcl_b200
        p = rmcl_b200.PFParams.defaults()
        p.dist_sigma = sigma
        return p

    @staticmethod
    def _tensor(a, width):
        import torch
        return torch.from_numpy(np.ascontiguousarray(a).view(np.float32).reshape(-1, width).copy()).cuda()

    @staticmethod
    def _surface(kind):
        import rmcl_b200
        if kind is None:
            return None
        s = rmcl_b200.SurfaceConfig.defaults()
        s.align = 1 if kind == "align1" else 0
        s.base_height = 0.5
        return s

    @staticmethod
    def _scan(gmap, Tgt, n_beams=180):
        """Tsb and n_beams beams of a 32 x 512 spherical scan from Tgt"""
        import rmcl_b200
        from rmcl_b200 import synth
        Tsb = synth.scenario_tsb()
        h = rmcl_b200.RCCB200Spherical(gmap)
        m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
        h.setTsb(Tsb); h.setModel(m); h.find(Tgt)
        return Tsb, synth.pf_beams(h.modelView()["points"], n_beams)


def _terrain():
    import rmcl_b200
    from rmcl_b200 import synth
    if not _TERRAIN:
        gmap = rmcl_b200.Map(*synth.terrain(200_000), device=0)
        _TERRAIN["f"] = (gmap, rmcl_b200.DistanceField(gmap, 0.05, 1.0))
    return _TERRAIN["f"]


def _building_scan(n_beams):
    """a scan from synth.building_gt_pose (the C3 scenario's pose) on building:1000000"""
    from rmcl_b200 import synth
    gmap, _ = G._field("building:1000000")
    return G._scan(gmap, synth.building_gt_pose(), n_beams)


def _check(up, f, Tsb, B, cfg, surface=None, prm=None, ratios=(0.0, 0.5, 1.0)):
    """the new call's records against the exhaustive call's at each min_ratio; -> the results"""
    prm = prm or G._params()
    res_x, recs_x = up.globalSearch(f, Tsb, B, cfg, surface, prm)
    out = []
    for ratio in ratios:
        res, recs = up.globalSearchBnB(f, Tsb, B, cfg, surface, prm, ratio)
        assert res["n_candidates"] == res_x["n_candidates"]
        if res_x["n_records"] == 0:
            assert res["n_records"] == 0 and res["best_score"] == -1.0
            continue
        best = np.float32(recs_x["score"][0])
        tau = np.float32(np.float32(ratio) * best)
        want = recs_x[recs_x["score"] >= tau]
        assert res["best_score"] == best and res["threshold"] == tau
        assert res["n_records"] == len(want), (ratio, res, res_x)
        assert recs.tobytes() == want.tobytes(), (ratio, recs, want)
        if ratio == 0.0:
            assert res["n_records"] == res_x["n_records"]
        assert res["n_passes"] == len(res["n_bounded_pass"]) and res["n_leaves"] == res["n_level"][0]
        out.append(res)
    return res_x, out


GRIDS = [  # name, (x0, y0, z0, step, nx, ny, K), surface, beams (int: random; "scan": the C3 scan), max_records, separations
    ("building:1000000", (0.1, 0.1, 0.5, 0.25, 239, 159, 72), None, "scan", 8, (1.0, math.radians(30))),        # the whole floor
    ("building:1000000", (20.0, 10.0, 0.5, 0.1, 200, 150, 180), None, "scan", 64, (1.0, math.radians(30))),
    ("building:1000000", (20.0, 10.0, 0.5, 0.1, 37, 23, 180), None, 180, 64, (0.0, 0.0)),
    ("building:1000000", (0.1, 0.1, 0.5, 0.25, 41, 29, 36), None, 1, 8, (1.0, math.radians(30))),
    ("building:1000000", (0.1, 0.1, 0.5, 0.25, 41, 29, 36), None, 0, 8, (1.0, math.radians(30))),
    ("building:1000000", (29.0, 19.0, 0.5, 0.25, 13, 1, 5), None, 180, 1, (0.0, 0.0)),
    ("terrain", (1.0, 1.0, 0.2, 0.25, 150, 100, 36), "align0", 180, 64, (1.0, math.radians(30))),
    ("terrain", (1.0, 1.0, 0.2, 0.25, 150, 100, 36), "align1", 180, 8, (0.0, 0.0)),
    ("terrain", (1.0, 1.0, 0.2, 0.25, 150, 100, 36), "align1", 1, 64, (1.0, math.radians(30))),
]


@pytest.mark.parametrize("name,grid,surf,beams,max_records,sep", GRIDS)
def test_records_equal_the_exhaustive_search(name, grid, surf, beams, max_records, sep):
    import rmcl_b200
    from rmcl_b200 import synth
    if name == "terrain":
        gmap, f = _terrain()
    else:
        gmap, f = G._field(name)
    if beams == "scan":
        Tsb, B = _building_scan(180)
    else:
        Tsb, B = synth.scenario_tsb(), G._beams(beams)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    cfg = G._cfg(*grid, max_records=max_records, sep_xy=sep[0], sep_yaw=sep[1])
    res_x, out = _check(up, f, Tsb, B, cfg, G._surface(surf))
    for r in out:
        print(f"{name} {grid} {surf} {beams}: {r['n_records']} records, passes {r['n_passes']}, leaves {r['n_leaves'] / r['n_candidates']:.4f}, "
              f"bounded {r['n_bounded']}, per level {r['n_level'][:r['depth'] + 1]}")


def test_the_square_rooms_four_symmetric_poses():
    import rmcl_b200
    gmap, f = G._field("cube29", 0.1)
    from rmcl_b200 import synth
    Tsb, B = G._scan(gmap, synth.make_transform((0.0, 0.0, -9.0), (0.0, 0.0, math.radians(20.0))))
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    for mr in (1, 8, 64):
        cfg = G._cfg(-2.0, -2.0, -9.0, 0.25, 17, 17, 72, max_records=mr, sep_xy=1.0, sep_yaw=math.radians(30))
        _check(up, f, Tsb, B, cfg)


def test_above_two_to_the_thirty_candidates():
    """200 x 200 x 32768 = 1.31e9 candidates.  x0 = 5 and y0 = 5 at step 0.25: every position is exact, so the tiles' positions (x0 + 99.75
    for the second) are the same bits.  Tile A: i in [0, 100), tile B: i in [99, 200) (one column of overlap)."""
    import rmcl_b200
    import torch
    gmap, f = G._field("building:1000000")
    Tsb, B = _building_scan(64)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    K = 32768
    cfg = G._cfg(5.0, 5.0, 0.5, 0.25, 200, 200, K, max_records=8, sep_xy=1.0, sep_yaw=math.radians(30))
    res, recs = up.globalSearchBnB(f, Tsb, B, cfg, None, G._params(), 0.0)
    assert res["n_candidates"] == 200 * 200 * K > 2 ** 30 and res["n_records"] >= 1
    print(res["n_records"], res["n_passes"], res["n_leaves"] / res["n_candidates"], res["n_level"][:res["depth"] + 1])
    best = None
    tiles = [(0, 100), (99, 101)]
    for i0, nxt in tiles:
        tc = G._cfg(float(np.float32(5.0) + np.float32(i0) * np.float32(0.25)), 5.0, 0.5, 0.25, nxt, 200, K, max_records=1)
        S = torch.empty(nxt * 200 * K, dtype=torch.float32, device="cuda")
        up.globalSearch(f, Tsb, B, tc, None, G._params(), S)
        m = S.max()
        idx = torch.nonzero(S == m).reshape(-1).cpu().numpy()
        # global c of each maximum: (k * ny + j) * nx + i0 + i
        i, j, k = idx % nxt + i0, idx // nxt % 200, idx // nxt // 200
        gc = ((k * 200 + j) * 200 + i).min()
        cand = (float(m), int(gc))
        if best is None or cand[0] > best[0] or (cand[0] == best[0] and cand[1] < best[1]):
            best = cand
        # every record inside this tile equals the tile's candidate there
        for r in recs:
            if i0 <= int(r["i"]) < i0 + nxt:
                tcs = (int(r["k"]) * 200 + int(r["j"])) * nxt + int(r["i"]) - i0
                assert np.float32(S[tcs].item()) == r["score"]
                P = R.poses(G._cfg(tc.x0 + 0.0, 5.0, 0.5, 0.25, nxt, 200, 1))          # position bits; the heading from the yaw table
                assert P["t"][int(r["j"]) * nxt + int(r["i"]) - i0].tobytes() == r["pose"]["t"].tobytes()
        del S
        torch.cuda.empty_cache()
    r0 = recs[0]
    assert (float(r0["score"]), (int(r0["k"]) * 200 + int(r0["j"])) * 200 + int(r0["i"])) == best


def test_repeats_over_calls_handles_and_streams_and_leaves_an_update_alone():
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    gmap, f = G._field("building:1000000")
    cfg = G._cfg(0.1, 0.1, 0.5, 0.25, 80, 60, 72, max_records=16, sep_xy=1.0, sep_yaw=0.5)
    Tsb, B = _building_scan(180)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    ups = [rmcl_b200.PCDSensorUpdaterB200(gmap) for _ in streams]
    outs = []
    for up, s in zip(ups, streams):
        up.setStream(s.cuda_stream)
        for _ in range(2):
            res, recs = up.globalSearchBnB(f, Tsb, B, cfg, G._surface("align1"), G._params(), 0.5)
            outs.append((res, recs.tobytes()))
    assert all(o == outs[0] for o in outs[1:])
    # a later sensor update is as it is without the search
    rng = np.random.default_rng(1)
    P = synth.transforms(20_000)
    P["t"] = np.stack([rng.uniform(1, 59, 20_000), rng.uniform(1, 39, 20_000), np.full(20_000, 0.5)], 1).astype(np.float32)
    after = []
    for search in (False, True):
        up = rmcl_b200.PCDSensorUpdaterB200(gmap)
        Pd, Ad = G._tensor(P, 8), torch.zeros((20_000, 9), dtype=torch.float32, device="cuda")
        Ad[:, 2] = 3.0
        if search:
            up.globalSearchBnB(f, Tsb, G._beams(64, seed=9), cfg, G._surface("align1"), G._params(), 0.0)
        up.setDistanceField(f)
        up.update(Pd, Ad, Tsb, G._beams(180), G._params())
        torch.cuda.synchronize()
        after.append((Pd.cpu().numpy().tobytes(), Ad.cpu().numpy().tobytes()))
    assert after[0] == after[1]


def test_refusals_launch_nothing_on_a_handle():
    import rmcl_b200
    from rmcl_b200 import synth
    gmap, f = G._field("cube29", 0.1)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    n0 = rmcl_b200.kernel_launch_count()
    for cfg, ratio in ((G._cfg(0, 0, 0, 0.25, 0, 4, 4), 0.0), (G._cfg(0, 0, 0, 0.25, (1 << 24) + 1, 4, 4), 0.0), (G._cfg(0, 0, 0, 0.25, 4, 4, 32769), 0.0),
                       (G._cfg(0, 0, 0, 0.25, 4, 4, 4), -0.1), (G._cfg(0, 0, 0, 0.25, 4, 4, 4), float("nan")), (G._cfg(0, 0, 0, 0.25, 4, 4, 4), 1.5)):
        with pytest.raises(rmcl_b200.B2Error):
            up.globalSearchBnB(f, synth.scenario_tsb(), G._beams(4), cfg, None, None, ratio)
    assert rmcl_b200.kernel_launch_count() == n0
