"""CPU tests of the global search (b2_pf_global_search): the product's functions compiled for the CPU (pf_search_ref/search_emul.cu) against
the C restatement of the definition (pf_search_ref/pf_search_ref.c, SURVEY appendix M) -- candidate poses, the per-cell surface probe with
its per-heading placement against pf_surface_pose on every candidate, the peak rule, the ranking and the separation pass -- and every
refusal of the C entry point (its arguments are checked before the handle), with no kernel launched."""
import ctypes as C
import math

import numpy as np
import pytest

import pf_search_ref as R
import rmcl_b200
from rmcl_b200 import synth


def cfg(x0=0.0, y0=0.0, z0=0.0, step=0.25, nx=4, ny=3, K=8, max_records=8, sep_xy=0.0, sep_yaw=0.0):
    return rmcl_b200.SearchConfig(x0, y0, z0, step, nx, ny, K, max_records, sep_xy, sep_yaw)


# ---------------------------------------------------------------- candidates
@pytest.mark.parametrize("K", [1, 2, 3, 72, 32768])
def test_candidate_poses_equal_the_restatement(K):
    nx, ny = (5, 3) if K < 32768 else (2, 1)
    c = cfg(-3.7, 12.1, 0.35, 0.3, nx, ny, K)
    want, got = R.poses(c), R.product_poses(c)
    assert got.tobytes() == want.tobytes()
    # x fastest, yaw slowest; psi_0 = -pi exactly, so q_0 = (0, 0, sin(-pi/2), cos(-pi/2)) = (0, 0, -1, 6e-17)
    assert got["t"][1, 0] == np.float32(np.float32(-3.7) + np.float32(1) * np.float32(0.3))
    assert got["R"][0, 2] == np.float32(-1.0) and got["R"][0, 3] == np.float32(math.cos(-math.pi / 2))
    last = got[-1]
    assert last["R"][2] == np.float32(math.sin((-math.pi + 2 * math.pi * (K - 1) / K) / 2))
    assert (got["stamp"] == 0).all() and (got["R"][:, :2] == 0).all()


def test_positions_far_from_the_origin_round_as_the_field_places_nodes():
    c = cfg(1.0e6, -2.5e5, 3.0, 0.1, 50, 7, 1)
    got = R.product_poses(c)
    i = np.arange(50, dtype=np.float32)
    assert np.array_equal(got["t"][:50, 0], (np.float32(1.0e6) + i * np.float32(0.1)).astype(np.float32))


def _ramp_stairs_walls():
    """a floor, a 20 deg ramp, three stair steps, a wall and a hole: every kind of cell the probe meets"""
    V, F = [], []

    def quad(a, b, c, d):
        k = len(V)
        V.extend([a, b, c, d])
        F.extend([[k, k + 1, k + 2], [k, k + 2, k + 3]])

    quad([0, 0, 0], [4, 0, 0], [4, 4, 0], [0, 4, 0])                                  # floor
    t = math.tan(math.radians(20.0))
    quad([4, 0, 0], [8, 0, 4 * t], [8, 4, 4 * t], [4, 4, 0])                          # ramp
    for s in range(3):                                                                 # stairs, rising in y
        z = 0.15 * (s + 1)
        quad([0, 4 + s, z], [4, 4 + s, z], [4, 5 + s, z], [0, 5 + s, z])
        quad([0, 4 + s, z - 0.15], [4, 4 + s, z - 0.15], [4, 4 + s, z], [0, 4 + s, z])
    quad([2, 0, 0], [2, 0, 2], [2, 4, 2], [2, 4, 0])                                  # wall at x = 2
    # x in [8, 10]: no ground (the hole)
    return np.array(V, np.float32), np.array(F, np.uint32)


@pytest.mark.parametrize("align", [0, 1])
@pytest.mark.parametrize("K", [1, 2, 3, 72])
def test_cell_probe_plus_placement_equals_the_rule_on_every_candidate(align, K):
    V, F = _ramp_stairs_walls()
    scene = R.ProductScene(V, F)
    s = rmcl_b200.SurfaceConfig(0.5, 1.0, 0.3, 0.6, align)
    c = cfg(-0.9, -0.45, 0.2, 0.5, 23, 17, K)
    a, va = scene.candidates(c, s, mode=1)
    b, vb = scene.candidates(c, s, mode=2)
    assert np.array_equal(va, vb) and a.tobytes() == b.tobytes()
    n_cells = c.nx * c.ny
    assert 0 < va[:n_cells].sum() < n_cells                          # ground and no ground both occur
    if align:
        # the rule tilts onto the ramp: some candidates leave the flat chart
        assert (np.abs(a["R"][va][:, :2]) > 1e-3).any()


def test_rotated_axis_is_not_always_e_z_exactly():
    """why the placement stays per heading: R_k e_z is e_z only up to rounding (sin^2 + cos^2 in float, signed zeros)"""
    K = 72
    half = (-math.pi + 2 * math.pi * np.arange(K) / K) / 2
    s, c = np.sin(half).astype(np.float32), np.cos(half).astype(np.float32)
    assert ((s * s + c * c) != np.float32(1.0)).any()


# ---------------------------------------------------------------- peaks
def _peaks_both(S, nx, ny, K):
    S = np.asarray(S, np.float32).reshape(-1)
    flags, nv, npk = R.peaks(S, nx, ny, K)
    assert np.array_equal(R.product_peaks(S, nx, ny, K), flags)
    assert npk == flags.sum() and nv == (S >= 0).sum()
    return flags.reshape(K, ny, nx)


def test_plateau_keeps_its_smallest_index():
    S = np.zeros((3, 4, 5), np.float32)
    S[1, 1:3, 1:4] = 2.0
    f = _peaks_both(S, 5, 4, 3)
    assert f.sum() == 1 and f[1, 1, 1]


def test_all_zero_scores_peak_at_zero_alone_and_single_cells():
    f = _peaks_both(np.zeros((4, 3, 5)), 5, 3, 4)
    assert f.sum() == 1 and f.reshape(-1)[0]
    f = _peaks_both([0.0], 1, 1, 1)
    assert f.sum() == 1
    f = _peaks_both([-1.0], 1, 1, 1)
    assert f.sum() == 0
    for K in (1, 2, 3):
        f = _peaks_both(np.arange(K, dtype=np.float32), 1, 1, K)
        assert f.sum() == 1 and f.reshape(-1)[K - 1]


def test_ridge_across_the_yaw_wrap_and_grid_edges():
    K, ny, nx = 8, 3, 3
    S = np.zeros((K, ny, nx), np.float32)
    S[K - 1, 0, 0], S[0, 0, 0] = 5.0, 5.0                           # equal across the wrap: the smaller index wins
    S[3, 2, 2] = 4.0                                                # a corner peak
    f = _peaks_both(S, nx, ny, K)
    assert f[0, 0, 0] and not f[K - 1, 0, 0] and f[3, 2, 2]
    S[K - 1, 0, 0] = 6.0
    f = _peaks_both(S, nx, ny, K)
    assert f[K - 1, 0, 0] and not f[0, 0, 0]
    # i and j do not wrap: a high value at the far edge is no neighbour of the near edge
    S = np.zeros((1, 1, 6), np.float32)
    S[0, 0, 0], S[0, 0, 5] = 1.0, 2.0
    f = _peaks_both(S, 6, 1, 1)
    assert f[0, 0, 0] and f[0, 0, 5]


def test_invalid_neighbours_are_ignored():
    S = np.full((3, 3, 3), -1.0, np.float32)
    S[1, 1, 1] = 0.5
    S[0, 0, 0] = 0.1
    f = _peaks_both(S, 3, 3, 3)
    assert f[1, 1, 1] and not f[0, 0, 0]                            # k = 0 and k = 2 are neighbours through the wrap
    S = np.full((5, 3, 3), -1.0, np.float32)
    S[0, 0, 0], S[2, 2, 2] = 0.1, 0.1                               # not neighbours (k differs by 2 of 5)
    f = _peaks_both(S, 3, 3, 5)
    assert f[0, 0, 0] and f[2, 2, 2]


@pytest.mark.parametrize("shape,seed", [((7, 5, 3), 1), ((72, 9, 11), 2), ((2, 4, 4), 3), ((1, 6, 6), 4), ((36, 1, 30), 5)])
def test_random_and_quantised_score_arrays(shape, seed):
    rng = np.random.default_rng(seed)
    S = rng.integers(0, 4, shape).astype(np.float32) * np.float32(0.25)   # many ties
    S[rng.random(shape) < 0.15] = -1.0
    K, ny, nx = shape
    f = _peaks_both(S, nx, ny, K)
    # two neighbours are never both peaks: at most one per 2 x 2 x 2 block
    assert f.sum() <= ((nx + 1) // 2) * ((ny + 1) // 2) * ((K + 1) // 2)


# ---------------------------------------------------------------- ranking and separation
def _records_both(S, peaks, c):
    S = np.asarray(S, np.float32)
    want = R.records(S, peaks, c)
    got = R.product_records(S, peaks, c)
    assert np.array_equal(got, want)
    return got


def test_ranking_breaks_ties_by_the_smaller_index():
    c = cfg(nx=10, ny=1, K=1, max_records=8)
    S = np.array([1, 3, 3, 2, 3, 0, 0, 2, 1, 3], np.float32)
    assert list(_records_both(S, [9, 4, 2, 1, 7, 3, 0], c)) == [1, 2, 4, 9, 3, 7, 0]
    c.max_records = 3
    assert list(_records_both(S, [9, 4, 2, 1, 7, 3, 0], c)) == [1, 2, 4]
    assert list(_records_both(S, [], c)) == []


def test_separation_needs_both_distances():
    K = 8                                                           # psi step 45 deg
    c = cfg(0.0, 0.0, 0.0, 1.0, 10, 1, K, max_records=8, sep_xy=2.5, sep_yaw=math.radians(50.0))
    idx = lambda i, k: k * 10 + i                                   # noqa: E731
    S = np.zeros(10 * K, np.float32)
    S[idx(0, 0)] = 9.0
    S[idx(2, 1)] = 8.0                                              # 2 m, 45 deg: both within, dropped
    S[idx(2, 2)] = 7.0                                              # 2 m, 90 deg: kept
    S[idx(3, 0)] = 6.0                                              # 3 m: kept
    S[idx(1, K - 1)] = 5.0                                          # 1 m, 45 deg across the wrap: dropped
    S[idx(2, 3)] = 5.0                                              # 2 m from (2, 2) at 45 deg: dropped; 2 m / 135 deg from (0, 0)
    peaks = [idx(0, 0), idx(2, 1), idx(2, 2), idx(3, 0), idx(1, K - 1), idx(2, 3)]
    assert list(_records_both(S, peaks, c)) == [idx(0, 0), idx(2, 2), idx(3, 0)]
    c.min_separation_xy, c.min_separation_yaw = 0.0, 0.0           # 0 / 0 keeps every peak
    assert len(_records_both(S, peaks, c)) == 6
    c.min_separation_xy, c.min_separation_yaw = 2.0, math.pi       # strictly within: exactly 2 m is not; every heading is within pi
    assert list(_records_both(S, peaks, c)) == [idx(0, 0), idx(2, 1)]


def test_random_peak_lists_with_ties():
    rng = np.random.default_rng(11)
    c = cfg(-5.0, 3.0, 0.0, 0.3, 40, 30, 36, max_records=64, sep_xy=1.0, sep_yaw=math.radians(30.0))
    S = (rng.integers(0, 20, 40 * 30 * 36) * 0.05).astype(np.float32)
    peaks = rng.choice(len(S), 3000, replace=False)
    got = _records_both(S, peaks, c)
    assert len(got) == 64 and S[got[0]] == S[peaks].max()


# ---------------------------------------------------------------- refusals
def _call(h=None, f=C.c_void_p(1), Tsb=True, beams=None, n_beams=0, prm=None, c=None, surface=None, records=True, scores=None, out=True):
    lib = rmcl_b200.load_library()
    T = np.zeros((), synth.TRANSFORM_DTYPE)
    recs = np.zeros(64, synth.SEARCH_RECORD_DTYPE)
    res = np.full(4, 7, np.uint64)
    p = prm if prm is not None else rmcl_b200.PFParams.defaults()
    cc = c if c is not None else cfg()
    rc = lib.b2_pf_global_search(h, f, C.c_void_p(T.ctypes.data) if Tsb else None, beams, C.c_uint32(n_beams), C.byref(p) if p is not False else None,
                                 C.byref(cc) if cc is not False else None, None if surface is None else C.byref(surface),
                                 C.c_void_p(recs.ctypes.data) if records else None, scores, C.c_void_p(res.ctypes.data) if out else None)
    assert (recs.view(np.uint8) == 0).all() and (res == 7).all()            # nothing written
    return rc, lib.b2_last_error().decode()


def test_refusals_launch_nothing():
    n0 = rmcl_b200.kernel_launch_count()
    assert "null argument 'h'" in _call()[1]                                 # valid arguments reach the handle
    assert "null argument 'f'" in _call(f=None)[1]
    bad_sigma = rmcl_b200.PFParams.defaults()
    tiny = rmcl_b200.PFParams.defaults()
    tiny.dist_sigma = 1e-30
    nan_sigma = rmcl_b200.PFParams.defaults()
    nan_sigma.dist_sigma = float("nan")
    bad_sigma.dist_sigma = 0.0
    s_bad = rmcl_b200.SurfaceConfig(0.5, 1.0, 0.0, 2.0, 1)
    s_align = rmcl_b200.SurfaceConfig(0.5, 1.0, 0.0, 0.6, 2)
    inf = float("inf")
    cases = [
        (dict(Tsb=False), "null argument 'Tsb'"), (dict(prm=False), "null argument 'prm'"), (dict(c=False), "null argument 'cfg'"),
        (dict(records=False), "null argument 'records_host'"), (dict(out=False), "null argument 'out_host'"),
        (dict(n_beams=3), "null argument 'beams'"),
        (dict(c=cfg(nx=0)), "grid"), (dict(c=cfg(ny=0)), "grid"), (dict(c=cfg(K=0)), "grid"), (dict(c=cfg(K=32769)), "grid"),
        (dict(c=cfg(nx=32768, ny=32768, K=2)), "2^30"), (dict(c=cfg(nx=1 << 15, ny=1 << 15, K=1, step=1.0)), None),
        (dict(c=cfg(step=0.0)), "step"), (dict(c=cfg(step=-0.25)), "step"), (dict(c=cfg(step=float("nan"))), "step"), (dict(c=cfg(step=inf)), "step"),
        (dict(c=cfg(x0=float("nan"))), "not finite"), (dict(c=cfg(y0=inf)), "not finite"), (dict(c=cfg(z0=-inf)), "not finite"),
        (dict(c=cfg(x0=3.0e38, step=1.0e38, nx=5)), "not finite"),
        (dict(c=cfg(max_records=0)), "max_records"), (dict(c=cfg(max_records=65)), "max_records"),
        (dict(c=cfg(sep_xy=-1.0)), "separations"), (dict(c=cfg(sep_yaw=float("nan"))), "separations"), (dict(c=cfg(sep_xy=inf)), "separations"),
        (dict(prm=bad_sigma), "dist_sigma"), (dict(prm=nan_sigma), "dist_sigma"), (dict(prm=tiny), "dist_sigma"),
        (dict(surface=s_bad), "max_slope"), (dict(surface=s_align), "align"),
    ]
    for kw, want in cases:
        rc, msg = _call(**kw)
        if want is None:                                                    # 2^30 candidates exactly: accepted
            assert "null argument 'h'" in msg, (kw, msg)
        else:
            assert rc == -1 and want in msg, (kw, want, msg)
    # 64 records and a good surface pass the checks
    assert "null argument 'h'" in _call(c=cfg(max_records=64), surface=rmcl_b200.SurfaceConfig.defaults())[1]
    assert rmcl_b200.kernel_launch_count() == n0


def test_config_defaults_cover_the_box():
    c = rmcl_b200.SearchConfig.defaults((0.1, 0.1), (59.9, 39.9), 0.5)
    assert (c.nx, c.ny, c.n_yaw, c.max_records) == (240, 160, 72, 8) and c.step == 0.25 and c.z0 == 0.5
    assert rmcl_b200.SearchConfig.defaults().nx == 0                        # no box: the grid is left for the caller
    assert synth.SEARCH_RECORD_DTYPE.itemsize == 48
