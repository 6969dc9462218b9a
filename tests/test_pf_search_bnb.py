"""CPU tests of the branch-and-bound global search (b2_pf_global_search_bnb): the product's pyramid and bound compiled for the CPU
(pf_search_bnb_ref/bnb_emul.cu) -- the pyramid equals a numpy restatement from the field's raw layout byte for byte, and every node's
bound is >= the exact score of every valid candidate in its block, at every level -- and the entry point's refusals, with no launch."""
import ctypes as C
import math

import numpy as np
import pytest

import pf_search_bnb_ref as R
import rmcl_b200
from rmcl_b200 import synth


def _ramp_stairs_walls():
    """a floor, a 20 deg ramp, three stair steps, a wall and a hole (tests/test_pf_search.py's map)"""
    V, F = [], []

    def quad(a, b, c, d):
        k = len(V)
        V.extend([a, b, c, d])
        F.extend([[k, k + 1, k + 2], [k, k + 2, k + 3]])

    quad([0, 0, 0], [4, 0, 0], [4, 4, 0], [0, 4, 0])
    t = math.tan(math.radians(20.0))
    quad([4, 0, 0], [8, 0, 4 * t], [8, 4, 4 * t], [4, 4, 0])
    for s in range(3):
        z = 0.15 * (s + 1)
        quad([0, 4 + s, z], [4, 4 + s, z], [4, 5 + s, z], [0, 5 + s, z])
        quad([0, 4 + s, z - 0.15], [4, 4 + s, z - 0.15], [4, 4 + s, z], [0, 4 + s, z])
    quad([2, 0, 0], [2, 0, 2], [2, 4, 2], [2, 4, 0])
    return np.array(V, np.float32), np.array(F, np.uint32)


_FIELDS = {}


def _field(name):
    if name not in _FIELDS:
        if name == "building":
            V, F = synth.building(20_000)
            V = V[:, :] * np.float32(0.25)                                  # a 15 x 10 m storey: a small field
            _FIELDS[name] = R.Field(V, F, 0.1, 0.5)
        elif name == "building_far":
            V, F = synth.building(20_000)
            V = (V * np.float32(0.25) + np.float32([1.0e6, 1.0e6, 0.0])).astype(np.float32)
            _FIELDS[name] = R.Field(V, F, 0.1, 0.5)
        elif name == "terrain":
            V, F = synth.terrain(20_000)
            keep = (V[F].max(1)[:, 0] < 24.0) & (V[F].max(1)[:, 1] < 16.0)
            _FIELDS[name] = R.Field(V, F[keep], 0.2, 0.6)
        elif name == "ramp":
            _FIELDS[name] = R.Field(*_ramp_stairs_walls(), 0.07, 0.5)
        elif name == "one_brick":
            _FIELDS[name] = R.Field(*_ramp_stairs_walls(), 0.5, 0.5, lo=(0.1, 0.1, -0.3), hi=(3.3, 2.9, 1.0))
    return _FIELDS[name]


def _restated_pyramid(fd):
    g, index, bricks = fd.g, fd.index, fd.bricks
    bx, by, bz = g.bdims
    n = len(bricks)
    fine2 = np.array([[bricks[s, 2 * (e >> 4):2 * (e >> 4) + 3, 2 * (e >> 2 & 3):2 * (e >> 2 & 3) + 3, 2 * (e & 3):2 * (e & 3) + 3].min() for e in range(64)]
                      for s in range(n)], np.float32).reshape(n, 64)
    fine4 = np.array([[bricks[s, 4 * (e >> 2):4 * (e >> 2) + 5, 4 * (e >> 1 & 1):4 * (e >> 1 & 1) + 5, 4 * (e & 1):4 * (e & 1) + 5].min() for e in range(8)]
                      for s in range(n)], np.float32).reshape(n, 8)
    lvl = np.full((bz, by, bx), np.float32(g.trunc), np.float32)
    alloc = index != 0xFFFFFFFF
    if n:
        lvl[alloc] = bricks.reshape(n, -1).min(1)[index[alloc]]
    levels = [lvl]
    while lvl.shape != (1, 1, 1):
        pad = [(0, s % 2) for s in lvl.shape]
        p = np.pad(lvl, pad, constant_values=np.inf)
        lvl = p.reshape(p.shape[0] // 2, 2, p.shape[1] // 2, 2, p.shape[2] // 2, 2).min((1, 3, 5)).astype(np.float32)
        levels.append(lvl)
    return fine2, fine4, levels


@pytest.mark.parametrize("name", ["building", "terrain", "ramp", "one_brick"])
def test_pyramid_equals_the_restatement(name):
    fd = _field(name)
    assert fd.g.refused is None
    if name in ("terrain", "ramp"):
        assert (fd.index == 0xFFFFFFFF).any() and (fd.index != 0xFFFFFFFF).any()     # unallocated bricks occur
    assert any((d - 1) % 8 for d in fd.g.dims) or name == "one_brick"
    a2, a4, ad = fd.pyramid()
    b2, b4, bd = _restated_pyramid(fd)
    assert a2.tobytes() == b2.tobytes() and a4.tobytes() == b4.tobytes()
    assert len(ad) == len(bd) and all(x.tobytes() == y.tobytes() for x, y in zip(ad, bd))
    if name == "one_brick":
        assert fd.g.bdims == (1, 1, 1)


def _beams(k, seed=3, far=False):
    rng = np.random.default_rng(seed)
    B = np.zeros(k, synth.RANGE_MEAS_DTYPE)
    a = rng.uniform(-np.pi, np.pi, k)
    el = rng.uniform(-0.4, 0.4, k)
    B["dir"] = np.stack([np.cos(a) * np.cos(el), np.sin(a) * np.cos(el), np.sin(el)], 1).astype(np.float32)
    B["range"] = rng.uniform(0.3, 40.0 if far else 4.0, k).astype(np.float32)
    B["orig"] = [0.05, 0.0, 0.2]
    return B


CASES = [  # field, (x0, y0, z0, step, nx, ny, K), surface (None / align), beams, far beams, some node bounded below the best score
    ("building", (0.3, 0.3, 0.5, 0.1, 23, 17, 3), None, 180, False, True),
    ("building", (1.0, 0.5, 0.5, 0.25, 13, 9, 72), None, 1, False, True),
    ("building", (1.0, 0.5, 0.5, 0.25, 13, 9, 2), None, 0, False, False),         # no beams: every bound and score is 0
    ("building", (2.0, 2.0, 0.5, 0.05, 31, 9, 1), None, 180, True, False),         # most end points outside the small field
    ("building_far", (1.0e6 + 1.0, 1.0e6 + 0.5, 0.5, 0.1, 19, 11, 3), None, 180, False, False),   # 0.5 m rounding margin at 10^6 m
    ("terrain", (2.0, 1.0, 0.2, 0.3, 20, 13, 3), 0, 180, False, False),            # the probe's 1.5 m z range: no pruning (DESIGN.md)
    ("terrain", (2.0, 1.0, 0.2, 0.3, 20, 13, 3), 1, 180, False, False),
    ("ramp", (-0.9, -0.45, 0.2, 0.5, 23, 17, 2), 0, 180, False, True),
    ("ramp", (-0.9, -0.45, 0.2, 0.5, 23, 17, 3), 1, 1, False, True),
    ("ramp", (0.1, 0.2, 0.2, 0.15, 40, 50, 1), 1, 180, True, False),
]


@pytest.mark.parametrize("name,grid,align,n_beams,far,prunes", CASES)
def test_bound_dominates_every_score_of_its_block(name, grid, align, n_beams, far, prunes):
    fd = _field(name)
    cfg = rmcl_b200.SearchConfig(*grid, 8, 0.0, 0.0)
    surface = None if align is None else rmcl_b200.SurfaceConfig(0.5, 1.0, 0.3, 0.6, align)
    prm = rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.2
    Tsb, B = synth.scenario_tsb(), _beams(n_beams, far=far)
    S = fd.eval(Tsb, B, prm, cfg, surface, 0)
    if surface is not None:
        assert (S >= 0).any()
    depth = max(1, math.ceil(math.log2(max(cfg.nx, cfg.ny))))
    tight = 0
    for level in range(1, depth + 1):
        bound = fd.eval(Tsb, B, prm, cfg, surface, level)
        K, nby, nbx = bound.shape
        s = 1 << level
        pad = np.full((K, nby * s, nbx * s), -1.0, np.float32)
        pad[:, :cfg.ny, :cfg.nx] = S
        best = pad.reshape(K, nby, s, nbx, s).max((2, 4))
        assert (bound >= best).all(), (level, np.argwhere(bound < best)[:5])
        tight += int((bound < S.max()).sum())
    print(name, grid, align, n_beams, "nodes bounded below the best score:", tight)
    if prunes:
        assert tight > 0                                                # the bound prunes: not a constant such as the top evaluation


@pytest.mark.parametrize("name", ["building", "terrain", "ramp"])
def test_pyramid_query_is_the_min_over_its_cells(name):
    """pyr_query over cell ranges: <= the min of the nodes of the cells (trunc in an unallocated brick) everywhere, equal to it when the
    range is one aligned block of 2, 4, 8 or 16 cells per axis inside the grid (the entry covers exactly those cells' nodes)"""
    fd = _field(name)
    g, index, bricks = fd.g, fd.index, fd.bricks
    d = np.array(g.dims)

    def exact(lo, hi):
        m = np.float32(np.inf)
        for cz in range(lo[2], hi[2] + 1):
            for cy in range(lo[1], hi[1] + 1):
                for cx in range(lo[0], hi[0] + 1):
                    slot = index[cz >> 3, cy >> 3, cx >> 3]
                    v = np.float32(g.trunc) if slot == 0xFFFFFFFF else bricks[slot, (cz & 7):(cz & 7) + 2, (cy & 7):(cy & 7) + 2, (cx & 7):(cx & 7) + 2].min()
                    m = min(m, v)
        return m

    rng = np.random.default_rng(5)
    for _ in range(150):
        lo = rng.integers(0, d - 1)
        hi = np.minimum(lo + rng.integers(0, 12, 3), d - 2)
        assert fd.query(lo, hi) <= exact(lo, hi)
    n_eq = 0
    for s in (1, 2, 3, 4):
        w = 1 << s
        for _ in range(40):
            blk = rng.integers(0, np.maximum(1, (d - 1) // w))
            lo, hi = blk * w, blk * w + w - 1
            if (hi + 1 > d - 1).any():
                continue
            assert fd.query(lo, hi) == exact(lo, hi), (s, lo, hi)
            n_eq += 1
    assert n_eq > 0


CASES_SEARCH = [  # field, grid, surface align, beams, max_records, separations
    ("building", (0.3, 0.3, 0.5, 0.1, 23, 17, 3), None, 180, 8, (0.5, math.radians(60))),
    ("building", (1.0, 0.5, 0.5, 0.25, 13, 9, 72), None, 180, 64, (0.0, 0.0)),      # the yaw wrap: 72 headings, every peak kept
    ("building", (1.0, 0.5, 0.5, 0.25, 13, 9, 2), None, 0, 8, (0.0, 0.0)),          # plateau: every score 0, ties at tau
    ("building", (1.0, 0.5, 0.5, 0.25, 13, 9, 3), None, 1, 64, (0.0, 0.0)),         # one beam: few distinct scores, ties
    ("terrain", (2.0, 1.0, 0.2, 0.3, 20, 13, 3), 1, 180, 16, (1.0, math.radians(30))),
    ("ramp", (-0.9, -0.45, 0.2, 0.5, 23, 17, 2), 0, 180, 4, (1.0, math.radians(30))),
]


@pytest.mark.parametrize("min_ratio", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("name,grid,align,n_beams,max_records,sep", CASES_SEARCH)
def test_threshold_passes_give_the_exhaustive_records(name, grid, align, n_beams, max_records, sep, min_ratio):
    """the passes (SURVEY N5) over the product's bounds and scores, with the product's peak rule over L, stable ranking and separation,
    give the exhaustive restatement's records (pf_search_ref) with score >= tau, in order"""
    import pf_search_ref as X
    fd = _field(name)
    cfg = rmcl_b200.SearchConfig(*grid, max_records, sep[0], sep[1])
    surface = None if align is None else rmcl_b200.SurfaceConfig(0.5, 1.0, 0.3, 0.6, align)
    prm = rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.2
    Tsb, B = synth.scenario_tsb(), _beams(n_beams)
    S = fd.eval(Tsb, B, prm, cfg, surface, 0)
    depth = math.ceil(math.log2(max(cfg.nx, cfg.ny)))
    bounds = {lv: fd.eval(Tsb, B, prm, cfg, surface, lv) for lv in range(1, depth + 1)}
    kc, ks, best, tau, passes = R.search(S, bounds, cfg, n_beams, prm.dist_sigma, min_ratio)
    flat = S.reshape(-1)
    _, kept = X.host_result(flat, cfg)
    assert len(kept) >= 1
    want_best = flat[kept[0]]
    assert best == want_best and tau == np.float32(np.float32(min_ratio) * want_best)
    want = kept[flat[kept] >= tau]
    assert np.array_equal(kc, want.astype(np.uint64)) and ks.tobytes() == flat[want].tobytes()
    for t, Lc in passes:                                                # every candidate >= t is in the pass's L
        assert np.array_equal(Lc, np.flatnonzero(flat >= t).astype(np.uint64))
    if n_beams == 0:
        assert len(passes) == 1 and passes[0][0] == 0.0                 # U = 0: one pass at 0 scores the whole plateau


def _call(f=C.c_void_p(1), c=None, ratio=0.0):
    lib = rmcl_b200.load_library()
    T = np.zeros((), synth.TRANSFORM_DTYPE)
    recs = np.zeros(64, synth.SEARCH_RECORD_DTYPE)
    res = np.zeros((), synth.SEARCH_BNB_RESULT_DTYPE)
    res.reshape(1).view(np.uint8)[:] = 7
    p = rmcl_b200.PFParams.defaults()
    cc = c if c is not None else rmcl_b200.SearchConfig(0.0, 0.0, 0.0, 0.25, 4, 3, 8, 8, 0.0, 0.0)
    rc = lib.b2_pf_global_search_bnb(None, f, C.c_void_p(T.ctypes.data), None, C.c_uint32(0), C.byref(p), C.byref(cc), None, C.c_float(ratio),
                                     C.c_void_p(recs.ctypes.data), C.c_void_p(res.ctypes.data))
    assert (recs.view(np.uint8) == 0).all() and (res.reshape(1).view(np.uint8) == 7).all()   # nothing written
    return rc, lib.b2_last_error().decode()


def test_refusals_launch_nothing():
    n0 = rmcl_b200.kernel_launch_count()
    cfg = lambda **k: rmcl_b200.SearchConfig(*[k.get(n, d) for n, d in (("x0", 0.0), ("y0", 0.0), ("z0", 0.0), ("step", 0.25), ("nx", 4), ("ny", 3),  # noqa: E731
                                                                        ("K", 8), ("mr", 8), ("sx", 0.0), ("sy", 0.0))])
    assert "null argument 'h'" in _call()[1]
    assert "null argument 'f'" in _call(f=None)[1]
    # above 2^30 candidates and the largest axes are accepted
    assert "null argument 'h'" in _call(c=cfg(nx=1 << 24, ny=1 << 24, K=32768, step=2.0 ** -10))[1]
    for kw, ratio, want in [(dict(nx=0), 0.0, "grid"), (dict(ny=(1 << 24) + 1), 0.0, "grid"), (dict(K=32769), 0.0, "grid"), (dict(step=0.0), 0.0, "step"),
                            (dict(x0=3.0e38, step=1.0e38), 0.0, "not finite"), (dict(mr=65), 0.0, "max_records"), (dict(sx=-1.0), 0.0, "separations"),
                            ({}, -0.01, "min_ratio"), ({}, 1.01, "min_ratio"), ({}, float("nan"), "min_ratio"), ({}, float("inf"), "min_ratio")]:
        rc, msg = _call(c=cfg(**kw), ratio=ratio)
        assert rc == -1 and want in msg, (kw, ratio, msg)
    assert rmcl_b200.kernel_launch_count() == n0
