"""CPU tests of the Stein variational step (b2_pf_stein_update, SURVEY appendix L): the product's functions compiled for the host
(tests/pf_stein_ref/stein_emul.cu) against float64 numpy restatements of the definition (tests/pf_stein_ref.py).

Tolerances, from the float error of each sum.
  * df_lookup_grad: the value is df_lookup's bytes.  The gradient is inv_h times lerps of differences of nodes <= trunc: within
    16 ulp(trunc) inv_h of the float64 derivative.  Central differences of the float64 lookup (step 0.1 h, 0.15 h away from cell faces)
    agree within 1e-3 trunc inv_h: the interpolant is linear along each axis within a cell, and the lookup's float cell coordinate
    (ulp <= 2^-16 cells on these grids) moves t by at most 1e-4 of the step.
  * exp_f within 2 ulp of exp in float64 over every normal result; the library forms (float) atan2 / sin / cos within 1 ulp.
  * score: each beam's term carries e's lookup error (8 ulp(trunc)) through a = -(e / sigma^2) ratio (slope <= 1 / sigma^2 + |e| / sigma^4),
    and the slot-order float sum of n_beams terms adds n_beams eps times their absolute sum: within 1e-4 S + n_beams 8 ulp(trunc)
    (1 / sigma^2 + trunc / sigma^4) (1 + r) G, S the float64 absolute sum of the terms, r the largest lever |q - t|, G the largest |grad|.
  * bandwidth: FP64 sums of float charts: within 1e-5 relative (psi's float rounding), the floors exactly.
  * pair sums: each term k (g + Delta / h^2) is a handful of rounded ops (k within 8 ulp plus |s| eps / 2 from its argument), and m terms
    are summed in float: within (1e-6 + m eps) A + 1e-30, A the float64 absolute sum of the terms.  The wrap's float 2 pi is 1.75e-7 above
    2 pi, which moves a wrapped Delta_psi by up to 2e-7: that adds 2e-7 / h_psi^2 per term to psi's sum and 2 pi 2e-7 / h_psi^2 A to all.
  * one step: delta = eps phi / (sqrt(v) + 1e-6) with v = phi^2 moves by at most 1e-3 eps where |phi| > 1e-2 (phi's relative error is
    far below 1e-4 there)."""
import ctypes as C
import math

import numpy as np
import pytest

import dfield_ref as DR
import pf_stein_ref as S

EPS32 = float(np.finfo(np.float32).eps)


def _ulp(x):
    return np.spacing(np.abs(np.float32(x))).astype(np.float64)


_FIELD = {}


def _field(name="indoor"):
    """the field of the indoor mesh (h 0.25, trunc 1.0) or of a 20 m cube (h 0.25, trunc 0.5: its inside has unallocated bricks), and the
    mesh's walls"""
    if name not in _FIELD:
        from rmcl_b200 import synth
        V, F = synth.indoor(2000) if name == "indoor" else synth.cube(5)
        trunc = 1.0 if name == "indoor" else 0.5
        lo, hi = DR.default_box(V, trunc)
        g = DR.Grid(lo, hi, 0.25, trunc)
        index, bricks = DR.ProductField(V, F).build(g)
        _FIELD[name] = dict(V=V, F=F, g=g, index=index, bricks=bricks, scene=S.Scene(V, F))
    return _FIELD[name]


def _beams(k, seed=3):
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    B = np.zeros(k, synth.RANGE_MEAS_DTYPE)
    a = rng.uniform(-np.pi, np.pi, k)
    el = rng.uniform(-0.3, 0.3, k)
    B["dir"] = np.stack([np.cos(a) * np.cos(el), np.sin(a) * np.cos(el), np.sin(el)], 1).astype(np.float32)
    B["range"] = rng.uniform(0.5, 6.0, k).astype(np.float32)
    B["orig"] = [0.05, 0.0, 0.2]
    return B


def _poses(n, seed=5, spread=0.4):
    """n poses around the indoor ground-truth pose, with the edge cases: psi = +pi and -pi, identical particles and non-finite poses"""
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    T0 = synth.indoor_gt_pose()
    P = synth.transforms(n)
    P["t"] = np.asarray(T0["t"], np.float32) + rng.normal(0, spread, (n, 3)).astype(np.float32) * [1, 1, 0.1]
    yaw = math.radians(30.0) + rng.normal(0, 0.3, n)
    yaw[: min(n, 2)] = [np.pi, -np.pi][: min(n, 2)]
    rp = rng.normal(0, 0.02, (n, 2))
    P["R"] = np.stack([synth.quat_from_rpy(rp[i, 0], rp[i, 1], yaw[i]) for i in range(n)]).astype(np.float32)
    if n >= 31:
        P[10:14] = P[9]                                  # identical particles
        P["t"][20, 0] = np.nan
        P["R"][21, 2] = np.inf
    return P


def _tsb():
    from rmcl_b200 import synth
    return synth.make_transform((0.1, 0.0, 0.3), (0.0, 0.0, 0.05))


# ---------------------------------------------------------------- field gradient --------------------------------------------------------
@pytest.mark.parametrize("name", ["indoor", "cube"])
def test_lookup_grad_value_and_gradient(name):
    d = _field(name)
    g, index, bricks = d["g"], d["index"], d["bricks"]
    rng = np.random.default_rng(1)
    span = (np.array(g.dims) - 1) * np.float32(g.h)
    pts = (g.lo + rng.uniform(-0.05, 1.05, (200_000, 3)) * span).astype(np.float32)
    pts[:5] = [[np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 0], [1e30, 0, 0], g.lo]
    val, grad = S.lookup_grad(g, index, bricks, pts)
    assert val.tobytes() == DR.lookup(g, index, bricks, pts).tobytes()
    v64, g64 = S.lookup_grad64(g, index, bricks, pts)
    inv_h = float(np.float32(g.inv_h))
    assert np.abs(grad - g64).max() <= 16 * _ulp(g.trunc) * inv_h
    # zero where nothing is interpolated: non-finite, outside the box, unallocated bricks
    G = (pts - g.lo) * np.float32(g.inv_h)
    inside = np.isfinite(pts).all(1) & (G >= 0).all(1) & (G <= np.array(g.dims) - 1).all(1)
    assert not grad[~inside].any() and np.isinf(val[:3]).all()
    c = np.minimum(np.floor(G[inside]).astype(np.int64), np.array(g.dims) - 2) >> 3
    unalloc = index[c[:, 2], c[:, 1], c[:, 0]] == DR.NOBRICK
    assert not grad[inside][unalloc].any()
    assert unalloc.any() or name == "indoor"
    # central differences of the float64 interpolant away from cell faces
    frac = G[inside] - np.floor(G[inside])
    away = ((frac > 0.15) & (frac < 0.85)).all(1) & ~unalloc
    P = pts[inside][away][:20000].astype(np.float64)
    st = 0.1 * g.h
    for k in range(3):
        e = np.zeros(3)
        e[k] = st
        fd = (S.lookup_grad64(g, index, bricks, (P + e).astype(np.float32))[0] - S.lookup_grad64(g, index, bricks, (P - e).astype(np.float32))[0])
        # the float32 points move by the rounded step: divide by it
        dx = (P + e).astype(np.float32)[:, k].astype(np.float64) - (P - e).astype(np.float32)[:, k].astype(np.float64)
        ok = dx > 0
        gk = S.lookup_grad64(g, index, bricks, P.astype(np.float32))[1][:, k]
        assert np.abs(fd[ok] / dx[ok] - gk[ok]).max() <= 1e-3 * inv_h * g.trunc


# ---------------------------------------------------------------- shared transcendentals ----------------------------------------------
def test_exp_f_within_2_ulp():
    x = np.concatenate([np.linspace(-87.3, 88.72, 4_000_001, dtype=np.float32), np.float32(np.random.default_rng(2).uniform(-5, 5, 1_000_000)),
                        np.array([0.0, -0.0, 1e-30, -1e-30, 0.5, -0.5, 88.7228, -87.33654], np.float32)])
    got = S.exp_f(x).astype(np.float64)
    want = np.exp(x.astype(np.float64))
    normal = want >= np.finfo(np.float32).tiny
    err = np.abs(got[normal] - want[normal]) / np.spacing(want[normal].astype(np.float32)).astype(np.float64)
    print(f"exp_f: max {err.max():.3f} ulp over {normal.sum()} arguments")
    assert err.max() <= 2.0
    sp = S.exp_f(np.array([np.nan, np.inf, -np.inf, 88.7228394, 100.0, -103.972084, -104.0, -200.0], np.float32))
    assert np.isnan(sp[0]) and sp[1] == np.inf and sp[2] == 0.0 and sp[3] == np.inf and sp[4] == np.inf and sp[6] == 0.0 and sp[7] == 0.0
    # subnormal results: within one subnormal step
    xs = np.linspace(-103.9, -87.4, 100_001, dtype=np.float32)
    ws = np.exp(xs.astype(np.float64))
    assert np.abs(S.exp_f(xs).astype(np.float64) - ws).max() <= 2 * 2.0 ** -149


@pytest.mark.parametrize("which", [0, 1, 2])
def test_library_forms_within_1_ulp(which):
    rng = np.random.default_rng(which)
    a = rng.uniform(-4, 4, 1_000_000).astype(np.float32)
    b = rng.uniform(-4, 4, 1_000_000).astype(np.float32)
    got = S.lib_f(which, a, b).astype(np.float64)
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    want = np.arctan2(a64, b64) if which == 0 else np.sin(a64) if which == 1 else np.cos(a64)
    err = np.abs(got - want) / np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    assert err.max() <= 1.0


# ---------------------------------------------------------------- draws of J ----------------------------------------------------------
def test_reference_draws_match_philox():
    assert [hex(x) for x in (int(w[0]) for w in S.philox([0], [0], [0], [0], 0, 0))] == ["0x6627e8d5", "0xe169c58d", "0xbc57ac4c", "0x9b00dbd8"]
    assert [hex(int(w[0])) for w in S.philox([0x243f6a88], [0x85a308d3], [0x13198a2e], [0x03707344], 0xa4093822, 0x299f31d0)] == \
        ["0xd16cfe09", "0x94fdcceb", "0x5001e420", "0x24126ea1"]
    for n, n_ref, seed, step, it in [(1000, 7, 1, 0, 0), (100_000, 4096, 0x1234567890ABCDEF, 9, 3), (33, 32, 5, 1, 29)]:
        got = S.ref_index(S.n_refs(n, n_ref), n, n_ref, seed, step, it)
        assert np.array_equal(got, S.ref_index64(S.n_refs(n, n_ref), n, n_ref, seed, step, it))
    assert np.array_equal(S.ref_index(10, 10, 0, 1, 0, 0), np.arange(10)) and np.array_equal(S.ref_index(10, 10, 15, 1, 0, 0), np.arange(10))
    a, b = S.ref_index(4096, 10**6, 4096, 7, 0, 0), S.ref_index(4096, 10**6, 4096, 7, 0, 1)
    assert not np.array_equal(a, b) and a.max() < 10**6


# ---------------------------------------------------------------- score, bandwidth, one step --------------------------------------------
@pytest.mark.parametrize("n_beams", [0, 1, 180])
@pytest.mark.parametrize("n_ref_kind", ["all", "one", "seven", "over"])
@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 1000])
def test_score_bandwidth_and_one_step_against_float64(n, n_ref_kind, n_beams):
    d = _field()
    g, index, bricks = d["g"], d["index"], d["bricks"]
    n_ref = {"all": 0, "one": 1, "seven": 7, "over": n + 5}[n_ref_kind]
    P, B, Tsb = _poses(n), _beams(n_beams), _tsb()
    sigma, w, seed = 0.2, 0.05, 99
    m = S.n_refs(n, n_ref)
    snap = S.score(g, index, bricks, P, n_ref, seed, 3, 0, Tsb, B, sigma, w)
    idx = S.ref_index64(m, n, n_ref, seed, 3, 0)
    sc64 = S.score64(g, index, bricks, P, idx, Tsb, B, sigma, w)
    c64 = S.chart64(P[idx])
    bad = np.isnan(sc64[:, 0])
    assert np.array_equal(np.isnan(snap[:, 0]), bad) and np.isnan(snap[bad]).all()
    assert np.abs(snap[~bad, :2] - c64[~bad, :2]).max(initial=0) == 0
    assert np.abs(S.wrap64(snap[~bad, 2] - c64[~bad, 2])).max(initial=0) <= 2 * _ulp(np.pi)
    if n_beams and (~bad).any():
        pts = DR.beam_points64(P[idx][~bad], Tsb, B)
        e, gr = S.lookup_grad64(g, index, bricks, pts.reshape(-1, 3))
        lever = 1 + np.abs(pts - P[idx][~bad]["t"][:, None, :].astype(np.float64)).max()
        s2 = sigma * sigma
        bound = n_beams * 8 * _ulp(g.trunc) * (1 / s2 + g.trunc / s2 ** 2) * lever * max(1.0, np.abs(gr).max())
        absum = np.abs(sc64[~bad]).sum(1, keepdims=True) + 1e-30
        # S, the absolute sum of the terms, is at least |sum|; bound it by the largest term magnitude times n_beams
        tmax = n_beams * (g.trunc / s2) * np.abs(gr).max() * lever
        assert (np.abs(snap[~bad, 3:] - sc64[~bad]) <= 1e-4 * np.minimum(absum, tmax) + 1e-4 * tmax * EPS32 * n_beams + bound).all()
    elif (~bad).any():
        assert not snap[~bad, 3:].any()
    # bandwidth
    h, tot = S.bandwidth(P, m, 0.05, 0.02)
    h64 = S.bandwidth64(P, m, 0.05, 0.02)
    fin = np.isfinite(S.chart64(P)).all(1)
    assert tot[0] == fin.sum()
    assert np.allclose(h, h64, rtol=1e-5, atol=0)
    # pair sums over the product's snapshot
    ci = S.chart(P)
    acc = S.pairs(ci, snap, h)
    a64 = S.pairs64(ci.astype(np.float64), snap.astype(np.float64), h.astype(np.float64))
    live = np.isfinite(ci).all(1)
    sn = snap[~np.isnan(snap[:, 0])].astype(np.float64)
    if len(sn):
        D = ci[live][:, None, :].astype(np.float64) - sn[None, :, :3]
        D[..., 2] = S.wrap64(D[..., 2])
        U = D / h.astype(np.float64) ** 2
        k = np.exp(-0.5 * (D * U).sum(2))
        A = np.einsum("ij,ijd->id", k, np.abs(sn[None, :, 3:] + U))
        wr = 2e-7 / float(h[2]) ** 2                      # the float 2 pi of the wrap is 1.75e-7 above 2 pi
        tol = (1e-6 + m * EPS32 + 2 * np.pi * wr) * A + np.array([0.0, 0.0, m * wr]) + 1e-30
        assert (np.abs(acc[live] - a64[live]) <= tol).all()
    else:
        assert not acc[live].any()
    # one step (iteration 0): the moved poses against delta from the float64 pair sums
    Pm = P.copy()
    v = np.zeros((n, 3), np.float32)
    rec = S.SteinResult()
    eps = np.array([0.02, 0.02, 0.01])
    d["scene"].move(Pm, snap, 0, 0.02, 0.01, v, h, rec)
    phi = a64 / m
    delta64 = eps * phi / (np.abs(phi) + 1e-6)
    cm = S.chart(Pm)
    moved = live & (np.abs(cm - ci) > 0).any(1)
    sure = moved[:, None] & (np.abs(phi) > 1e-2)
    got = cm.astype(np.float64) - ci
    got[:, 2] = S.wrap64(got[:, 2])
    tol = 1e-3 * eps + 2 * np.spacing(np.abs(ci).astype(np.float32)).astype(np.float64) + np.array([0, 0, 4 * _ulp(np.pi)])
    assert (np.abs(got - delta64)[sure] <= np.broadcast_to(tol, got.shape)[sure]).all()
    # non-finite particles keep their pose; z, roll and pitch stay
    assert Pm[~live].tobytes() == P[~live].tobytes()
    assert np.array_equal(Pm["t"][:, 2], P["t"][:, 2])
    # a particle that did not move was blocked by a wall or had no step to take
    assert rec.n_blocked <= (live & ~moved).sum()


def test_no_spread_gives_the_floors_and_identical_particles_do_not_repel():
    d = _field()
    P = _poses(1)
    P = np.repeat(P, 50)
    h, _ = S.bandwidth(P, 50, 0.05, 0.02)
    assert h.tolist() == [np.float32(0.05), np.float32(0.05), np.float32(0.02)]
    snap = S.score(d["g"], d["index"], d["bricks"], P, 0, 1, 0, 0, _tsb(), _beams(0), 0.2, 0.05)
    assert not snap[:, 3:].any()
    acc = S.pairs(S.chart(P), snap, h)
    assert not acc.any()                                  # Delta = 0: k = 1, no score, no repulsion


# ---------------------------------------------------------------- SVGD dynamics --------------------------------------------------------
def _svgd(repulsion, iters=200, n=400, seed=11):
    mu = np.array([1.0, -2.0, 3.0])                      # psi near pi: the set straddles the wrap
    sd = np.array([0.3, 0.2, 0.25])
    rng = np.random.default_rng(seed)
    c = (mu + rng.normal(0, 1, (n, 3)) * sd * 0.3 + sd * 0.5).astype(np.float32)
    c[:, 2] = S.wrap64(c[:, 2]).astype(np.float32)
    v = np.zeros((n, 3), np.float32)
    eps = np.array([0.01, 0.01, 0.01], np.float32)
    for it in range(iters):
        dlt = c.astype(np.float64) - mu
        dlt[:, 2] = S.wrap64(dlt[:, 2])
        g = (-dlt / sd ** 2).astype(np.float32)
        snap = np.concatenate([c, g], 1)
        R = np.hypot(np.cos(c[:, 2].astype(np.float64)).mean(), np.sin(c[:, 2].astype(np.float64)).mean())
        s = np.array([c[:, 0].std(), c[:, 1].std(), np.sqrt(2 * (1 - R))])
        h = np.maximum(s * n ** (-1 / 7), [1e-3, 1e-3, 1e-3]).astype(np.float32)
        if repulsion:
            acc = S.pairs(c, snap, h)
        else:
            D = c[:, None, :].astype(np.float64) - c[None, :, :]
            D[..., 2] = S.wrap64(D[..., 2])
            k = np.exp(-0.5 * (D ** 2 / h.astype(np.float64) ** 2).sum(2))
            acc = (k @ g.astype(np.float64)).astype(np.float32)
        phi = acc / np.float32(n)
        v = phi * phi if it == 0 else np.float32(0.9) * v + np.float32(0.1) * phi * phi
        c = c + eps * phi / (np.sqrt(v) + np.float32(1e-6))
        c[:, 2] = S.wrap64(c[:, 2]).astype(np.float32)
    d = c.astype(np.float64) - mu
    d[:, 2] = S.wrap64(d[:, 2])
    return d.mean(0) / sd, d.std(0) / sd


def test_svgd_pair_pass_samples_a_gaussian_and_collapses_without_repulsion():
    """the host-compiled pair pass fed the analytic score -(c - mu) / sd^2 of a Gaussian in the chart: after 200 RMSProp steps of 400
    particles the set's mean is within 0.05 sd and its spread within 15 % of sd per dimension; without the repulsion term it collapses"""
    mean, std = _svgd(True)
    print(f"SVGD: mean / sd {np.round(mean, 4)}, std / sd {np.round(std, 3)}")
    assert np.abs(mean).max() <= 0.05 and np.abs(std - 1).max() <= 0.15
    _, std0 = _svgd(False)
    print(f"without repulsion: std / sd {np.round(std0, 3)}")
    assert std0.max() < 0.3


# ---------------------------------------------------------------- ABI -------------------------------------------------------------------
def test_abi_records_and_null_handle():
    import rmcl_b200
    assert C.sizeof(rmcl_b200.SteinConfig) == 32 and C.sizeof(rmcl_b200.api._SteinResult) == 32
    c = rmcl_b200.SteinConfig.defaults()
    assert (c.iterations, c.n_ref) == (10, 4096) and c.step_t > 0 and c.step_r > 0 and 0 <= c.w_rand < 1
    assert "b2_pf_stein_update" in rmcl_b200.api.EXPORTS
    import os
    if not os.path.exists(rmcl_b200.lib_path()):
        pytest.skip("library not built")
    lib = rmcl_b200.load_library()
    assert lib.b2_pf_stein_update(None, None, None, 0, None, None, 0, None, None, C.c_uint64(0), 0, None) == -1
