"""CPU tests of KLD-sampling (b2_pf_resample_kld; SURVEY appendix G): the product's per-element functions compiled for the CPU against the C
restatement of tests/pf_kld_ref (bounds, keys, weights, draws), the bound against scipy's chi-square quantile, the yaw sector against a
float64 atan2, the draws against their weights, the restatement's stop rule against a literal Python transcription of the sequential loop,
and the properties the feature is for."""
import math

import numpy as np
import pytest
from scipy import stats as sps

import pf_kld_ref as ref
from rmcl_b200.api import KLDConfig
from rmcl_b200.synth import TRANSFORM_DTYPE
from test_pf_residual import CFG, FAMILIES, particles

f32 = np.float32
BOUND_CASES = [(0.01, 0.99), (0.05, 2.326), (0.01, 3.0), (0.2, -1.0), (1e-4, 1.5)]
SECTORS = (1, 2, 3, 4, 36, 360, 32768)


def kcfg(**kw):
    c = KLDConfig.defaults()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


# ---- the bound ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("eps,z", BOUND_CASES)
def test_bound_product_matches_restatement(eps, z):
    k = np.arange(0, 1_000_001, dtype=np.uint64)
    a, b = ref.bounds(k, eps, z, 100), ref.product_bounds(k, eps, z, 100)
    assert np.array_equal(a, b)
    assert a[0] == a[1] == 100


@pytest.mark.parametrize("eps,z", [c for c in BOUND_CASES if c[1] > 0])
def test_bound_is_the_wilson_hilferty_chi_square_quantile(eps, z):
    """Fox's bound is chi2.ppf(1 - delta, k - 1) / (2 eps) with z = norm.ppf(1 - delta), by the Wilson-Hilferty approximation, rounded up.
    Stated error beyond the rounding: < 3 % for k >= 2, < 1 % for k >= 10, < 0.1 % for k >= 100 (at z <= 3)."""
    k = np.arange(2, 200_001)
    b = ref.bounds(k.astype(np.uint64), eps, z, 1).astype(np.float64)
    exact = sps.chi2.ppf(sps.norm.cdf(z), k - 1) / (2 * eps)
    err = np.maximum(0.0, np.maximum(exact - b, b - 1.0 - exact)) / exact
    assert err.max() < 0.03 and err[8:].max() < 0.01 and err[98:].max() < 1e-3, (err.max(), err[8:].max(), err[98:].max())


def test_stop_rule_product_matches_python():
    rng = np.random.default_rng(3)
    j = rng.integers(0, 2_000_000, 200_000).astype(np.uint64)
    k = np.minimum(j + 1, rng.integers(0, 50_000, 200_000).astype(np.uint64))
    for eps, z, n_min, n_max in ((0.01, 0.99, 100, 1_000_000), (0.05, 2.0, 1, 65_537), (0.2, 3.0, 5000, 5000)):
        got = ref.product_stop(j, k, eps, z, n_min, n_max)
        want = [int(jj) + 1 >= max(n_min, _bound(int(kk), eps, z, n_min)) or int(jj) + 1 == n_max for jj, kk in zip(j, k)]
        assert np.array_equal(got, np.array(want))


# ---- keys ---------------------------------------------------------------------------------------------------------------------------
def _poses(n, seed, span=30.0):
    rng = np.random.default_rng(seed)
    P = np.zeros(n, TRANSFORM_DTYPE)
    P["t"] = rng.uniform(-span, span, (n, 3)).astype(f32)
    q = rng.normal(size=(n, 4))
    P["R"] = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(f32)
    return P


@pytest.mark.parametrize("K", SECTORS)
@pytest.mark.parametrize("res_xy,res_z", [(0.5, 0.0), (0.05, 0.25), (7.0, 1e-3)])
def test_keys_product_matches_restatement_random(K, res_xy, res_z):
    P = _poses(20_000, K)
    a, b = ref.keys(P, res_xy, res_z, K), ref.product_keys(P, res_xy, res_z, K)
    assert np.array_equal(a, b)
    assert np.all((a >> np.uint64(15)) & np.uint64(1) == 0)        # bit 15 is never set in a real key
    assert np.all((a & np.uint64(0x7FFF)) < K)


def _yaw_pose(x, y, z, w, t=(0.0, 0.0, 0.0)):
    P = np.zeros(1, TRANSFORM_DTYPE)
    P["R"] = np.array([x, y, z, w], f32)
    P["t"] = np.array(t, f32)
    return P


def _heading(R):
    x, y, z, w = (f32(v) for v in R)
    return f32(1) - f32(2) * (y * y + z * z), f32(2) * (x * y + w * z)


def _exact_boundary_quats(K, limit=300, stride=1):
    """quaternions (0, 0, z, w) whose heading equals the tabulated boundary vector (c_k, s_k) exactly, for the boundaries k where such
    floats exist (hx = 1 - 2 z^2 and hy = 2 w z rounded as the product rounds them)"""
    cs = ref.table(K)
    out = []
    for k in range(1, K, stride):
        c, s = cs[k]
        if c == 1 and s == 0:
            out.append((k, (0.0, 0.0, 0.0, 1.0)))
            continue
        z0 = f32(math.sqrt(max(0.0, (1.0 - float(c)) / 2.0)))
        zs = (z0.view(np.int32) + np.arange(-limit, limit + 1, dtype=np.int32)).view(f32)
        zs = zs[((f32(1) - f32(2) * (zs * zs)) == c) & (zs > 0)]
        for zz in zs[:4]:
            w0 = f32(float(s) / (2.0 * float(zz)))
            ws = (w0.view(np.int32) + np.arange(-limit, limit + 1, dtype=np.int32)).view(f32)
            ws = ws[f32(2) * (ws * zz) == s]
            if len(ws):
                out.append((k, (0.0, 0.0, float(zz), float(ws[0]))))
                break
    return out


def test_keys_edges():
    res = 0.5
    rows = []
    for m in range(-6, 7):                                          # exact multiples of the resolution, and -0.0
        rows.append(((0, 0, 0, 1), (m * res, -m * res, m * 0.25)))
    rows.append(((0, 0, 0, 1), (-0.0, -0.0, -0.0)))
    big = 2.0 ** 19 * res
    for v in (big, -big, np.nextafter(f32(big), f32(0)), np.nextafter(f32(-big), f32(0)), np.nextafter(f32(-big), f32(-1e9)), 1e30, -1e30, 3.4e38, -3.4e38):
        rows.append(((0, 0, 0, 1), (float(v), float(v), float(v))))
    for v in (32.0, -32.0, 31.999998, -32.000004, 1e10, -1e10):      # res_z 0.25: iz limits at +-2^7 cells
        rows.append(((0, 0, 0, 1), (0.0, 0.0, v)))
    # phi = -pi (h = (-1, 0) and (-1, -0)), a hair above -pi on the upper side, h = (0, 0), the +x axis
    rows += [((0, 0, 1, 0), (0, 0, 0)), ((0, 0, 1, -0.0), (0, 0, 0)), ((0, 0, 1, 1e-30), (0, 0, 0)), ((0, 0, 1, -1e-30), (0, 0, 0)),
             ((-0.5, 0.5, 0.5, 0.5), (0, 0, 0)), ((0, 0, 0, 1), (0, 0, 0)), ((0, 0, 0, -1), (0, 0, 0))]
    bad = [float("nan"), float("inf"), -float("inf")]
    for i in range(7):
        for b in bad:
            R, t = [0.0, 0.0, 0.0, 1.0], [1.0, 2.0, 3.0]
            (R if i < 4 else t)[i % 4 if i < 4 else i - 4] = b
            rows.append((tuple(R), tuple(t)))
    P = np.concatenate([_yaw_pose(*R, t=t) for R, t in rows])
    for K in SECTORS:
        for res_z in (0.0, 0.25):
            a, b = ref.keys(P, res, res_z, K), ref.product_keys(P, res, res_z, K)
            assert np.array_equal(a, b), K
            nonfinite = ~np.all(np.isfinite(P["t"]), 1) | ~np.all(np.isfinite(P["R"]), 1)
            assert np.all(a[nonfinite] == np.uint64(0xFFFFFFFFFFFFFFFF)) and not np.any(a[~nonfinite] == np.uint64(0xFFFFFFFFFFFFFFFF))
            ix = (a[~nonfinite] >> np.uint64(44)).astype(np.int64) - 2 ** 19
            assert ix.min() >= -2 ** 19 and ix.max() < 2 ** 19
            sec = {r: int(k & np.uint64(0x7FFF)) for r, k in zip(range(len(rows)), a)}
            first_phi = len(rows) - 21 - 7
            assert sec[first_phi] == 0 and sec[first_phi + 1] == 0            # phi = -pi: sector 0
            assert sec[first_phi + 2] == K - 1 and sec[first_phi + 3] == 0    # just above -pi on the upper side: the last sector
            assert sec[first_phi + 4] == 0                                     # h = (0, 0)
            assert sec[first_phi + 5] == K // 2 and sec[first_phi + 6] == K // 2   # phi = 0: boundaries with 2k <= K lie at or before it
    # iz: res_z = 0 leaves z out; res_z = 0.25 clamps to [-128, 127]
    ks = ref.keys(P, res, 0.25, 36)
    iz = ((ks >> np.uint64(16)) & np.uint64(0xFF)).astype(np.int64) - 128
    assert iz.min() == -128 and iz.max() == 127
    assert np.all((ref.keys(P, res, 0.0, 36)[:13] >> np.uint64(16)) & np.uint64(0xFF) == 128)


@pytest.mark.parametrize("K", [4, 36, 360, 32768])
def test_headings_on_the_tabulated_boundaries(K):
    """a heading exactly on boundary k lies at it: sector k (the cross product is exactly 0)"""
    found = _exact_boundary_quats(K, stride=1 if K <= 360 else 97)
    assert len(found) >= (1 if K == 4 else 10), len(found)
    cs = ref.table(K)
    for k, q in found:
        assert _heading(q) == tuple(cs[k])
    P = np.concatenate([_yaw_pose(*q) for _, q in found])
    a, b = ref.keys(P, 0.5, 0.0, K), ref.product_keys(P, 0.5, 0.0, K)
    assert np.array_equal(a, b)
    assert [int(v & np.uint64(0x7FFF)) for v in a] == [k for k, _ in found]


@pytest.mark.parametrize("K", SECTORS)
def test_sector_matches_float64_atan2(K):
    """the sector is floor((atan2(h.y, h.x) + pi) / (2 pi / K)) of the float heading, except within 1e-6 rad of a boundary"""
    P = _poses(50_000, 100 + K)
    sec = (ref.product_keys(P, 0.5, 0.0, K) & np.uint64(0x7FFF)).astype(np.int64)
    R = P["R"]
    x, y, z, w = (R[:, i] for i in range(4))
    hx = f32(1) - f32(2) * (y * y + z * z)
    hy = f32(2) * (x * y + w * z)
    phi = np.arctan2(hy.astype(np.float64), hx.astype(np.float64))
    u = (phi + math.pi) / (2 * math.pi / K)
    want = np.floor(u).astype(np.int64) % K
    d = np.abs(u - np.round(u)) * (2 * math.pi / K)
    ok = d > 1e-6
    assert ok.mean() > 0.98                                         # 2e-6 of every 2 pi / K is left out
    assert np.array_equal(sec[ok], want[ok])


def test_sector_count_of_the_suggested_resolution():
    assert ref.sectors(f32(math.radians(10.0))) == 36 and ref.sectors(f32(math.radians(1.0))) == 360
    assert ref.sectors(f32(2 * math.pi)) == 1 and ref.sectors(f32(2 * math.pi / 32768)) == 32768
    assert ref.sectors(f32(2 * math.pi / 40000)) == 0 and ref.sectors(f32(-0.1)) == 0


# ---- weights and draws --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", FAMILIES)
def test_weights_and_parents_product_match_restatement(family):
    P, A = particles(5000, family, seed=11)
    L_max = float(A["likelihood"]["mean"].max())
    W = ref.prefix(A, L_max)
    assert np.array_equal(W, ref.product_prefix(A["likelihood"]["mean"], L_max))
    w = np.diff(np.concatenate([[0], W.astype(object)])).astype(np.float64)
    assert w.max() == 2.0 ** 32
    assert np.array_equal(ref.parents(9, 4, 0, 100_000, W), ref.product_parents(9, 4, 0, 100_000, W))
    assert np.array_equal(ref.parents(9, 4, 2 ** 33 + 5, 1000, W), ref.product_parents(9, 4, 2 ** 33 + 5, 1000, W))   # counters above 2^32


@pytest.mark.parametrize("family", FAMILIES)
def test_draws_follow_the_weights(family):
    n, draws = 40, 400_000
    P, A = particles(n, family, seed=21)
    L = A["likelihood"]["mean"].astype(np.float64)
    A["likelihood"]["mean"][3] = 0.0
    L[3] = 0.0
    W = ref.prefix(A, L.max())
    par = ref.parents(5, 0, 0, draws, W)
    cnt = np.bincount(par, minlength=n)
    w = np.diff(np.concatenate([[0], W.astype(object)])).astype(np.float64)
    assert np.all(cnt[w == 0] == 0)                                 # a zero weight is never drawn
    live = w > 0
    exp = draws * w[live] / w.sum()
    big = exp >= 5
    chi2 = (((cnt[live][big] - exp[big]) ** 2) / exp[big]).sum()
    assert sps.chi2.sf(chi2, big.sum() - 1) > 1e-4, chi2


# ---- the stop rule against a literal transcription --------------------------------------------------------------------------------
def _bound(k, eps, z, n_min):
    if k <= 1:
        return n_min
    km1 = float(k - 1)
    a = 2.0 / (9.0 * km1)
    x = (1.0 - a) + math.sqrt(a) * z
    v = (km1 / (2.0 * eps)) * ((x * x) * x)
    return 0 if not v > 0.0 else math.ceil(v)


def _python_kld(keys, n_max, eps, z, n_min):
    """Fox's loop (AMCL's pf_update_resample, one sample at a time): insert the draw's bin, stop once the count reaches the bound"""
    seen = set()
    for j in range(n_max):
        seen.add(int(keys[j]))
        if j + 1 >= max(n_min, _bound(len(seen), eps, z, n_min)) or j + 1 == n_max:
            return j + 1, len(seen)


def _set(n, spread, seed):
    """n particles, likelihoods lognormal, poses within `spread` m and all headings"""
    P, A = particles(n, "lognormal", seed=seed)
    P["t"] *= f32(spread / 20.0)
    return P, A


@pytest.mark.parametrize("n,spread,n_max,eps,z,n_min", [(1, 1.0, 5000, 0.01, 0.99, 100), (2, 20.0, 5000, 0.01, 0.99, 100),
                                                        (1000, 0.2, 70_000, 0.01, 0.99, 100), (1000, 3.0, 70_000, 0.05, 2.326, 50),
                                                        (20_000, 20.0, 200_000, 0.01, 0.99, 100), (20_000, 5.0, 100_000, 0.2, 3.0, 1),
                                                        (5000, 1.0, 5000, 0.01, 0.99, 5000)])
def test_stop_rule_matches_python_transcription(n, spread, n_max, eps, z, n_min):
    P, A = _set(n, spread, n + 7)
    k = kcfg(epsilon=eps, z=z, n_min=n_min)
    r = ref.resample(P, A, n_max, k, CFG, seed=3, step=1)
    _, _, L_max = __import__("pf_residual_ref").stats(A)
    par = ref.parents(3, 1, 0, n_max, ref.prefix(A, L_max))
    keys = ref.keys(P[par], k.res_xy, k.res_z, ref.sectors(k.res_yaw))
    assert (r["n_particles"], r["bins"]) == _python_kld(keys, n_max, eps, z, n_min)
    assert np.array_equal(r["parents"], par[: r["n_particles"]]) and np.array_equal(r["keys"], keys[: r["n_particles"]])
    m = r["n_particles"]
    assert np.array_equal(r["P"]["stamp"][:m], par[:m])             # slot j is a copy of draw j's parent
    assert np.all(r["P"].view(np.uint8).reshape(n_max, -1)[m:] == 0)


# ---- properties -------------------------------------------------------------------------------------------------------------------
def test_one_bin_gives_n_min():
    P, A = particles(3000, "uniform", seed=4)
    P["t"] = np.array([1.1, 2.2, 0.3], f32)
    P["R"] = np.array([0, 0, 0, 1], f32)
    for n_min in (1, 100, 2999):
        r = ref.resample(P, A, 100_000, kcfg(n_min=n_min), CFG)
        assert (r["n_particles"], r["bins"]) == (n_min, 1)


def test_wide_spread_fills_n_max():
    """poses over far more than n_max * 2 eps bins: the bound outruns the draws to the end"""
    P, A = particles(50_000, "uniform", seed=5)
    P["t"] *= f32(10.0)
    n_max = 60_000
    r = ref.resample(P, A, n_max, kcfg(), CFG)
    assert r["n_particles"] == n_max and r["bins"] > 2 * 0.01 * n_max * 10


def test_smaller_epsilon_never_fewer_particles():
    P, A = _set(5000, 4.0, 9)
    last = 0
    for eps in (0.5, 0.2, 0.1, 0.05, 0.02, 0.01, 0.005):
        r = ref.resample(P, A, 300_000, kcfg(epsilon=eps), CFG, seed=8)
        assert r["n_particles"] >= last
        last = r["n_particles"]
    assert last > 1000


@pytest.mark.parametrize("bad", [0.0, -1e-3, float("nan"), float("inf")])
def test_invalid_sets_give_nothing(bad):
    P, A = particles(500, "uniform", seed=2)
    if bad == 0.0:
        A["likelihood"]["mean"] = 0.0
    else:
        A["likelihood"]["mean"][100] = bad
    r = ref.resample(P, A, 1000, kcfg(), CFG)
    assert (r["n_particles"], r["bins"]) == (0, 0)
    assert np.all(r["P"].view(np.uint8) == 0) and np.all(r["A"].view(np.uint8) == 0)
