"""CPU tests of the filter's pose hypotheses (b2_pf_cluster_stats; SURVEY appendix H): the sequential C restatement (tests/pf_cluster_ref) against
a literal flood fill over a dict of bins, the product's bin-neighbour function compiled for the host against the restatement, crafted
topologies, and the properties a caller relies on.  The device is compared with the same restatement in test_gpu_pf_cluster.py."""
import itertools
import math

import numpy as np
import pytest

import pf_cluster_ref as ref
import pf_kld_ref
from rmcl_b200.api import ClusterConfig
from rmcl_b200.synth import PARTICLE_ATTR_DTYPE, TRANSFORM_DTYPE
from test_pf_residual import particles

NONE, NONE_KEY = ref.NONE, ref.NONE_KEY
RES_XY, RES_Z = 0.5, 0.25


def cfg(**kw):
    c = ClusterConfig.defaults()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def unpack(key):
    key = int(key)
    return (key >> 44) - 524288, ((key >> 24) & 0xFFFFF) - 524288, ((key >> 16) & 0xFF) - 128, key & 0xFFFF


def python_neighbour(key, dx, dy, dz, ds, K, has_z):
    ix, iy, iz, s = unpack(key)
    ix, iy, iz = ix + dx, iy + dy, iz + dz
    if not (-524288 <= ix < 524288 and -524288 <= iy < 524288):
        return NONE_KEY
    if (not has_z and dz != 0) or not (-128 <= iz < 128):
        return NONE_KEY
    return ref.make_key(ix, iy, iz, (s + ds) % K)


def flood_fill(keys, w, K, has_z):
    """the rule of include/rmcl_b200.h, literally: a dict of bins, a flood fill over the 80 neighbours, clusters sorted by (-weight, key)"""
    bins = {}
    for i, (k, wi) in enumerate(zip(keys, w)):
        if int(wi) > 0 and k != NONE_KEY:
            bins.setdefault(int(k), []).append(i)
    comp, comps = {}, []
    for k0 in sorted(bins):
        if k0 in comp:
            continue
        comp[k0] = len(comps)
        todo, mine = [k0], []
        while todo:
            k = todo.pop()
            mine.append(k)
            for d in itertools.product((-1, 0, 1), repeat=4):
                nk = int(python_neighbour(k, *d, K, has_z))
                if nk in bins and nk not in comp:
                    comp[nk] = len(comps)
                    todo.append(nk)
        comps.append(mine)
    stats = [(sum(int(w[i]) for k in c for i in bins[k]), min(c), len(c), sum(len(bins[k]) for k in c)) for c in comps]
    order = sorted(range(len(comps)), key=lambda j: (-stats[j][0], stats[j][1]))
    rank = {j: r for r, j in enumerate(order)}
    labels = np.full(len(keys), NONE, np.uint32)
    for k, members in bins.items():
        labels[members] = rank[comp[k]]
    return labels, [stats[j] for j in order]


def check_against_flood_fill(keys, w, K, has_z):
    got = ref.cluster(keys, w, K, has_z)
    labels, stats = flood_fill(keys, w, K, has_z)
    assert np.array_equal(got["labels"], labels)
    assert got["n_clusters"] == len(stats)
    assert [tuple(int(v) for v in t) for t in zip(got["weight_int"], got["key"], got["cbins"], got["members"])] == stats
    assert got["bins"] == sum(s[2] for s in stats) and got["n_clustered"] == sum(s[3] for s in stats) and got["weight_total"] == sum(s[0] for s in stats)
    return got


def poses_in_bins(cells, K, res_xy=RES_XY, res_z=RES_Z):
    """one pose in the middle of each bin (ix, iy, iz, sector)"""
    cells = np.asarray(cells, np.int64).reshape(-1, 4)
    P = np.zeros(len(cells), TRANSFORM_DTYPE)
    P["t"][:, 0] = (cells[:, 0] + 0.5) * res_xy
    P["t"][:, 1] = (cells[:, 1] + 0.5) * res_xy
    P["t"][:, 2] = (cells[:, 2] + 0.5) * res_z
    yaw = -math.pi + 2.0 * math.pi * (cells[:, 3] + 0.5) / K
    P["R"][:, 2] = np.sin(yaw / 2)
    P["R"][:, 3] = np.cos(yaw / 2)
    P["stamp"] = np.arange(len(cells), dtype=np.uint32)
    return P


def attrs_of(L):
    A = np.zeros(len(L), PARTICLE_ATTR_DTYPE)
    A["likelihood"]["mean"] = np.asarray(L, np.float32)
    A["likelihood"]["n_meas"] = 10
    return A


def keys_of(cells):
    return np.array([ref.make_key(*c) for c in np.asarray(cells).reshape(-1, 4)], np.uint64)


def snake(rows=200, length=500):
    """a one-bin-wide path of rows * (length + 1) - 1 bins: rows two cells apart, joined at alternating ends"""
    cells = []
    for r in range(rows):
        xs = range(length) if r % 2 == 0 else range(length - 1, -1, -1)
        cells += [(x, 2 * r, 0, 0) for x in xs]
        if r + 1 < rows:
            cells.append((cells[-1][0], 2 * r + 1, 0, 0))
    return cells


def blob(x0, y0, side=3, z=0, s=5):
    return [(x0 + i, y0 + j, z, s) for i in range(side) for j in range(side)]


def test_poses_in_bins_land_in_their_bins():
    for K in (3, 36):
        cells = blob(-4, 7, s=K // 2) + [(0, 0, -128, 0), (100, -100, 127, K - 1)]
        assert np.array_equal(pf_kld_ref.keys(poses_in_bins(cells, K), RES_XY, RES_Z, K), keys_of(cells))


EDGE_CELLS = [(3, -7, 2, 0), (-524288, 0, 0, 0), (524287, 0, 0, 0), (0, -524288, 0, 0), (0, 524287, 0, 0), (0, 0, -128, 0), (0, 0, 127, 0),
              (-524288, 524287, 127, 0), (524287, -524288, -128, 0)]


@pytest.mark.parametrize("has_z", [0, 1])
@pytest.mark.parametrize("K", [1, 2, 3, 36, 32768])
def test_neighbour_product_matches_restatement(K, has_z):
    """every one of the 81 offsets at an interior bin, at each clamp and at sectors 0 and K - 1"""
    cells = [(x, y, z if has_z else 0, s) for x, y, z, _ in EDGE_CELLS for s in sorted({0, K - 1, K // 2})]
    keys = keys_of(cells)
    around = set()
    for d in itertools.product((-1, 0, 1), repeat=4):
        want = np.array([python_neighbour(k, *d, K, has_z) for k in keys], np.uint64)
        assert np.array_equal(ref.neighbours(keys, *d, K, has_z), want), d
        assert np.array_equal(ref.product_neighbours(keys, *d, K, has_z), want), d
        around.update((i, int(v)) for i, v in enumerate(want))
    off = ref.product_offsets(keys, K, has_z)                       # what the hook kernel visits: the same set of bins, whatever the order
    assert {(i, int(v)) for i in range(len(keys)) for v in off[i]} | {(i, int(NONE_KEY)) for i in range(len(keys))} == around | {(i, int(NONE_KEY)) for i in range(len(keys))}
    assert np.all((off == NONE_KEY) | ((off & np.uint64(0x8000)) == 0))


@pytest.mark.parametrize("n,span,K,has_z", [(1, 1.0, 36, 0), (2, 1.0, 36, 1), (500, 6.0, 36, 0), (500, 3.0, 36, 1), (3000, 30.0, 8, 0), (2000, 4.0, 2, 1),
                                            (2000, 40.0, 1, 0), (4000, 12.0, 360, 0)])
def test_restatement_matches_flood_fill_random(n, span, K, has_z):
    P, A = particles(n, "half_zero", seed=n + K)
    P["t"] *= np.float32(span / 20.0)
    P["t"][::97, 0] = np.nan
    keys = pf_kld_ref.keys(P, RES_XY, RES_Z if has_z else 0.0, K)
    w = ref.weights(A, float(A["likelihood"]["mean"].max()))
    got = check_against_flood_fill(keys, w, K, has_z)
    assert np.all(got["labels"][::97] == NONE) and np.all(got["labels"][w == 0] == NONE)


def test_two_blobs_one_empty_bin_apart_and_touching_diagonally():
    K = 36
    apart = keys_of(blob(0, 0) + blob(4, 0))                        # columns 0-2 and 4-6: column 3 is empty
    got = check_against_flood_fill(apart, np.ones(len(apart), np.uint64), K, 1)
    assert got["n_clusters"] == 2 and list(got["cbins"]) == [9, 9]
    diagonal = keys_of([(0, 0, 0, 5), (1, 1, 1, 6)])                # one step in each of x, y, z and yaw
    assert check_against_flood_fill(diagonal, [1, 1], K, 1)["n_clusters"] == 1
    assert check_against_flood_fill(keys_of([(0, 0, 0, 5), (1, 1, 1, 7)]), [1, 1], K, 1)["n_clusters"] == 2
    assert check_against_flood_fill(keys_of([(0, 0, 0, 5), (1, 1, 1, 6)]), [1, 1], K, 0)["n_clusters"] == 2    # z not compared: keys with iz != 0 never arise


def test_snake_of_100000_bins_is_one_cluster():
    keys = keys_of(snake())
    assert len(keys) == 100_199
    got = ref.cluster(keys, np.ones(len(keys), np.uint64), 36, 0)
    assert got["n_clusters"] == 1 and got["bins"] == len(keys) and int(got["key"][0]) == int(keys.min())
    cut = np.delete(keys, 50_000)                                   # one bin out: two pieces
    got = ref.cluster(cut, np.ones(len(cut), np.uint64), 36, 0)
    assert got["n_clusters"] == 2 and sorted(int(b) for b in got["cbins"]) == [50_000, 50_198]


def test_yaw_ring_wraps_and_position_does_not():
    K = 36
    ring = keys_of([(0, 0, 0, s) for s in range(0, K, 1) if s not in (10, 20)])     # two gaps: the pieces 21..35 + 0..9 and 11..19
    got = check_against_flood_fill(ring, np.ones(len(ring), np.uint64), K, 0)
    assert got["n_clusters"] == 2 and sorted(int(b) for b in got["cbins"]) == [9, 25]
    ends = keys_of([(-524288, 0, 0, 0), (524287, 0, 0, 0)])
    assert check_against_flood_fill(ends, [1, 1], K, 0)["n_clusters"] == 2
    for K_small in (1, 2):                                          # every sector touches every other: offsets that coincide change nothing
        cells = [(0, 0, 0, s) for s in range(K_small)] + [(2, 0, 0, 0)]
        assert check_against_flood_fill(keys_of(cells), np.ones(len(cells), np.uint64), K_small, 0)["n_clusters"] == 2


def test_zero_likelihood_does_not_bridge_and_nan_is_no_member():
    K = 36
    cells = blob(0, 0) + blob(4, 0) + [(3, 1, 0, 5)]
    P, L = poses_in_bins(cells, K), np.ones(len(cells))
    L[-1] = 0.0                                                     # the particle in the gap
    c = cfg(res_z=RES_Z)
    got = ref.clusters(P, attrs_of(L), c)
    assert got["n_clusters"] == 2 and got["labels"][-1] == NONE and got["n_clustered"] == 18
    L[-1] = 1.0
    assert ref.clusters(P, attrs_of(L), c)["n_clusters"] == 1
    P["R"][-1, 0] = np.nan
    got = ref.clusters(P, attrs_of(L), c)
    assert got["n_clusters"] == 2 and got["labels"][-1] == NONE
    assert ref.clusters(P, attrs_of(np.zeros(len(cells))), c) is None             # every likelihood 0: the set is refused, 0 clusters
    L[3] = -1.0
    assert ref.clusters(P, attrs_of(L), c) is None


def test_one_particle_and_equal_weights():
    K = 36
    got = ref.clusters(poses_in_bins([(2, 3, 0, 1)], K), attrs_of([0.25]), cfg(res_z=RES_Z))
    assert got["n_clusters"] == 1 and got["labels"][0] == 0 and got["weight_total"] == 2 ** 32 and int(got["key"][0]) == int(ref.make_key(2, 3, 0, 1))
    cells = blob(10, 0, side=1) + blob(0, 0, side=1) + blob(5, 0, side=1) + blob(5, 5, side=1) * 2
    got = check_against_flood_fill(keys_of(cells), np.full(len(cells), 7, np.uint64), K, 0)
    assert list(got["weight_int"]) == [14, 7, 7, 7]                 # the tie goes to the smaller key
    assert list(got["key"][1:]) == sorted(got["key"][1:]) and list(got["labels"]) == [3, 1, 2, 0, 0]


def _random_set(n, seed, span):
    P, A = particles(n, "lognormal", seed=seed)
    P["t"] *= np.float32(span / 20.0)
    return P, A


def test_properties():
    P, A = _random_set(5000, 3, 25.0)
    c = cfg()
    got = ref.clusters(P, A, c)
    assert got["n_clusters"] > 10
    assert int(got["weight_int"].sum()) == got["weight_total"] and int(got["members"].sum()) == got["n_clustered"] and int(got["cbins"].sum()) == got["bins"]
    assert np.all(np.diff(got["weight_int"].astype(np.float64)) <= 0)
    perm = np.random.default_rng(1).permutation(len(P))
    again = ref.clusters(P[perm], A[perm], c)
    assert np.array_equal(again["labels"], got["labels"][perm]) and np.array_equal(again["key"], got["key"])
    fine = ref.clusters(P, A, cfg(res_xy=c.res_xy / 2))            # halving res_xy never merges: a fine cluster lies within one coarse cluster
    assert fine["n_clusters"] >= got["n_clusters"]
    for r in range(fine["n_clusters"]):
        assert len(np.unique(got["labels"][fine["labels"] == r])) == 1
