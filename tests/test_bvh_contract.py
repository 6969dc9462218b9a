"""CPU tests of the host SAH build (bvh_build.cpp) and the per-node refit against the BVH layout contract (tests/bvh_contract.py), through
the emulation harness's export of the host-built tree in the blob layout.

Power-of-two scale invariance: scaling every vertex by 2^k scales every box, centre, area (by 4^k), SAH cost (by 4^k) and octant slot
cost exactly, as long as none of them leaves the normal float range.  The build must then make the same decisions, so the scaled tree is
the unscaled one byte for byte, boxes times 2^k.  A cost sentinel below the largest cost, or an overflow to inf or NaN, breaks that first.
Beyond that range, up to coordinates near FLT_MAX, the build either refuses the mesh or builds a tree that keeps the contract."""
import numpy as np
import pytest

import bvh_contract as bc
from conftest import mesh


@pytest.fixture(scope="module")
def pe():
    import pyemul
    pyemul.lib()
    return pyemul


def soup(n, scale=1.0, seed=0):
    """n triangles of a few percent of the scene's size, centres in [0.5, 1]^3 * scale"""
    rng = np.random.default_rng(seed)
    c = rng.uniform(0.5, 1.0, (n, 1, 3))
    V = (c * (1 + rng.uniform(-0.05, 0.05, (n, 3, 3))) * scale).reshape(-1, 3).astype(np.float32)
    return V, np.arange(3 * n, dtype=np.uint32).reshape(n, 3)


def awkward_soup(scale, seed=0):
    """400 triangles with zero-area faces, exact duplicates, a coplanar sheet and slivers mixed in (as test_emul_parity's soups)"""
    rng = np.random.default_rng(100 + seed)
    n = 400
    tri = rng.uniform(-1, 1, (n, 1, 3)) * scale + rng.normal(0, 0.15 * scale, (n, 3, 3))
    tri[:20, 2] = tri[:20, 1]
    tri[20:40] = tri[40:60]
    tri[60:80, :, 2] = 0.25 * scale
    tri[80:100, 2] = tri[80:100, 0] + (tri[80:100, 1] - tri[80:100, 0]) * 0.5 + rng.normal(0, 1e-6 * scale, (20, 3))
    return tri.reshape(-1, 3).astype(np.float32), np.arange(3 * n, dtype=np.uint32).reshape(n, 3)


def duplicates(n=1000):
    V = np.tile(np.array([[1.0, 2.0, 3.0], [2.5, 2.0, 3.5], [1.5, 4.0, 3.0]], np.float32), (n, 1))
    return V, np.arange(3 * n, dtype=np.uint32).reshape(n, 3)


def one_centroid(n=1000):
    """n different triangles whose boxes all have the exact centre (1, 2, 3): vertices c - a, c + a and c + a * w, w in (-1, 1), all dyadic"""
    rng = np.random.default_rng(4)
    c = np.array([1.0, 2.0, 3.0])
    a = rng.integers(100, 1024, (n, 3)) / 1024.0
    w = rng.integers(-1023, 1024, (n, 3)) / 1024.0
    tri = np.stack([c - a, c + a, c + a * w], 1)
    return tri.reshape(-1, 3).astype(np.float32), np.arange(3 * n, dtype=np.uint32).reshape(n, 3)


def sheets():
    """two axis-aligned sheets of 2 x 30 x 30 triangles: every triangle of one sheet has the same z (the other the same x)"""
    g = np.linspace(0.0, 9.0, 31)
    X, Y = np.meshgrid(g, g, indexing="ij")
    q = np.stack([X[:-1, :-1], Y[:-1, :-1], X[1:, :-1], Y[1:, :-1], X[1:, 1:], Y[1:, 1:], X[:-1, 1:], Y[:-1, 1:]], -1).reshape(-1, 4, 2)
    quads = np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]])                      # (1800, 3, 2)
    z = np.concatenate([quads, np.full(quads.shape[:2] + (1,), 1.5)], 2)
    x = np.concatenate([np.full(quads.shape[:2] + (1,), 4.25), quads], 2)
    tri = np.concatenate([z, x])
    return tri.reshape(-1, 3).astype(np.float32), np.arange(3 * len(tri), dtype=np.uint32).reshape(-1, 3)


def geometric(n=2000, r=1.02):
    """triangles at x = r^i: the binned SAH peels one end at a time, the deepest tree of these meshes"""
    x = r ** np.arange(n)
    tri = np.zeros((n, 3, 3))
    tri[:, :, 0] = x[:, None]
    tri[:, 1, 1] = 1.0
    tri[:, 2, 2] = 1.0
    return tri.reshape(-1, 3).astype(np.float32), np.arange(3 * n, dtype=np.uint32).reshape(n, 3)


def degenerate():
    from test_gpu_trace_edges import degenerate_mesh
    return degenerate_mesh()


MESHES = {
    **{f"soup{n}": (lambda n=n: soup(n, seed=n)) for n in (1, 2, 3, 4, 8, 9, 24, 25)},
    "duplicates1000": duplicates,
    "one_centroid1000": one_centroid,
    "degenerate": degenerate,
    "sheets": sheets,
    "geometric2000": geometric,
    **{f"awkward_soup:{s:g}": (lambda s=s: awkward_soup(s, seed=int(s * 1000) % 7)) for s in (1e-3, 0.1, 1.0, 300.0)},
    "building:60000": lambda: mesh("building:60000"),
    "indoor:20000": lambda: mesh("indoor:20000"),
}


def build(pe, V, F):
    s = pe.Scene(V, F)
    return s, s.export_blob()


@pytest.mark.parametrize("name", list(MESHES))
def test_host_build_contract(pe, name):
    V, F = MESHES[name]()
    _, blob = build(pe, V, F)
    r = bc.check(blob, V, F)
    if name == "geometric2000":
        assert r["max_depth"] >= 12, r                                          # keeps the deep case deep
    print(name, r)


def half_area(V):
    e = V.astype(np.float64).max(0) - V.astype(np.float64).min(0)
    return e[0] * e[1] + e[1] * e[2] + e[2] * e[0]


def assert_scaled(blob0, blob, k):
    """blob is blob0's tree with every box and vertex times 2^k: everything else byte-identical"""
    h0, n0, t0 = bc.parse(blob0)
    h, n, t = bc.parse(blob)
    assert (len(n0), len(t0), int(h0["max_depth"])) == (len(n), len(t), int(h["max_depth"])), (k, "tree size / depth")
    for f in ("child_base", "tri_base", "masks", "pad0", "meta", "pad"):
        assert np.array_equal(n0[f], n[f]), (k, f, int(np.argwhere((n0[f] != n[f]).reshape(len(n), -1).any(1))[0, 0]))
    for f in ("lo", "hi"):
        bad = ~(n0[f].astype(np.float64) * 2.0 ** k == n[f]).all((1, 2))
        assert not bad.any(), (k, f"{f} is not the unscaled box times 2^k", int(np.flatnonzero(bad)[0]))
    assert np.array_equal(t0["face"], t["face"]), (k, "record face order")


@pytest.mark.parametrize("name", ["soup2000", "degenerate"])
def test_host_build_power_of_two_scale_invariance(pe, name):
    """Every k with log2(root half-area * n_faces) in [-100, 120]: the tree of V * 2^k is the tree of V, boxes times 2^k (at the parent
    commit a 1e30 cost sentinel made the 2000-face soup build a different tree from k = 46 on and one node holding every face from 48)."""
    V, F = soup(2000) if name == "soup2000" else degenerate()
    _, blob0 = build(pe, V, F)
    bc.check(blob0, V, F)
    l0 = np.log2(half_area(V) * len(F))
    ks = [k for k in range(-80, 80) if -100 <= l0 + 2 * k <= 120]
    assert len(ks) >= 100
    for k in ks:
        Vk = (V.astype(np.float64) * 2.0 ** k).astype(np.float32)
        assert np.array_equal(Vk.astype(np.float64), V.astype(np.float64) * 2.0 ** k)
        _, blob = build(pe, Vk, F)
        assert_scaled(blob0, blob, k)
    print(name, f"k = {ks[0]} .. {ks[-1]}: identical trees")


def test_host_build_huge_coordinates(pe):
    """Past the scale-invariant range, up to coordinates near FLT_MAX: either the build refuses the mesh (coordinates above 2^62) or the
    tree keeps the contract; no face may be lost (the parent packed 2000 faces into one leaf slot from extents of 1e15 on, and lost every
    face at 3e38)."""
    V, F = soup(2000)
    l0 = np.log2(half_area(V) * len(F))
    built, refused = [], []
    for k in list(range(int(np.floor((120 - l0) / 2)) + 1, 128)):
        Vk = (V.astype(np.float64) * 2.0 ** k).astype(np.float32)
        assert np.isfinite(Vk).all()
        try:
            _, blob = build(pe, Vk, F)
        except RuntimeError as e:
            assert "2^62" in str(e), e
            assert np.abs(Vk).max() > 2.0 ** 62
            refused.append(k)
            continue
        bc.check(blob, Vk, F)
        built.append(k)
    # the issue's meshes: fresh soups at extents 1e15 .. 1e19 and 64 faces at 3e38
    for ext, n in ((1e15, 2000), (1e16, 2000), (1e18, 2000), (1e19, 2000), (3e38, 64)):
        Vs, Fs = soup(n, ext / 1.05, seed=int(np.log10(ext)))
        try:
            _, blob = build(pe, Vs, Fs)
        except RuntimeError as e:
            assert "2^62" in str(e) and np.abs(Vs).max() > 2.0 ** 62, (ext, e)
            continue
        bc.check(blob, Vs, Fs)
    assert built and refused
    print(f"built and checked at k = {built}, refused at k = {refused[0]} .. {refused[-1]}")


def deform(V, seed=21):
    """test_refit_dynamic_map_gpu's deformation: every vertex moved by centimetres plus a smooth bend"""
    rng = np.random.default_rng(seed)
    V2 = (V + rng.normal(0, 0.02, V.shape)).astype(np.float32)
    V2[:, 0] += (0.3 * np.sin(V[:, 1] * 0.2)).astype(np.float32)
    return V2


def test_host_refit_contract(pe):
    """emul_refit (the product's bvh8_refit_node over the host-built tree): the contract holds on the deformed mesh and on the mesh scaled
    by 1000 and shifted by 1e4 (abs_max follows), and refitting back to V gives the original tree byte for byte."""
    V, F = mesh("building:60000")
    s, blob0 = build(pe, V, F)
    for what, V2 in (("deformed", deform(V)), ("scaled and shifted", (V.astype(np.float64) * 1000 + 1e4).astype(np.float32))):
        s.refit(V2, F)
        b = s.export_blob()
        bc.check(b, V2, F)
        assert (bc.parse(b)[0]["abs_max"] == np.abs(V2).max(0)).all(), what
        s.refit(V, F)
        assert np.array_equal(s.export_blob(), blob0), what
