"""The map's BVH on the device, read back through Map.export_blob and checked against the layout contract (tests/bvh_contract.py): the
device LBVH build (the default), the host SAH build, refits and blob imports, on the CPU suite's awkward meshes and on the meshes the
benchmark and the particle-filter tests use.  Then Map.intersect on every build path against the float64 admissible-ray model of
test_gpu_trace_edges.py, with one ray family aimed where a box test that is not conservative would cull a hit.

Printed per mesh and build path: nodes, depth, leaf records, the build and check wall time, and for the traced paths the largest t error
of an admissible ray as a fraction of its bound."""
import time

import numpy as np
import pytest

import bvh_contract as bc
from conftest import mesh
from test_bvh_contract import MESHES, deform, half_area, soup
from test_gpu_trace_edges import EDGE_MARGIN, K_T, U, Scene64, check_intersect, grazing_rays, log, make_rays_for, redraw, unit

HOST_SAH, DEVICE_LBVH = 0, 1


def build(V, F, mode):
    import rmcl_b200
    t0 = time.perf_counter()
    m = rmcl_b200.Map(V, F, device=0, build_mode=mode)
    return m, m.export_blob(), time.perf_counter() - t0


@pytest.mark.gpu
def test_builds_keep_the_contract():
    """Both build modes on every CPU-suite mesh and on building:1000000 / indoor:500000: every node and record checked, info() agrees."""
    big = {"building:1000000": lambda: mesh("building:1000000"), "indoor:500000": lambda: mesh("indoor:500000")}
    for name, make in {**MESHES, **big}.items():
        V, F = make()
        for mode in (DEVICE_LBVH, HOST_SAH):
            m, blob, tb = build(V, F, mode)
            t0 = time.perf_counter()
            info = m.info()
            assert info["build_mode"] == mode and info["n_faces"] == len(F)
            r = bc.check(blob, V, F, info)
            print(f"{name} {'lbvh' if mode else 'sah'}: nodes {r['n_nodes']} depth {r['max_depth']} records {r['n_tris']}; "
                  f"build {tb * 1e3:.0f} ms, check {(time.perf_counter() - t0) * 1e3:.0f} ms")


@pytest.mark.gpu
def test_lbvh_canonical_form():
    """The LBVH build allocates nodes and records with atomics, so their order may vary, but two builds of one mesh are the same tree; and
    the tree of V * 2^k is the tree of V with boxes times 2^k (the Morton code (c - lo) / ext, the area comparisons and the octant costs
    all scale exactly) for k across log2(root half-area * n_faces) in [-100, 120]."""
    for name in ("soup25", "duplicates1000", "one_centroid1000", "degenerate", "sheets", "geometric2000", "awkward_soup:300", "building:60000",
                 "indoor:20000"):
        V, F = MESHES[name]()
        a, b = bc.canonical(build(V, F, DEVICE_LBVH)[1]), bc.canonical(build(V, F, DEVICE_LBVH)[1])
        assert a == b, (name, bc.first_difference(a, b))
    V, F = soup(2000)
    blob0 = build(V, F, DEVICE_LBVH)[1]
    l0 = np.log2(half_area(V) * len(F))
    ks = [k for k in range(-80, 80, 3) if -100 <= l0 + 2 * k <= 120]
    for k in ks:
        Vk = (V.astype(np.float64) * 2.0 ** k).astype(np.float32)
        _, blob, _ = build(Vk, F, DEVICE_LBVH)
        bc.check(blob, Vk, F)
        ck, want = bc.canonical(blob), bc.canonical(blob0, 2.0 ** k)
        assert ck == want, (k, bc.first_difference(ck, want))
    print(f"lbvh soup2000: identical trees at k = {ks[0]} .. {ks[-1]} (step 3)")


@pytest.mark.gpu
def test_refit_keeps_the_contract():
    """b2_mesh_refit after test_refit_dynamic_map_gpu's deformation and after scaling by 1000 and shifting by 1e4: the contract holds on the
    moved mesh and abs_max follows; a refitted map survives export_blob -> from_blob; refitting back to V reproduces the original export."""
    import rmcl_b200
    V, F = mesh("building:200000")
    m, blob0, _ = build(V, F, DEVICE_LBVH)
    bc.check(blob0, V, F, m.info())
    for what, V2 in (("deformed", deform(V, 12)), ("scaled and shifted", (V.astype(np.float64) * 1000 + 1e4).astype(np.float32))):
        m.refit(V2)
        b = m.export_blob()
        r = bc.check(b, V2, F, m.info())
        assert (bc.parse(b)[0]["abs_max"] == np.abs(V2).max(0)).all(), what
        m2 = rmcl_b200.Map.from_blob(b)
        b2 = m2.export_blob()
        assert np.array_equal(b2, b), what
        bc.check(b2, V2, F, m2.info())
        m.refit(V)
        assert np.array_equal(m.export_blob(), blob0), what
        print(f"refit {what}: nodes {r['n_nodes']} depth {r['max_depth']} records {r['n_tris']}; blob round trip and refit back identical")
    with pytest.raises(rmcl_b200.B2Error):
        m.refit(np.full_like(V, 2.0 ** 63))
    assert np.array_equal(m.export_blob(), blob0)


def box_edge_rays(sc, blob, reach):
    """Rays at the box test's weak spot: for a random leaf slot and a random side of its box on a random axis, the triangle that attains
    that plane, aimed at an interior point next to the vertex on the plane (twice the model's edge margin in from its edges), at grazing incidence
    (|cos| in [0.02, 0.2]) from reach * [0.5, 5] before it.  A box that misses its triangles by an ulp, or slack that is not conservative,
    turns these hits into misses."""
    hd, nodes, tris = bc.parse(blob)
    meta = nodes["meta"].astype(np.int64)
    leaf = (meta != 0) & (((nodes["masks"][:, None].astype(np.int64) & 0xFF) >> np.arange(8)) & 1 == 0)
    ln, ls = np.nonzero(leaf)
    cnt = bc._counts(meta)[ln, ls]
    first = nodes["tri_base"][ln].astype(np.int64) + (meta[ln, ls] & 0x1F)
    P = np.stack([tris["v0"], tris["v1"], tris["v2"]], 1).astype(np.float64)        # (T, 3, 3)
    face = tris["face"].astype(np.int64)

    def make(k, rng):
        o, d = np.zeros((k, 3), np.float32), np.zeros((k, 3), np.float32)
        done = 0
        for _ in range(200 * k):
            if done == k:
                break
            j = rng.integers(0, len(ln))
            ax, side = rng.integers(0, 3), rng.integers(0, 2)
            plane = (nodes["hi"] if side else nodes["lo"])[ln[j], ax, ls[j]]
            recs = first[j] + np.arange(cnt[j])
            hitv = np.argwhere(P[recs, :, ax] == plane)                             # (record, vertex) on the plane
            r, vi = hitv[rng.integers(0, len(hitv))]
            f = face[recs[r]]
            if sc.zero[f]:
                continue
            v = P[recs[r]]
            vj, vk = v[(vi + 1) % 3], v[(vi + 2) % 3]
            c = rng.uniform(0.02, 0.2)
            margin = 2 * (EDGE_MARGIN + K_T * U * sc.kappa[f] * 3 * sc.E) / c             # twice the model's margin across the ray at S = 3 E
            delta = margin * sc.diam[f] / sc.nNg[f]                                     # p is delta |Ng| / |edge| >= margin from both edges at vi
            if delta > 0.3:
                continue                                                             # a sliver: no interior point far enough from its edges
            p = (1 - 2 * delta) * v[vi] + delta * (vj + vk)
            n = sc.Ng[f] / sc.nNg[f]
            t = unit(np.cross(n, rng.normal(size=3)))
            dd = unit(np.sqrt(1 - c * c) * t - c * n * rng.choice([-1.0, 1.0]))
            o[done], d[done] = p - dd * (rng.uniform(0.5, 5.0) * reach + 2 * sc.diam[f]), dd      # from afar: rho <= 1.5 in COS_MIN
            done += 1
        assert done == k, "no leaf slot offers a box-plane ray"
        return o, d
    return make


def trace_case(label, sc, gm, blob, main, reach, seed):
    """1200 admissible rays of `main` (with grazing rays mixed in) and 600 box-plane rays through Map.intersect against the float64 model"""
    t0 = time.perf_counter()
    r = bc.check(blob, sc.V, sc.F, gm.info())
    edge = box_edge_rays(sc, blob, reach)
    worst = 0.0
    for fam, make, n in (("mixed", main, 1200), ("box planes", edge, 600)):
        o, d, ref, redrawn = redraw(sc, make, n, seed)
        t, f, ng, h = gm.intersect(o, d)
        s = check_intersect(sc, ref, t, f, ng, h, np.inf, f"{label} {fam}")
        log(f"{label} {fam}", s, redrawn)
        assert s["hits"] >= n // 3, (label, fam, s)
        worst = max(worst, s["worst_t"])
    print(f"{label}: nodes {r['n_nodes']} depth {r['max_depth']} records {r['n_tris']}; worst t error / bound {worst:.3f}; "
          f"{time.perf_counter() - t0:.1f} s")


def shifted(make, s, shift):
    def f(k, rng):
        o, d = make(k, rng)
        return (o.astype(np.float64) * s + shift).astype(np.float32), d
    return f


@pytest.mark.gpu
def test_trace_on_every_build_path():
    """Map.intersect against the float64 model on the host SAH build, a map re-imported from a blob, a deformed refit and a scaled and
    shifted refit (the default LBVH build is traced by test_gpu_trace_edges.py)."""
    import rmcl_b200
    for name in ("degenerate", "indoor"):
        sc = Scene64(name)
        gm, blob, _ = build(sc.V, sc.F, HOST_SAH)
        trace_case(f"{name} host sah", sc, gm, blob, make_rays_for(sc), 1.0, 3)
        lb, lblob, _ = build(sc.V, sc.F, DEVICE_LBVH)
        imp = rmcl_b200.Map.from_blob(lblob)
        trace_case(f"{name} lbvh from blob", sc, imp, imp.export_blob(), make_rays_for(sc), 1.0, 4)
    base = Scene64("indoor")
    V2 = deform(base.V, 12)
    sc2 = Scene64("indoor", V2, base.F)                                               # room rays of the indoor scene
    gm, _, _ = build(base.V, base.F, DEVICE_LBVH)
    gm.refit(V2)
    trace_case("indoor lbvh deformed refit", sc2, gm, gm.export_blob(), make_rays_for(sc2), 1.0, 5)
    V3 = (base.V.astype(np.float64) * 1000 + 1e4).astype(np.float32)
    sc3 = Scene64("indoor scaled", V3, base.F)
    gm.refit(V3)
    main = shifted(make_rays_for(base), 1000.0, 1e4)
    graze = grazing_rays(sc3)

    def mixed(k, rng):
        a, b = main(k, rng), graze(k, rng)
        g = rng.random(k) < 0.25
        return np.where(g[:, None], b[0], a[0]), np.where(g[:, None], b[1], a[1])
    trace_case("indoor lbvh refit x1000 + 1e4", sc3, gm, gm.export_blob(), mixed, 1000.0, 6)


@pytest.mark.gpu
def test_huge_coordinates():
    """Near FLT_MAX (2e38) both builds refuse the mesh, as do a refit to such vertices; at exactly 2^62 both build a tree that keeps the
    contract and one ulp above they refuse.  (A tree built at 2e38 would lose faces: the octant assignment's centres overflow and a child is
    written to slot -1; the contract's face count catches that.)"""
    import rmcl_b200
    V, F = soup(64)
    for mode in (DEVICE_LBVH, HOST_SAH):
        Vh = (V.astype(np.float64) * (2e38 / 1.05)).astype(np.float32)
        assert np.isfinite(Vh).all()
        with pytest.raises(rmcl_b200.B2Error) as e:
            build(Vh, F, mode)
        assert "2^62" in str(e.value)
        s = 2.0 ** 62 / np.abs(V.astype(np.float64)).max()
        Ve = (V.astype(np.float64) * s).astype(np.float32)
        if np.abs(Ve).max() > 2.0 ** 62:
            Ve = np.minimum(Ve, np.float32(2.0 ** 62))
        assert np.abs(Ve).max() == 2.0 ** 62
        m, blob, _ = build(Ve, F, mode)
        bc.check(blob, Ve, F, m.info())
        Vo = Ve.copy()
        i = np.unravel_index(np.argmax(np.abs(Vo)), Vo.shape)
        Vo[i] = np.nextafter(Vo[i], np.float32(np.inf))
        with pytest.raises(rmcl_b200.B2Error):
            build(Vo, F, mode)
