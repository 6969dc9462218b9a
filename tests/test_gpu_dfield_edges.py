"""GPU tests of the distance field's device build (k_dfield_classify, the exclusive scan, k_dfield_index, k_dfield_fill), its lookup
(k_dfield_query) and the field update (k_pf_update_field, pf_prepare_beams' tile) at their grid and launch edges.  The primary reference is
the oracle's closest point (tests/dfield_ref.py: RefField) and the float64 restatements (node_points, lookup64, beam_points64, evaluate64,
merge64); the product's functions compiled for the host (ProductField, lookup, pf_update) are the secondary, bit-exact one.

Tolerances.
  * node values, allocation, unallocated bricks, fields built on different trees: exact (bit patterns).  The allocation rule is
    dist(brick centre) < trunc + 8h with the limit rounded as the product rounds it (add(trunc, mul(8, h))).
  * lookup: bit-identical to the host product; within 8 ulp of trunc of lookup64 over the downloaded nodes (test_dfield.py); inside the
    box, within (sqrt(3)/2) h + 1e-5 (1 + max |coordinate|) of the clamped oracle distance (test_accuracy_bound).
  * field update: bit-identical to the host product; n_meas exact against merge64.  Mean and sigma against merge64 within
    2e-6 + 5 k 2^-24 M, k the number of merged beams and M the largest magnitude entering a merge step (the evaluations, the initial
    mean and sigma, the squared evaluations).  Each merge step rounds a few float32 operations of size at most M, its float32 weights
    n / (n + 1) and 1 / (n + 1) are within 2^-24 of the exact ones, and a step multiplies the error already made by w1 <= 1, so the
    error grows at most linearly in k.  After the MAX_N_MEAS clamp the weights' rounding biases every step the same way, so the
    linear growth is reached (about 1e-4 at 19 000 beams).
The build-edge cases print the grid, the bricks total and allocated and the grid-stride passes of classify / index and of fill."""
import math

import numpy as np
import pytest

import dfield_ref as R

pytestmark = pytest.mark.gpu

C_HALF_SQRT3 = math.sqrt(3.0) / 2.0


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cap():
    """threads of one grid-stride pass of the build: dfield_grid's n_sm * 64 blocks of 256"""
    return _n_sm() * 64 * 256


def _passes(n):
    """grid-stride passes of dfield_grid(n_sm, n)"""
    grid = max(1, min(-(-n // 256), _n_sm() * 64))
    return -(-n // (grid * 256))


def _two(V, F, off):
    """the mesh and a copy shifted by off"""
    V = np.asarray(V, np.float32)
    return np.concatenate([V, V + np.asarray(off, np.float32)]), np.concatenate([F, F + len(V)]).astype(np.uint32)


def _map(V, F, mode):
    import rmcl_b200
    return rmcl_b200.Map(V, F, build_mode=mode)


def _field(m, h, trunc, lo=None, hi=None):
    import rmcl_b200
    return rmcl_b200.DistanceField(m, h, trunc, lo, hi)


def _grid(V, h, trunc, lo=None, hi=None):
    if lo is None:
        lo, hi = R.default_box(V, trunc)
    g = R.Grid(lo, hi, h, trunc)
    assert g.refused is None, g.refused
    return g


def _centre_dist(ref, g, ta):
    """the oracle's distance from every brick centre, +inf where a float64 lower bound (RefField.lower_bound) already exceeds ta by more
    than the oracle's float32 rounding could make up (1e-5 of the coordinates' size): the rule leaves those bricks unallocated either way"""
    c = R.brick_centres(g)
    far = ref.lower_bound(c) > float(ta) + 1e-5 * (1.0 + np.abs(c.astype(np.float64)).max(1))
    dc = np.full(len(c), np.inf, np.float32)
    dc[~far] = ref.dist(c[~far])
    return dc


def check_build(what, V, F, f, g, ref, host=True, brute=2000, margin=1024):
    """the downloaded field against the contract: grid and info, slots in brick order, every node of every allocated brick equal to the
    oracle's clamped distance (through its BVH; a sample brute force), the allocation rule over every brick centre, every node of the
    `margin` unallocated bricks nearest the margin equal to trunc, and (host) the host product's build byte for byte -> (index, bricks)"""
    inf = f.info()
    assert inf["dims"] == g.dims and inf["brick_dims"] == g.bdims and inf["bricks_total"] == g.n_bricks
    assert np.array_equal(np.asarray(inf["origin"], np.float32), g.lo) and inf["inv_resolution"] == g.inv_h
    index, bricks = f.download()
    flat = index.reshape(-1)
    ids = np.flatnonzero(flat != R.NOBRICK)
    assert inf["bricks_allocated"] == len(ids) == len(bricks)
    assert np.array_equal(flat[ids], np.arange(len(ids), dtype=np.uint32))
    assert inf["bytes"] == 4 * g.n_bricks + 4 * 729 * len(ids)
    trunc = np.float32(g.trunc)
    if len(ids):
        P = R.node_points(g, ids).reshape(-1, 3)
        got = bricks.reshape(-1)
        assert np.array_equal(_bits(ref.values(P, g.trunc)), _bits(got)), what
        k = np.random.default_rng(11).choice(len(P), min(len(P), brute), replace=False)
        assert np.array_equal(_bits(ref.values(P[k], g.trunc, brute=True)), _bits(got[k])), what
    ta = trunc + np.float32(8.0) * np.float32(g.h)
    dc = _centre_dist(ref, g, ta)
    assert np.array_equal(flat != R.NOBRICK, dc < ta), (what, int(((flat != R.NOBRICK) != (dc < ta)).sum()))
    un = np.flatnonzero(flat == R.NOBRICK)
    if len(un):
        near = un if len(un) <= margin else un[np.argpartition(dc[un], margin)[:margin]]
        assert (ref.values(R.node_points(g, near).reshape(-1, 3), g.trunc) == trunc).all(), what
    if host:
        hi_, hb = R.ProductField(V, F).build(g)
        assert hi_.tobytes() == index.tobytes() and hb.tobytes() == bricks.tobytes(), what
    print(f"{what}: dims {g.dims} bricks {g.bdims} = {g.n_bricks} total, {len(ids)} allocated; classify/index passes {_passes(g.n_bricks)}, "
          f"fill passes {_passes(len(ids) * 729) if len(ids) else 0} (cap {_cap()} threads)")
    return index, bricks


# ---------------------------------------------------------------- 1. node values and allocation on every tree ------------------------
def _small(name):
    from rmcl_b200 import synth
    return {"cube": synth.cube(5), "uvsphere": synth.uvsphere(12, 8), "indoor": synth.indoor(2000)}[name]


# (mesh, h, trunc, box growth beyond the map's AABB): growth None is the default box (trunc), which for the cube puts the origin at
# -11.5 so that nodes lie on its faces and exactly trunc from them; growth trunc + 24h puts brick centres within h outside the margin;
# growth trunc + 12h puts the cube's outer brick centres exactly trunc + 8h off its faces (all values binary-exact), where the strict
# rule leaves them unallocated
TREE_CASES = [("cube", 0.5, 1.5, None), ("cube", 0.5, 1.5, "margin"), ("cube", 0.5, 1.5, "tie"), ("cube", 0.3, 0.7, "margin"),
              ("uvsphere", 0.25, 0.6, "margin"), ("indoor", 0.2, 0.3, "margin"), ("indoor", 0.25, 0.5, None)]


@pytest.mark.parametrize("name,h,trunc,box", TREE_CASES)
def test_every_tree_gives_the_oracle_field(name, h, trunc, box):
    """fields on the host SAH tree, the device LBVH and an LBVH refitted from moved vertices to the mesh download byte-identically, and
    that field is the oracle's; a field built before the refit stays as built"""
    V, F = _small(name)
    lo = hi = None
    if box == "margin":
        lo, hi = R.default_box(V, trunc + 24 * h)
    if box == "tie":
        lo, hi = R.default_box(V, trunc + 12 * h)
    g = _grid(V, h, trunc, lo, hi)
    ref = R.RefField(V, F)
    f_sah = _field(_map(V, F, 0), h, trunc, lo, hi)
    index, bricks = check_build(f"{name} h {h} trunc {trunc} {box or 'default'} box (SAH)", V, F, f_sah, g, ref)
    if name == "cube" and box is None:
        P = R.node_points(g, np.flatnonzero(index.reshape(-1) != R.NOBRICK)).reshape(-1, 3)
        assert (bricks == 0).any() and (np.abs(np.abs(P).max(1) - 11.5) == 0).any()       # on the faces, exactly trunc off them
    if box in ("margin", "tie"):
        dc = ref.dist(R.brick_centres(g))
        ta = np.float32(trunc) + np.float32(8.0) * np.float32(h)
        assert ((dc >= ta) & (dc < ta + np.float32(h))).any()
        if box == "tie":
            assert (dc == ta).any()
    want = (index.tobytes(), bricks.tobytes())
    f_lbvh = _field(_map(V, F, 1), h, trunc, lo, hi)
    assert f_lbvh.download()[0].tobytes() == want[0] and f_lbvh.download()[1].tobytes() == want[1]
    rng = np.random.default_rng(3)
    Vm = (V * np.float32(1.07) + rng.normal(0, 0.05, V.shape)).astype(np.float32)
    m = _map(Vm, F, 1)
    before = _field(m, h, trunc, lo, hi)
    snap = [a.tobytes() for a in before.download()]
    m.refit(V)
    after = _field(m, h, trunc, lo, hi)
    ia, ba = after.download()
    assert ia.tobytes() == want[0] and ba.tobytes() == want[1]
    assert [a.tobytes() for a in before.download()] == snap


_LARGE = {}


def _large():
    """indoor:500000 at h 0.05, trunc 1: built once per module on both trees (more allocated nodes than one grid-stride pass of fill)"""
    if not _LARGE:
        from conftest import mesh
        V, F = mesh("indoor:500000")
        h, trunc = 0.05, 1.0
        maps = {mode: _map(V, F, mode) for mode in (0, 1)}
        _LARGE.update(V=V, F=F, g=_grid(V, h, trunc), ref=R.RefField(V, F), maps=maps, fields={mode: _field(maps[mode], h, trunc) for mode in maps})
    return _LARGE


def test_large_map_on_both_trees():
    L = _large()
    index, bricks = check_build("indoor:500000 h 0.05 trunc 1 (LBVH)", L["V"], L["F"], L["fields"][1], L["g"], L["ref"], host=False)
    assert len(bricks) * 729 > _cap()
    i0, b0 = L["fields"][0].download()
    assert i0.tobytes() == index.tobytes() and b0.tobytes() == bricks.tobytes()
    L["index"], L["bricks"] = index, bricks


# ---------------------------------------------------------------- 2. grid and launch-geometry edges of the build -----------------------
def _edge_case(case):
    """-> (V, F, h, trunc, lo, hi) of a build edge"""
    from rmcl_b200 import synth
    V, F = synth.cube(5)                                                              # [-10, 10]^3
    if case == "one_cell_z":                                                          # dims z 2; 46 x 31 cells: last bricks part outside
        return V, F, 0.5, 1.5, (-11.3, -11.3, 0.1), (11.2, 3.9, 0.4)
    if case == "one_cell_x":
        return V, F, 0.25, 0.6, (9.9, -10.7, -10.9), (10.1, 10.7, 3.3)
    if case == "trunc_below_h":                                                       # origin -11.5: nodes on the faces hold 0
        return V, F, 0.5, 0.01, (-11.5, -11.5, -11.5), (11.5, 11.5, 11.5)
    if case == "trunc_above_map":                                                     # every brick allocated; fill over the cap
        return V, F, 0.5, 50.0, (-40.0, -40.0, -40.0), (40.0, 40.0, 40.0)
    if case == "far_from_origin":                                                     # node positions round at 1e4 m
        V = (V + np.float32([1e4, -1e4, 1e4])).astype(np.float32)
        lo, hi = R.default_box(V, 0.7)
        return V, F, 0.3, 0.7, lo, hi
    if case == "over_the_cap":
        # a thin box (one brick in z) of more than two grid-stride passes of bricks, a cube in each far corner: the far cube's bricks are
        # classified in the last pass
        h, bx = 0.5, 1024
        by = -(-int(2.2 * _cap()) // bx)
        off = (8 * h * (bx - 6), 8 * h * (by - 6), 0.0)
        V2, F2 = _two(V, F, off)
        return V2, F2, h, 1.0, (-12.0, -12.0, -11.0), (-12.0 + 8 * h * bx, -12.0 + 8 * h * by, -9.0)
    if case == "axis_limit":
        # 8 (2^21 - 1) cells on x: 2^24 - 7 nodes, the last brick's far face at node 2^24 - 8; a cube at each end
        n = 8 * (2 ** 21 - 1)
        V2, F2 = _two(V, F, (n - 40.0, 0.0, 0.0))
        return V2, F2, 1.0, 1.0, (-12.0, -1.5, -1.5), (-12.0 + n, -0.5, -0.5)
    raise KeyError(case)


EDGE_CASES = ["one_cell_z", "one_cell_x", "trunc_below_h", "trunc_above_map", "far_from_origin", "over_the_cap", "axis_limit"]


@pytest.mark.parametrize("case", EDGE_CASES)
def test_build_edges(case):
    V, F, h, trunc, lo, hi = _edge_case(case)
    g = _grid(V, h, trunc, np.float32(lo), np.float32(hi))
    ref = R.RefField(V, F)
    f = _field(_map(V, F, 1), h, trunc, lo, hi)
    index, bricks = check_build(f"{case}", V, F, f, g, ref)
    n_alloc = len(bricks)
    if case == "one_cell_z":
        assert g.dims[2] == 2 and g.dims[0] % 8 != 1 and g.dims[1] % 8 != 1
    if case == "one_cell_x":
        assert g.dims[0] == 2 and g.dims[1] % 8 != 1 and g.dims[2] % 8 != 1
    if case == "trunc_below_h":
        assert 0 < n_alloc < g.n_bricks and (bricks == 0).any() and (bricks == np.float32(trunc)).any()
    if case == "trunc_above_map":
        assert n_alloc == g.n_bricks and n_alloc * 729 > _cap()
    if case == "over_the_cap":
        assert g.n_bricks > 2 * _cap() and _passes(g.n_bricks) >= 3
        ids = np.flatnonzero(index.reshape(-1) != R.NOBRICK)
        assert ids.min() < _cap() and ids.max() >= 2 * _cap()                          # bricks allocated in the first and the last pass
    if case == "axis_limit":
        assert g.dims[0] == 2 ** 24 - 7 and g.bdims[0] == 2 ** 21 - 1
        ids = np.flatnonzero(index.reshape(-1) != R.NOBRICK)
        assert ids.min() < 8 and ids.max() > 2 ** 21 - 8
    # lookups on the device: near both ends of every axis and at random
    rng = np.random.default_rng(5)
    top = (g.lo + (np.array(g.dims) - 1).astype(np.float32) * np.float32(g.h)).astype(np.float64)
    span = np.minimum(top - g.lo, 40.0)
    pts = np.concatenate([rng.uniform(g.lo - 1.0, g.lo + span, (50_000, 3)), rng.uniform(top - span, top + 1.0, (50_000, 3)),
                          rng.uniform(g.lo, top, (50_000, 3)), np.stack([g.lo, top])]).astype(np.float32)
    got = f.query(pts)
    assert got.tobytes() == R.lookup(g, index, bricks, pts).tobytes()
    want = R.lookup64(g, index, bricks, pts)
    assert np.abs(got.astype(np.float64) - want).max() <= 8 * float(np.spacing(np.float32(trunc)))


def test_no_brick_allocated():
    """a box farther than trunc + 8h from the map everywhere: no brick, the index all B2_NOBRICK, lookups trunc (finite) and +inf
    (non-finite), and the field update is the float64 update with e = trunc"""
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    V, F = synth.cube(5)
    h, trunc, lo, hi = 0.5, 1.0, (100.0, 100.0, 100.0), (110.0, 103.0, 102.7)
    m = _map(V, F, 1)
    f = _field(m, h, trunc, lo, hi)
    g = _grid(V, h, trunc, np.float32(lo), np.float32(hi))
    index, bricks = check_build("no brick", V, F, f, g, R.RefField(V, F))
    inf = f.info()
    assert inf["bricks_allocated"] == 0 and len(bricks) == 0 and inf["bytes"] == 4 * inf["bricks_total"]
    assert (index == R.NOBRICK).all()
    rng = np.random.default_rng(8)
    pts = np.concatenate([rng.uniform(95.0, 115.0, (10_000, 3)),
                          [[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1e30, 0, 0], [101, 101, 101], [0, 0, 0]]]).astype(np.float32)
    fin = np.isfinite(pts).all(1)
    for got in (f.query(pts), f.query(torch.from_numpy(pts).cuda()).cpu().numpy()):
        assert (got[fin] == np.float32(trunc)).all() and np.isposinf(got[~fin]).all()
    # the update
    up = rmcl_b200.PCDSensorUpdaterB200(m)
    up.setDistanceField(f)
    P, A, B, Tsb = _pf_case(257, 33, 4, centre=(105.0, 101.5, 101.3))
    prm = rmcl_b200.PFParams.defaults()
    out = _update(up, P, A, Tsb, B, prm)
    assert out.tobytes() == R.pf_update(g, index, bricks, P, A, Tsb, B, prm).tobytes()
    q = R.beam_points64(P, Tsb, B)
    e = np.where(np.isfinite(q).all(2), float(np.float32(trunc)), np.inf)
    _check_update64(out, A, e, prm)


# ---------------------------------------------------------------- 3. lookup at cell, brick and box faces -----------------------------
_BOX0 = {}


def _box0():
    """indoor(2000) over an explicit box with origin (0, 0, 0): 50 x 33 x 13 cells"""
    if not _BOX0:
        from rmcl_b200 import synth
        V, F = synth.indoor(2000)
        h, trunc, lo, hi = 0.25, 0.5, (0.0, 0.0, 0.0), (12.3, 8.1, 3.05)
        m = _map(V, F, 1)
        f = _field(m, h, trunc, lo, hi)
        g = _grid(V, h, trunc, np.float32(lo), np.float32(hi))
        index, bricks = f.download()
        _BOX0.update(V=V, F=F, m=m, f=f, g=g, index=index, bricks=bricks)
    return _BOX0


def _edge_points(g, n, seed):
    """n points: first the special ones (origin, -0.0, one ulp outside, the far face, non-finite, huge), then points with coordinates on
    nodes (g an integer), brick faces (a multiple of 8), the far face (dims - 1) and random, in the box and a cell beyond it"""
    rng = np.random.default_rng(seed)
    lo = g.lo
    h = np.float32(g.h)
    dims = np.array(g.dims)
    top = lo + (dims - 1).astype(np.float32) * h
    neg0 = np.where(lo == 0, np.float32(-0.0), lo)
    sp = [lo, neg0, np.nextafter(lo, np.float32(-np.inf)), top, np.nextafter(top, np.float32(np.inf)),
          [lo[0], top[1], lo[2]], [top[0], lo[1], top[2]],
          [np.nan, lo[1], lo[2]], [lo[0], np.inf, lo[2]], [lo[0], lo[1], -np.inf], [np.nan] * 3,
          [1e30, lo[1], lo[2]], [lo[0], -1e30, lo[2]], [3.4e38, 3.4e38, 3.4e38], [-3.4e38, lo[1], lo[2]], [1e-45, 1e-45, 1e-45]]
    for k in range(3):
        for v in (np.nextafter(lo[k], np.float32(-np.inf)), np.nextafter(top[k], np.float32(np.inf)), top[k], -0.0):
            p = (lo + top) / 2
            p[k] = v
            sp.append(p)
    sp = np.asarray(sp, np.float32)
    m = max(n, 0)
    i = rng.integers(0, dims, (m, 3))
    kind = rng.integers(0, 4, (m, 3))
    i = np.where(kind == 1, (i // 8) * 8, i)                                            # brick faces
    i = np.where(kind == 2, dims - 1, i)                                                # far face
    on = lo + i.astype(np.float32) * h
    r = rng.uniform(lo - h, top + h, (m, 3)).astype(np.float32)
    pts = np.where(kind == 3, r, on).astype(np.float32)
    return np.concatenate([sp, pts])[:n]


def _check_lookup(f, g, index, bricks, pts, device, ref=None):
    import torch
    if device:
        got = f.query(torch.from_numpy(pts).cuda()).cpu().numpy()
    else:
        got = f.query(pts)
    assert got.shape == (len(pts),) and got.dtype == np.float32
    assert got.tobytes() == R.lookup(g, index, bricks, pts).tobytes()
    if not len(pts):
        return
    want = R.lookup64(g, index, bricks, pts)
    fin = np.isfinite(pts).all(1)
    assert np.isposinf(got[~fin]).all()
    assert np.abs(got[fin].astype(np.float64) - want[fin]).max() <= 8 * float(np.spacing(np.float32(g.trunc)))
    if ref is not None:
        with np.errstate(over="ignore", invalid="ignore"):
            G = (pts - g.lo) * np.float32(g.inv_h)
        inside = fin & (G >= 0).all(1) & (G <= (np.array(g.dims) - 1).astype(np.float32)).all(1)
        k = np.flatnonzero(inside)[:100_000]
        d = ref.dist(pts[k]).astype(np.float64)
        eps = 1e-5 * (1.0 + float(np.abs(pts[k]).max()))
        err = np.abs(got[k].astype(np.float64) - np.minimum(d, g.trunc))
        assert err.max() <= C_HALF_SQRT3 * g.h + eps, err.max()


@pytest.mark.parametrize("device", [False, True], ids=["host_points", "device_points"])
@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 1_000_003])
def test_lookup_at_faces(n, device):
    B = _box0()
    g = B["g"]
    assert g.lo.tolist() == [0.0, 0.0, 0.0] and all(d % 8 != 1 for d in g.dims)
    _check_lookup(B["f"], g, B["index"], B["bricks"], _edge_points(g, n, n), device)


@pytest.mark.parametrize("device", [False, True], ids=["host_points", "device_points"])
@pytest.mark.parametrize("n", [257, 1_000_003])
def test_lookup_on_the_large_map(n, device):
    L = _large()
    if "index" not in L:
        L["index"], L["bricks"] = L["fields"][1].download()
    _check_lookup(L["fields"][1], L["g"], L["index"], L["bricks"], _edge_points(L["g"], n, n + 1), device, ref=L["ref"])


# ---------------------------------------------------------------- 4. the field update's tile ------------------------------------------
def _smem_optin(m):
    """the dynamic shared memory a PF handle grants one block: the device's opt-in limit less 1024 bytes, as the ray-cast update reports it
    (b2_pf_debug_launch_geometry word 0)"""
    import ctypes as C
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    up = rmcl_b200.PCDSensorUpdaterB200(m)
    P, A, B, Tsb = _pf_case(1, 1, 0)
    Pd, Ad = _dev(P, A)
    up.update(Pd, Ad, Tsb, B)
    geom = np.zeros(12, np.uint32)
    assert rmcl_b200.load_library().b2_pf_debug_launch_geometry(up._h, C.c_void_p(geom.ctypes.data)) == 0
    assert int(geom[0]) == torch.cuda.get_device_properties(0).shared_memory_per_block_optin - 1024
    return int(geom[0])


def _ppb(n_beams, optin):
    """pf_prepare_beams: min(smem_optin / (4 n_beams), 64, ceil(1024 / n_beams)), at least 1"""
    return max(1, min(optin // (4 * n_beams), 64, -(-1024 // n_beams)))


def _pf_case(n, n_beams, seed, centre=(6.0, 4.0, 1.5)):
    from rmcl_b200 import synth
    rng = np.random.default_rng(seed)
    P = synth.transforms(n)
    P["t"] = (np.asarray(centre) + rng.uniform((-5.5, -3.5, -1.3), (5.5, 3.5, 1.3), (n, 3))).astype(np.float32)
    yaw = rng.uniform(-np.pi, np.pi, n)
    P["R"][:, 2], P["R"][:, 3] = np.sin(yaw / 2), np.cos(yaw / 2)
    A = np.zeros(n, synth.PARTICLE_ATTR_DTYPE)
    A["likelihood"]["mean"] = rng.uniform(0, 0.2, n).astype(np.float32)
    A["likelihood"]["sigma"] = rng.uniform(0, 0.01, n).astype(np.float32)
    A["likelihood"]["n_meas"] = rng.choice([0, 3, 9999, 10000], n)
    B = np.zeros(n_beams, synth.RANGE_MEAS_DTYPE)
    d = rng.normal(size=(n_beams, 3))
    B["dir"] = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    B["range"] = rng.uniform(0.1, 9.0, n_beams).astype(np.float32)
    B["orig"] = rng.normal(0, 0.05, (n_beams, 3)).astype(np.float32)
    if n_beams > 3:
        B["range"][1] = np.nan
        B["range"][2] = np.inf
    return P, A, B, synth.scenario_tsb()


def _dev(P, A):
    import torch
    return (torch.from_numpy(np.ascontiguousarray(P).view(np.float32).reshape(-1, 8).copy()).cuda(),
            torch.from_numpy(np.ascontiguousarray(A).view(np.float32).reshape(-1, 9).copy()).cuda())


def _update(up, P, A, Tsb, B, prm):
    from rmcl_b200 import synth
    Pd, Ad = _dev(P, A)
    up.update(Pd, Ad, Tsb, B, prm)
    return Ad.cpu().numpy().reshape(-1).view(synth.PARTICLE_ATTR_DTYPE)


def _check_update64(out, A, e, prm):
    ev = R.evaluate64(e, prm.dist_sigma)
    mean, sig, nm = R.merge64(A, ev)
    assert np.array_equal(out["likelihood"]["n_meas"], nm)
    M = max(float(ev.max(initial=0.0)), float(ev.max(initial=0.0)) ** 2, float(A["likelihood"]["mean"].max()), float(A["likelihood"]["sigma"].max()))
    tol = 2e-6 + 5 * e.shape[1] * 2.0 ** -24 * M
    assert np.abs(out["likelihood"]["mean"] - mean).max() <= tol
    assert np.abs(out["likelihood"]["sigma"] - sig).max() <= tol


# beam counts around ppb's transitions: the cap of 64 (ceil(1024 / n) = 64 at 16), 3 -> 2 particles per block at 511 / 512, 2 -> 1 at
# 1023 / 1024, and
# "max" = smem_optin / 4, the largest count that fits with ppb 1
TILE_BEAMS = [1, 15, 16, 17, 63, 64, 65, 511, 512, 513, 1023, 1024, 1025, "max"]


@pytest.mark.parametrize("n_beams", TILE_BEAMS)
def test_update_tile(n_beams):
    import rmcl_b200
    B0 = _box0()
    optin = _smem_optin(B0["m"])
    nb = optin // 4 if n_beams == "max" else n_beams
    ppb = _ppb(nb, optin)
    if n_beams == "max":
        assert ppb == 1 and 4 * nb <= optin < 4 * (nb + 1)
    up = rmcl_b200.PCDSensorUpdaterB200(B0["m"])
    up.setDistanceField(B0["f"])
    prm = rmcl_b200.PFParams.defaults()
    g, index, bricks = B0["g"], B0["index"], B0["bricks"]
    counts = [3, 2] if ppb == 1 else [ppb - 1, 3 * ppb + 1, 37 * ppb + ppb // 2 + 1]
    for n in counts:
        P, A, B, Tsb = _pf_case(n, nb, 1000 * nb + n)
        out = _update(up, P, A, Tsb, B, prm)
        assert out.tobytes() == R.pf_update(g, index, bricks, P, A, Tsb, B, prm).tobytes(), (nb, n)
        q = R.beam_points64(P, Tsb, B)
        e = R.lookup64(g, index, bricks, q.reshape(-1, 3).astype(np.float32)).reshape(q.shape[:2])
        _check_update64(out, A, e, prm)
    print(f"beams {nb}: ppb {ppb}, particles {counts}")


def test_update_refuses_one_beam_more_than_fits():
    import rmcl_b200
    from rmcl_b200 import synth
    B0 = _box0()
    optin = _smem_optin(B0["m"])
    up = rmcl_b200.PCDSensorUpdaterB200(B0["m"])
    up.setDistanceField(B0["f"])
    P, A, B, Tsb = _pf_case(5, optin // 4 + 1, 9)
    Pd, Ad = _dev(P, A)
    k0 = rmcl_b200.kernel_launch_count()
    with pytest.raises(rmcl_b200.B2Error):
        up.update(Pd, Ad, Tsb, B)
    assert rmcl_b200.kernel_launch_count() == k0
    assert Ad.cpu().numpy().reshape(-1).view(synth.PARTICLE_ATTR_DTYPE).tobytes() == A.tobytes()


def test_stein_beam_limit():
    """Stein's score tile needs 3 * 4 * n_beams bytes per particle: smem_optin / 12 beams run and equal the host-compiled product, one
    more is refused before anything is launched or moved"""
    import rmcl_b200
    import pf_stein_ref as S
    from rmcl_b200 import synth
    B0 = _box0()
    optin = _smem_optin(B0["m"])
    up = rmcl_b200.PCDSensorUpdaterB200(B0["m"])
    up.setDistanceField(B0["f"])
    prm = rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.2
    cfg = rmcl_b200.SteinConfig.defaults()
    cfg.iterations, cfg.n_ref = 1, 0
    nb = optin // 12
    P, A, B, Tsb = _pf_case(5, nb + 1, 12)
    Pd = _dev(P, A)[0]
    k0 = rmcl_b200.kernel_launch_count()
    with pytest.raises(rmcl_b200.B2Error):
        up.steinUpdate(Pd, Tsb, B, cfg, prm, seed=3)
    assert rmcl_b200.kernel_launch_count() == k0 and Pd.cpu().numpy().reshape(-1).view(synth.TRANSFORM_DTYPE).tobytes() == P.tobytes()
    res = up.steinUpdate(Pd, Tsb, B[:nb], cfg, prm, seed=3)
    assert rmcl_b200.kernel_launch_count() == k0 + 3
    want, rec = S.Scene(B0["V"], B0["F"]).update(B0["g"], B0["index"], B0["bricks"], P, Tsb, B[:nb], 0.2, cfg, 3, 0)
    assert Pd.cpu().numpy().reshape(-1).view(synth.TRANSFORM_DTYPE).tobytes() == want.tobytes()
    assert (res["n_ref"], res["n_blocked"]) == (rec.n_ref, rec.n_blocked)
    print(f"Stein: {nb} beams accepted, {nb + 1} refused (smem_optin {optin})")
