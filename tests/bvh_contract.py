"""The layout contract of the map's 8-wide BVH (rmcl_b200/csrc/bvh8.h), checked in plain numpy on a blob as Map.export_blob writes it:
a 64-byte B2BlobHeader, n_nodes nodes of 224 B, n_tris leaf triangle records of 48 B.

The traversal (trace.cuh) reads the tree through every clause checked here: a node's inner children form one run from child_base and slot s
is child_base + popc(imask & ((1 << s) - 1)); a leaf slot's records are found the same way through trimask; empty slots are (+inf, -inf)
and never hit; a child box is the exact float AABB of the triangles below it, so the box test can only cull what a ray cannot hit; at
most 3 triangles per leaf slot (the meta byte cannot say more); at most B2_TRAVERSAL_STACK - 4 levels.  check() names the node, slot or
record and the clause that broke.  canonical() gives the tree independently of where the builder allocated nodes and records."""
import numpy as np

HEADER = np.dtype([("magic", "S8"), ("version", "<u4"), ("node_bytes", "<u4"), ("tri_bytes", "<u4"), ("n_nodes", "<u4"), ("n_tris", "<u4"),
                   ("n_faces", "<u4"), ("n_verts", "<u4"), ("max_depth", "<u4"), ("build_mode", "<i4"), ("abs_max", "<f4", 3), ("sah", "<f4"),
                   ("pad", "<u4")])
NODE = np.dtype([("lo", "<f4", (3, 8)), ("hi", "<f4", (3, 8)), ("child_base", "<u4"), ("tri_base", "<u4"), ("masks", "<u4"), ("pad0", "<u4"),
                 ("meta", "u1", 8), ("pad", "<u4", 2)])
TRI = np.dtype([("v0", "<f4", 3), ("face", "<u4"), ("v1", "<f4", 3), ("pad1", "<u4"), ("v2", "<f4", 3), ("pad2", "<u4")])
assert HEADER.itemsize == 64 and NODE.itemsize == 224 and TRI.itemsize == 48

TRAVERSAL_STACK = 40
MAX_DEPTH = TRAVERSAL_STACK - 4
POS_INF, NEG_INF = 0x7F800000, 0xFF800000
SLOTS = np.arange(8)


def parse(blob):
    """-> (header record, nodes, records) as structured arrays (views of the blob)"""
    blob = np.ascontiguousarray(blob, np.uint8)
    assert blob.size >= 64, "blob shorter than its header"
    hd = blob[:64].view(HEADER)[0]
    assert hd["magic"] == b"B2BVH8F" and hd["version"] == 2 and hd["node_bytes"] == 224 and hd["tri_bytes"] == 48, ("header", hd)
    nn, nt = int(hd["n_nodes"]), int(hd["n_tris"])
    assert blob.size == 64 + 224 * nn + 48 * nt, ("blob size", blob.size, nn, nt)
    nodes = blob[64:64 + 224 * nn].view(NODE)
    tris = blob[64 + 224 * nn:].view(TRI)
    return hd, nodes, tris


def _require(ok, clause, what="node"):
    """ok: bool array over nodes (N,) or (node, slot) (N, 8), or over records / faces (what names the index)"""
    ok = np.asarray(ok, bool)
    if ok.all():
        return
    bad = np.argwhere(~ok)
    f = bad[0]
    where = f"node {f[0]} slot {f[1]}" if ok.ndim == 2 else f"{what} {f[0]}"
    raise AssertionError(f"BVH contract: {clause}: {len(bad)} violation(s), first at {where}")


def _counts(meta):
    """triangles of each leaf slot from its unary count (0 for empty and inner slots)"""
    u = meta >> 5
    return np.where(u == 7, 3, np.where(u == 3, 2, np.where(u == 1, 1, 0)))


def check(blob, V, F, info=None):
    """Assert every clause of the layout contract for the tree in `blob`, built over float32 vertices V (nv, 3) and faces F (nf, 3).
    info: Map.info() of the map the blob came from (n_nodes, n_leaf_tris, max_depth and bvh_bytes must agree).  -> dict of sizes."""
    V = np.ascontiguousarray(V, np.float32).reshape(-1, 3)
    F = np.ascontiguousarray(F, np.int64).reshape(-1, 3)
    hd, nodes, tris = parse(blob)
    N, T = len(nodes), len(tris)
    assert N >= 1, "no root node"
    meta = nodes["meta"].astype(np.uint32)                                        # (N, 8)
    masks = nodes["masks"].astype(np.uint32)
    imask, trimask = masks & 0xFF, masks >> 8
    empty = meta == 0
    inner = ((imask[:, None] >> SLOTS) & 1) == 1
    leaf = ~empty & ~inner

    # ---- encoding
    marker = ((meta & 0x18) == 0x18) & ((meta >> 5) == 1)
    want = np.zeros(N, np.uint32)
    for s in range(8):
        want |= np.where(empty[:, s], 0, np.where(marker[:, s], np.uint32(1 << s), (meta[:, s] >> 5) << np.uint32(8 + 3 * s))).astype(np.uint32)
    _require(masks == want, "masks != b2_masks_from_meta(meta)")
    lob, hib = nodes["lo"].view(np.uint32), nodes["hi"].view(np.uint32)         # (N, 3, 8)
    _require(~empty | ((lob == POS_INF).all(1) & (hib == NEG_INF).all(1)), "an empty slot's box is not (+inf, -inf) on every axis")
    _require(~inner | (meta == (0x20 | (24 + SLOTS))), "an inner slot's meta is not 0x20 | (24 + s)")
    unary = meta >> 5
    _require(~leaf | (unary == 1) | (unary == 3) | (unary == 7), "a leaf slot's unary count is not 1, 3 or 7")
    cnt = np.where(leaf, _counts(meta), 0)
    off_want = np.cumsum(cnt, 1) - cnt                                            # popc(trimask & ((1 << 3s) - 1)) for a consistent trimask
    _require(~leaf | ((meta & 0x1F) == off_want), "a leaf slot's offset is not the popcount of the trimask bits below 3s")
    _require((nodes["pad0"] == 0) & (nodes["pad"] == 0).all(1), "node padding is not zero")
    _require((tris["pad1"] == 0) & (tris["pad2"] == 0), "record padding is not zero", "record")

    # ---- topology: every node but the root is the child of exactly one slot of an earlier node
    n_inner = inner.sum(1)
    cb = nodes["child_base"].astype(np.int64)
    _require((n_inner == 0) | (cb > np.arange(N)), "child_base is not after the node")
    _require((n_inner == 0) | (cb + n_inner <= N), "inner children run past n_nodes")
    rank = np.cumsum(inner, 1) - inner
    pn, ps = np.nonzero(inner)
    child = cb[pn] + rank[pn, ps]
    refs = np.bincount(child, minlength=N)
    _require(refs[1:] == 1, "a node is not referenced exactly once")
    assert refs[0] == 0, "BVH contract: the root (node 0) is referenced as a child"
    parent = np.full(N, -1, np.int64)
    parent[child] = pn
    pslot = np.full(N, -1, np.int64)
    pslot[child] = ps
    depth = np.zeros(N, np.int64)
    depth[0] = 1
    for _ in range(N + 1):                                                       # parent < child: converges in max_depth rounds
        nd = depth.copy()
        nd[1:] = depth[parent[1:]] + (depth[parent[1:]] > 0)
        if np.array_equal(nd, depth):
            break
        depth = nd
    _require(depth >= 1, "a node is not reached from the root")

    # ---- records
    tb = nodes["tri_base"].astype(np.int64)
    ln, ls = np.nonzero(leaf)
    first = tb[ln] + (meta[ln, ls] & 0x1F)
    c = cnt[ln, ls]
    _require(first + c <= T, "a leaf slot's records run past n_tris", "leaf slot")
    rec = np.repeat(first, c) + (np.arange(c.sum()) - np.repeat(np.cumsum(c) - c, c))
    _require(np.bincount(rec, minlength=T)[:T] == 1, "a record is not referenced exactly once", "record")
    assert T == len(F) == int(hd["n_faces"]), f"BVH contract: n_tris {T}, header n_faces {int(hd['n_faces'])}, mesh faces {len(F)}"
    fid = tris["face"].astype(np.int64)
    _require(fid < len(F), "a record's face id is out of range", "record")
    _require(np.bincount(fid, minlength=len(F))[:len(F)] == 1, "a face does not appear exactly once", "face")
    for j, k in enumerate(("v0", "v1", "v2")):
        _require((tris[k].view(np.uint32) == V[F[fid, j]].view(np.uint32)).all(1), f"a record's {k} is not bit-equal to V[F[face, {j}]]", "record")

    # ---- boxes, exactly: a leaf slot's box is the min / max over its records' vertices
    pts = np.stack([tris["v0"], tris["v1"], tris["v2"]], 1)                       # (T, 3 vertices, 3 axes)
    rlo, rhi = pts.min(1), pts.max(1)
    order = np.argsort(first, kind="stable")                                      # the leaf slots' record runs partition [0, T)
    starts = first[order]
    slo, shi = np.empty((len(first), 3), np.float32), np.empty((len(first), 3), np.float32)
    if len(first):
        slo[order], shi[order] = np.minimum.reduceat(rlo, starts), np.maximum.reduceat(rhi, starts)
    lo, hi = nodes["lo"], nodes["hi"]                                             # (N, 3, 8)
    ok = np.ones((N, 8), bool)
    ok[ln, ls] = (lo[ln, :, ls] == slo).all(1) & (hi[ln, :, ls] == shi).all(1)
    _require(ok, "a leaf slot's box is not the float AABB of its triangles")
    # an inner slot's box is the union of the child node's non-empty slot boxes
    ulo = np.where(empty[:, None, :], np.inf, lo).min(2)                          # (N, 3)
    uhi = np.where(empty[:, None, :], -np.inf, hi).max(2)
    ok = np.ones((N, 8), bool)
    ok[pn, ps] = (lo[pn, :, ps] == ulo[child]).all(1) & (hi[pn, :, ps] == uhi[child]).all(1)
    _require(ok, "an inner slot's box is not the union of its child node's boxes")
    _require(~empty.all(1), "a node has no children")

    # ---- depth and levels
    measured = int(depth.max())
    assert measured == int(hd["max_depth"]), f"BVH contract: measured depth {measured}, header max_depth {int(hd['max_depth'])}"
    assert measured <= MAX_DEPTH, f"BVH contract: depth {measured} exceeds B2_TRAVERSAL_STACK - 4 = {MAX_DEPTH}"
    _require(np.diff(depth) >= 0, "node depth decreases with node index (the level-by-level refit relies on it)")

    # ---- the box test's slack constant covers every referenced vertex
    amax = np.abs(pts).max((0, 1)) if T else np.zeros(3, np.float32)
    for k in range(3):
        assert hd["abs_max"][k] >= amax[k], f"BVH contract: header abs_max[{k}] = {hd['abs_max'][k]!r} below max |coordinate| {amax[k]!r}"

    if info is not None:
        got = (info["n_nodes"], info["n_leaf_tris"], info["max_depth"], info["bvh_bytes"])
        assert got == (N, T, measured, 224 * N + 48 * T), f"BVH contract: info() {got} disagrees with the blob {(N, T, measured, 224 * N + 48 * T)}"
    return dict(n_nodes=N, max_depth=measured, n_tris=T)


def canonical(blob, scale=1.0):
    """The tree as nested tuples keyed by slot, independent of where the builder placed nodes and records: per slot None (empty),
    ("inner", lo, hi, <child node>) or ("leaf", lo, hi, face ids in record order); boxes as float64 times `scale`."""
    hd, nodes, tris = parse(blob)
    N = len(nodes)
    meta = nodes["meta"].astype(np.int64)
    imask = nodes["masks"].astype(np.int64) & 0xFF
    lo = nodes["lo"].astype(np.float64) * scale
    hi = nodes["hi"].astype(np.float64) * scale
    face = tris["face"].astype(np.int64)
    cnt = _counts(meta)
    sub = [None] * N
    for i in range(N - 1, -1, -1):                                               # children have larger indices than their parent
        row, r = [], 0
        for s in range(8):
            m = int(meta[i, s])
            box_lo, box_hi = tuple(lo[i, :, s]), tuple(hi[i, :, s])
            if (imask[i] >> s) & 1:
                row.append(("inner", box_lo, box_hi, sub[int(nodes["child_base"][i]) + r]))
                r += 1
            elif m:
                f0 = int(nodes["tri_base"][i]) + (m & 0x1F)
                row.append(("leaf", box_lo, box_hi, tuple(face[f0:f0 + int(cnt[i, s])])))
            else:
                row.append(None)
        sub[i] = tuple(row)
    return sub[0]


def first_difference(a, b, path="root"):
    """the first slot path at which two canonical trees differ, or None"""
    if a == b:
        return None
    if isinstance(a, tuple) and isinstance(b, tuple) and len(a) == len(b) == 8:
        for s in range(8):
            if a[s] != b[s]:
                x, y = a[s], b[s]
                if x is not None and y is not None and x[0] == y[0] == "inner" and x[1:3] == y[1:3]:
                    return first_difference(x[3], y[3], f"{path}/{s}")
                return f"{path}/{s}: {x if x is None or x[0] == 'leaf' else x[:3]} != {y if y is None or y[0] == 'leaf' else y[:3]}"
    return f"{path}: {a} != {b}"
