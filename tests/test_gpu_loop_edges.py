"""The ICP loop (k_icp_loop), the single reduction (k_p2l_reduce) and the v1 batch path (k_rcc_fused_batch -> k_umeyama_from_partials) at
the edges of their launch geometry, against a float64 restatement of the same operations.

The oracle restates the device's FP32 arithmetic op for op; that pins the per-pair maths but not what exists only on the GPU: how the pairs
are spread over blocks, warps and the three storage tiers of the loop (registers, shared memory, streamed from L2), the fixed-point
exchange of block sums, the block split between sensors.  Here the device's own find output (modelView / datasetView after the call, find
itself is pinned bit-exactly elsewhere) goes through a plain float64 model of MICP-L's correctOnce, at pair counts placed on those
boundaries by the launch shape the library reports (b2_rcc_debug_loop_geometry).

Tolerances (float64 reference vs FP32 device):
  n_meas    exact, provided every pair's float64 gate margin | |sd| - max_dist | exceeds GATE_MARGIN * max_dist in every iteration (asserted
            on each case's own inputs: inside the margin an FP32 rounding may legitimately flip the gate)
  means     TOL_MEAN * (1 + |mean|)
  cov       TOL_COV * (1 + max |C|)
  pose      TOL_POSE on t and on the quaternion up to sign, required only where the merged covariance is well conditioned in every iteration
            (sigma_3 >= COND_MIN * sigma_1); below that the rotation is not unique and only the statistics are compared
Results must be bit-identical across exec-mode-2 reruns and across the three ways a scan reaches the device.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import gpu_map, oracle_scene, quat_close

GATE_MARGIN = 1e-4
TOL_MEAN = 1e-6
TOL_COV = 2e-5
TOL_POSE = 1e-5
COND_MIN = 1e-3
B2_MAX_SENSORS = 4
ICP_BLOCK = 512                # threads per k_icp_loop block
NAME = "building:200000"


# =====================================================================================================================================
# float64 reference (formulas of rmagine's statistics_p2l / CrossStatistics / umeyama_transform and of micp_localization.cpp:915-984)
# =====================================================================================================================================
def tf_mat(T):
    """TRANSFORM_DTYPE record -> 4x4 float64"""
    q = np.asarray(T["R"], np.float64)
    x, y, z, w = q / np.linalg.norm(q)
    M = np.eye(4)
    M[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                 [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                 [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
    M[:3, 3] = np.asarray(T["t"], np.float64)
    return M


def mat_quat(M):
    """rotation part of a 4x4 -> unit quaternion (x, y, z, w), float64"""
    R = M[:3, :3]
    K = np.array([[R[0, 0] - R[1, 1] - R[2, 2], R[1, 0] + R[0, 1], R[2, 0] + R[0, 2], R[2, 1] - R[1, 2]],
                  [R[1, 0] + R[0, 1], R[1, 1] - R[0, 0] - R[2, 2], R[2, 1] + R[1, 2], R[0, 2] - R[2, 0]],
                  [R[2, 0] + R[0, 2], R[2, 1] + R[1, 2], R[2, 2] - R[0, 0] - R[1, 1], R[1, 0] - R[0, 1]],
                  [R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1], R[0, 0] + R[1, 1] + R[2, 2]]]) / 3.0
    w, v = np.linalg.eigh(K)
    return v[:, np.argmax(w)]


def stats_identity():
    return dict(n=0, dm=np.zeros(3), mm=np.zeros(3), C=np.zeros((3, 3)))


def p2l_f64(T, D, dmask, I, N, hits, max_dist):
    """statistics_p2l in float64: pairs with both masks set, D' = T D, sd = (I - D') . N, gate |sd| < max_dist, M = D' + N sd.
    -> dict(n, dm, mm, C = sum (M - mm)(D' - dm)^T / n  (C[r, c]), margin = min | |sd| - max_dist | over the pairs that reach the gate)"""
    T = tf_mat(T) if not isinstance(T, np.ndarray) or T.shape != (4, 4) else T
    D, I, N = (np.asarray(a, np.float64).reshape(-1, 3) for a in (D, I, N))
    ok = (np.asarray(dmask).reshape(-1) > 0) & (np.asarray(hits).reshape(-1) > 0)
    Dt = D[ok] @ T[:3, :3].T + T[:3, 3]
    Ip, Np = I[ok], N[ok]
    sd = np.einsum("ij,ij->i", Ip - Dt, Np)
    margin = float(np.abs(np.abs(sd) - max_dist).min()) if len(sd) else np.inf
    g = np.abs(sd) < max_dist
    Dg, Mg = Dt[g], Dt[g] + Np[g] * sd[g][:, None]
    n = int(g.sum())
    if n == 0:
        s = stats_identity()
    else:
        dm, mm = Dg.mean(0), Mg.mean(0)
        s = dict(n=n, dm=dm, mm=mm, C=(Mg - mm).T @ (Dg - dm) / n)
    s["margin"] = margin
    return s


def stats_transform(T, s):
    """T * CrossStatistics: means as points, C -> R C R^T"""
    R, t = T[:3, :3], T[:3, 3]
    return dict(n=s["n"], dm=R @ s["dm"] + t, mm=R @ s["mm"] + t, C=R @ s["C"] @ R.T)


def stats_merge(a, b):
    """pooled first and second moments (CrossStatistics::operator+=)"""
    n = a["n"] + b["n"]
    if n == 0:
        return stats_identity()
    wa, wb = a["n"] / n, b["n"] / n
    dm, mm = wa * a["dm"] + wb * b["dm"], wa * a["mm"] + wb * b["mm"]
    C = wa * (a["C"] + np.outer(a["mm"] - mm, a["dm"] - dm)) + wb * (b["C"] + np.outer(b["mm"] - mm, b["dm"] - dm))
    return dict(n=n, dm=dm, mm=mm, C=C)


def umeyama_f64(s):
    """-> (4x4 transform taking the dataset onto the model, singular values of C); identity for n == 0"""
    T = np.eye(4)
    if s["n"] == 0:
        return T, np.zeros(3)
    U, S, Vt = np.linalg.svd(s["C"])
    Dg = np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt)) or 1.0])
    T[:3, :3] = U @ Dg @ Vt
    T[:3, 3] = s["mm"] - T[:3, :3] @ s["dm"]
    return T, S


def correct_once_f64(sensors, Tom, iterations, cp, weights=None):
    """MICPLocalizationNode::correctOnce after find (micp_localization.cpp:915-984) in float64.  sensors: dicts with Tbo, Tsb, max_dist,
    adaptive_max_dist_min and the device's own buffers D, dmask (datasetView), I, N, hits (modelView).
    -> dict(Tom_new, T_onew_oold (4x4), Cmerged (last iteration), margin (relative, minimum over sensors and iterations), cond (min s3/s1))"""
    weights = [1.0] * len(sensors) if weights is None else weights
    T = np.eye(4)
    margin, cond = np.inf, np.inf
    merged = stats_identity()
    for _ in range(iterations):
        merged, merged_w = stats_identity(), stats_identity()
        for s, w in zip(sensors, weights):
            Tbo, Tsb = tf_mat(s["Tbo"]), tf_mat(s["Tsb"])
            T_bnew_bold = np.linalg.inv(Tbo) @ T @ Tbo                                         # :926
            T_snew_sold = np.linalg.inv(Tsb) @ T_bnew_bold @ Tsb                               # MICPSensor.hpp:178
            md = s["max_dist"] * (1.0 - cp) + s.get("adaptive_max_dist_min", 0.15) * cp           # CorrespondencesCPU.cpp:21-23
            Cs = p2l_f64(T_snew_sold, s["D"], s["dmask"], s["I"], s["N"], s["hits"], md)
            margin = min(margin, Cs["margin"] / md)
            Cs_o = stats_transform(Tbo, stats_transform(Tsb, Cs))                              # :931 (stats_b = Tsb * stats_s)
            Cw = dict(Cs_o, n=int(np.floor(Cs_o["n"] * w)))                                    # :933-934
            merged, merged_w = stats_merge(merged, Cs_o), stats_merge(merged_w, Cw)            # :936-937
        T_inner, S = umeyama_f64(merged_w)                                                     # :952-953
        if merged_w["n"] > 0:                                                                  # (no pairs: the identity, on both sides)
            cond = min(cond, S[2] / S[0] if S[0] > 0 else 0.0)
        T = T @ T_inner                                                                        # :963
    Tom_new = tf_mat(Tom) @ T if merged["n"] > 0 else tf_mat(Tom)                                # :972-984
    return dict(Tom_new=Tom_new, T_onew_oold=T, Cmerged=merged, margin=margin, cond=cond)


def assert_stats(dev, ref, what=""):
    """device CROSS_STATS record (odom / base frame, column-major C) vs a reference dict"""
    assert int(dev["n_meas"]) == ref["n"], (what, int(dev["n_meas"]), ref["n"])
    if ref["n"] == 0:
        return
    for k, r in (("dataset_mean", ref["dm"]), ("model_mean", ref["mm"])):
        assert np.all(np.abs(np.asarray(dev[k], np.float64) - r) <= TOL_MEAN * (1 + np.abs(r))), (what, k, dev[k], r)
    Cd = np.asarray(dev["covariance"], np.float64).reshape(3, 3).T                             # [c*3 + r] -> C[r, c]
    assert np.abs(Cd - ref["C"]).max() <= TOL_COV * (1 + np.abs(ref["C"]).max()), (what, Cd, ref["C"])


def assert_pose(dev, M, what=""):
    assert np.abs(np.asarray(dev["t"], np.float64) - M[:3, 3]).max() <= TOL_POSE, (what, dev["t"], M[:3, 3])
    assert quat_close(dev["R"], mat_quat(M), TOL_POSE), (what, dev["R"], mat_quat(M))


def verify(run, inputs, Tom, what="", weights=None):
    """run(iterations) -> correctOnce result (Tom_new, T_onew_oold, Cmerged_o); inputs() -> its correct_once_f64 sensors.  Five iterations against
    the reference; where the merged covariance is ill-conditioned the rotation is not unique and every later iteration's statistics depend on
    the rotation chosen, so then only the first iteration's statistics (a call with one iteration) are compared."""
    out = run(5)
    ref = correct_once_f64(inputs(), Tom, 5, 0.0, weights)
    assert ref["margin"] > GATE_MARGIN, (what, "the case's own inputs put a pair within the gate margin", ref["margin"])
    if ref["cond"] >= COND_MIN:
        assert_stats(out[2], ref["Cmerged"], what)
        assert_pose(out[0], ref["Tom_new"], what)
        assert_pose(out[1], ref["T_onew_oold"], what)
    else:
        ref1 = correct_once_f64(inputs(), Tom, 1, 0.0, weights)
        assert ref1["margin"] > GATE_MARGIN, what
        assert_stats(run(1)[2], ref1["Cmerged"], what + " (first iteration)")
    return out


def device_inputs(h, Tbo, Tsb, max_dist=1.0, amin=0.15):
    """the handle's buffers after its last find, as a correct_once_f64 sensor"""
    mv, ds = h.modelView(), h.datasetView()
    return dict(Tbo=Tbo, Tsb=Tsb, max_dist=max_dist, adaptive_max_dist_min=amin, D=ds["points"], dmask=ds["mask"], I=mv["points"], N=mv["normals"],
                hits=mv["hits"])


# =====================================================================================================================================
# scene: map-surface points and scan rays of one oracle scan in the building, seen from a pose guess off by a known small offset
# =====================================================================================================================================
_SCENE = {}


def scene(po, synth, n_min):
    """Scan of the building from the ground-truth pose with >= n_min valid points, and a pose guess a few centimetres / tenths of a degree off.
    rays (dirs) are the scan's rays whose first-pass plane distance at the guess is below 0.4 m (or that have no pair at all), so that the
    gate margin holds through the iterations for ray-casting handles built from any prefix of them."""
    key = "scan"
    if key in _SCENE and _SCENE[key]["n_valid"] >= n_min:
        return _SCENE[key]
    osc = oracle_scene(NAME)
    cols = 2048
    rows = max(64, int(np.ceil(1.35 * n_min / cols)))
    m = synth.SphericalModel(np.radians(-35.0), np.radians(60.0) / (rows - 1), rows, -np.pi, 2 * np.pi / cols, cols, 0.5, 120.0)
    o, d = po.model_rays(m)
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    Tbo = synth.make_transform((0.05, 0.02, 0.0), (0, 0, 0.1))
    offset = synth.make_transform((0.03, -0.02, 0.01), (0.0, 0.0, np.radians(0.3)))
    Tom = synth.compose(synth.compose(Tgt, offset), synth.inverse(Tbo))
    ranges = synth.noisy_ranges(osc.simulate(Tgt, Tsb, o, d, m.range_max)["ranges"], m.range_max, seed=11)
    dp, dmk, nv = po.dataset_from_ranges(o, d, ranges, m.range_min, m.range_max)
    assert nv >= n_min, (nv, n_min)
    rng = np.random.default_rng(4)
    pts = dp[dmk > 0][rng.permutation(nv)]                                        # map-surface points (sensor frame, with noise)
    sim = osc.simulate(synth.compose(Tom, Tbo), Tsb, o, d, m.range_max)           # what find sees from the guess
    sd = np.einsum("ij,ij->i", sim["points"].astype(np.float64) - dp, sim["normals"].astype(np.float64))
    keep = (dmk == 0) | (sim["hits"] == 0) | (np.abs(sd) < 0.4)
    perm = rng.permutation(int(keep.sum()))
    _SCENE[key] = dict(osc=osc, Tsb=Tsb, Tbo=Tbo, Tom=Tom, Tgt=Tgt, pts=pts, n_valid=nv, dirs=d[keep][perm], ranges=ranges[keep][perm],
                       range_min=m.range_min, range_max=m.range_max)
    return _SCENE[key]


# =====================================================================================================================================
# launch shape
# =====================================================================================================================================
def geometry(h):
    import rmcl_b200
    out = np.zeros(4 + 4 * B2_MAX_SENSORS, np.uint32)
    assert rmcl_b200.load_library().b2_rcc_debug_loop_geometry(h._h, C.c_void_p(out.ctypes.data)) == 0
    ns = int(out[2])
    sensors = [dict(zip(("n", "blk0", "nblk", "smem_u"), map(int, out[4 + 4 * k: 8 + 4 * k]))) for k in range(ns)]
    return dict(G=int(out[0]), cap=int(out[1]), ns=ns, grid=int(out[3]), sensors=sensors)


def tier(s):
    """storage tier of a sensor's pairs: 'reg' (<= 2 per thread), 'smem' (the rest fits in shared memory), 'stream' (beyond: read from L2)"""
    stride = s["nblk"] * ICP_BLOCK
    per_thread = -(-s["n"] // stride)
    if per_thread <= 2:
        assert s["smem_u"] == 0
        return "reg"
    return "smem" if per_thread == 2 + s["smem_u"] else "stream"


def limits(h):
    g = geometry(h)
    assert g["G"] >= 1 and g["cap"] >= 1, g
    R = ICP_BLOCK * g["G"]
    return g["G"], g["cap"], R


def _cpc(synth, sc, pts, mask=None):
    import rmcl_b200
    h = rmcl_b200.CPCB200(gpu_map(NAME))
    h.setTsb(sc["Tsb"]); h.setParams(1.0, 0.15)
    h.setDataset(pts, mask)
    return h


def _o1dn(synth, sc, n):
    import rmcl_b200
    h = rmcl_b200.RCCB200O1Dn(gpu_map(NAME))
    h.setTsb(sc["Tsb"]); h.setParams(1.0, 0.15)
    h.setModel(synth.O1DnModel(n, 1, np.zeros(3, np.float32), sc["dirs"][:n].copy(), sc["range_min"], sc["range_max"]))
    return h


def _sweep(G, cap, R):
    return [1, 2, 31, 32, 33, 255, 256, 257, 511, 512, 513, 2 * R - 1, 2 * R, 2 * R + 1, (2 + cap) * R - 1, (2 + cap) * R, (2 + cap) * R + 1]


def _expected_tier(n, cap, R):
    return "reg" if n <= 2 * R else ("smem" if n <= (2 + cap) * R else "stream")


# =====================================================================================================================================
# tests
# =====================================================================================================================================
def test_f64_reference_against_oracle(po, synth):
    """The float64 reference itself, against the oracle's correctOnce with FP64 sums (single ray-casting sensor and a ray-casting +
    closest-point pair): runs without a GPU, so the yardstick of the GPU tests below is checked rather than assumed."""
    name = "building:60000"
    osc = oracle_scene(name)
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 256, 256, 0.5, 120.0)
    o, d = po.model_rays(m)
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    ranges = synth.noisy_ranges(osc.simulate(Tgt, Tsb, o, d, m.range_max)["ranges"], m.range_max, seed=21)
    dp, dm, _ = po.dataset_from_ranges(o, d, ranges, m.range_min, m.range_max)
    Tbo = synth.make_transform((0.05, 0.02, 0.0), (0, 0, 0.1))
    Tom = synth.compose(synth.compose(Tgt, synth.make_transform((0.04, -0.03, 0.02), (0, 0, np.radians(0.5)))), synth.inverse(Tbo))
    sim = osc.simulate(synth.compose(Tom, Tbo), Tsb, o, d, m.range_max)
    rcc = dict(Tbo=Tbo, Tsb=Tsb, max_dist=1.0, adaptive_max_dist_min=0.15, D=dp, dmask=dm, I=sim["points"], N=sim["normals"], hits=sim["hits"])
    for cp in (0.0, 0.5):
        ref = correct_once_f64([rcc], Tom, 5, cp)
        orc = osc.micp_correct_once(o, d, m.range_max, dp, dm, Tom, Tbo, Tsb, 5, 1.0, 0.15, cp, f64_accum=True)
        assert ref["Cmerged"]["n"] >= 5000 and ref["cond"] >= COND_MIN
        assert abs(int(orc[2]["n_meas"]) - ref["Cmerged"]["n"]) <= 2
        for dev, M in ((orc[0], ref["Tom_new"]), (orc[1], ref["T_onew_oold"])):
            assert np.abs(np.asarray(dev["t"], np.float64) - M[:3, 3]).max() <= 2e-6 and quat_close(dev["R"], mat_quat(M), 2e-6)
    # a closest-point sensor (other mounting, merge weight 0.5) next to the ray-casting one
    Tbo2 = synth.make_transform((-0.1, 0.05, 0.1), (0, 0, -0.2))
    pts = dp[dm > 0][::2].copy()
    cpc = osc.cpc_find(synth.compose(Tom, Tbo2), Tsb, pts, 1.0)
    s2 = dict(Tbo=Tbo2, Tsb=Tsb, max_dist=1.0, adaptive_max_dist_min=0.15, D=pts, dmask=np.ones(len(pts), np.uint8), I=cpc["points"], N=cpc["normals"],
              hits=cpc["hits"])
    ref = correct_once_f64([rcc, s2], Tom, 5, 0.0, weights=[1.0, 0.5])
    orc = osc.micp_correct_once_multi([dict(origs=o, dirs=d, range_max=m.range_max, dataset_points=dp, dataset_mask=dm, Tbo=Tbo, Tsb=Tsb, weight=1.0),
                                       dict(dirs=None, dataset_points=pts, dataset_mask=np.ones(len(pts), np.uint8), Tbo=Tbo2, Tsb=Tsb, weight=0.5)],
                                      Tom, 5, 0.0, f64_accum=True)
    assert abs(int(orc[2]["n_meas"]) - ref["Cmerged"]["n"]) <= 2
    assert np.abs(np.asarray(orc[0]["t"], np.float64) - ref["Tom_new"][:3, 3]).max() <= 2e-6 and quat_close(orc[0]["R"], mat_quat(ref["Tom_new"]), 2e-6)
    # the single-reduction statistics as well (the oracle's FP64-sum statistics_p2l)
    T = synth.make_transform((0.01, -0.02, 0.005), (0.001, 0.0, 0.003))
    st = po.statistics_p2l(T, dp, dm, sim["points"], sim["normals"], sim["hits"], 1.0, f64=True)
    assert_stats(st, p2l_f64(T, dp, dm, sim["points"], sim["normals"], sim["hits"], 1.0))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [2, 1, 0])
def test_loop_single_sensor_sweep(po, synth, mode):
    """One closest-point sensor with n pairs at every block / warp / storage-tier boundary of k_icp_loop (exec modes 2 and 1) and at the same
    counts through the multi-launch chain (mode 0)."""
    probe = _cpc(synth, {"Tsb": synth.scenario_tsb()}, np.zeros((1, 3), np.float32))
    G, cap, R = limits(probe)
    counts = _sweep(G, cap, R)
    sc = scene(po, synth, counts[-1])
    h = _cpc(synth, sc, sc["pts"][:1])
    h.setExecMode(mode)
    for n in counts:
        h.setDataset(sc["pts"][:n])
        out = verify(lambda it: h.correctOnce(sc["Tom"], sc["Tbo"], it, 0.0), lambda: [device_inputs(h, sc["Tbo"], sc["Tsb"])], sc["Tom"], f"mode {mode} n {n}")
        if mode != 0:
            g = geometry(h)
            assert g["ns"] == 1 and g["sensors"][0]["n"] == n and g["grid"] == min(G, -(-n // ICP_BLOCK)), (n, g)
            assert tier(g["sensors"][0]) == _expected_tier(n, cap, R), (n, g)
        if mode == 2:
            again = h.correctOnce(sc["Tom"], sc["Tbo"], 5, 0.0)
            assert again[0].tobytes() == out[0].tobytes() and again[2].tobytes() == out[2].tobytes(), n


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [2, 1])
def test_loop_ray_casting_sweep_and_scan_sources(po, synth, mode):
    """Ray-casting sensors (O1Dn of width n) at the small counts and on both sides of the end of the shared-memory tier, with the scan resident,
    passed as a pageable host array and as a pinned host tensor (the loop then unpacks it itself, up to (2 + cap) R pairs): bit-identical."""
    import torch
    probe = _cpc(synth, {"Tsb": synth.scenario_tsb()}, np.zeros((1, 3), np.float32))
    G, cap, R = limits(probe)
    counts = [1, 2, 31, 32, 33, 255, 256, 257, 511, 512, 513, (2 + cap) * R, (2 + cap) * R + 1]
    sc = scene(po, synth, counts[-1])
    assert len(sc["dirs"]) >= counts[-1]
    for n in counts:
        h = _o1dn(synth, sc, n)
        h.setExecMode(mode)
        ranges = sc["ranges"][:n].copy()
        h.setRanges(ranges)
        outs = [verify(lambda it: h.correctOnce(sc["Tom"], sc["Tbo"], it, 0.0), lambda: [device_inputs(h, sc["Tbo"], sc["Tsb"])], sc["Tom"], f"mode {mode} n {n}")]
        assert tier(geometry(h)["sensors"][0]) == _expected_tier(n, cap, R), n
        outs.append(h.correctOnce(sc["Tom"], sc["Tbo"], 5, 0.0, ranges=ranges))
        h.setRanges(np.full_like(ranges, 3.0))                                   # scramble the resident scan: the pinned call must rebuild it
        outs.append(h.correctOnce(sc["Tom"], sc["Tbo"], 5, 0.0, ranges=torch.from_numpy(ranges.copy()).pin_memory()))
        for k, o in enumerate(outs[1:]):
            assert o[0].tobytes() == outs[0][0].tobytes() and o[2].tobytes() == outs[0][2].tobytes(), (n, k)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [2, 1])
def test_loop_masks(po, synth, mode):
    """All pairs masked but one, and NaN dataset points under the mask, in the shared-memory tier and in the streamed tier."""
    probe = _cpc(synth, {"Tsb": synth.scenario_tsb()}, np.zeros((1, 3), np.float32))
    G, cap, R = limits(probe)
    sc = scene(po, synth, (2 + cap) * R + 1)
    rng = np.random.default_rng(8)
    for n in (2 * R + 1, (2 + cap) * R + 1):
        h = _o1dn(synth, sc, n)
        h.setExecMode(mode)
        pts, vm, _ = po.dataset_from_ranges(np.zeros((1, 3), np.float32), sc["dirs"][:n], sc["ranges"][:n], sc["range_min"], sc["range_max"])
        h.find(synth.compose(sc["Tom"], sc["Tbo"]))
        one = int(np.flatnonzero((h.modelView()["hits"] > 0) & (vm > 0))[-1])      # the last pair with a partner: in the last tier of this n
        for case in ("one", "nan"):
            mask = np.zeros(n, np.uint8)
            if case == "one":
                mask[one] = 1
            else:
                mask[:] = (rng.random(n) < 0.5) & (vm > 0)
            p = pts.copy()
            p[mask == 0] = np.nan
            h.setDataset(p, mask)
            out = verify(lambda it: h.correctOnce(sc["Tom"], sc["Tbo"], it, 0.0), lambda: [device_inputs(h, sc["Tbo"], sc["Tsb"])], sc["Tom"], f"{case} n {n}")
            if case == "one":
                assert int(out[2]["n_meas"]) == 1
            else:
                assert np.isfinite(out[0]["t"]).all() and int(out[2]["n_meas"]) > n // 3


@pytest.mark.gpu
def test_cross_statistics_reduction_edges(po, synth):
    """computeCrossStatistics (k_p2l_reduce: per-block partials, the last block to finish sums them) at block and grid boundaries, and on an
    empty dataset (no pairs: n_meas 0, like the reference's reduction over nothing)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sc = scene(po, synth, 256 * sms + 1)
    h = _cpc(synth, sc, sc["pts"][:1])
    T = synth.make_transform((0.02, -0.01, 0.005), (0.001, -0.002, 0.004))
    Tbm = synth.compose(sc["Tom"], sc["Tbo"])
    for n in (1, 255, 256, 257, 256 * sms - 1, 256 * sms, 256 * sms + 1):
        h.setDataset(sc["pts"][:n])
        h.find(Tbm)
        st = h.computeCrossStatistics(T, 0.0)
        s = device_inputs(h, sc["Tbo"], sc["Tsb"])
        ref = p2l_f64(T, s["D"], s["dmask"], s["I"], s["N"], s["hits"], 1.0)
        assert ref["margin"] > GATE_MARGIN and ref["n"] >= 1
        assert_stats(st, ref, f"n {n}")
    h.setDataset(np.zeros((0, 3), np.float32))
    h.find(Tbm)
    st = h.computeCrossStatistics(T, 0.0)
    assert int(st["n_meas"]) == 0


@pytest.mark.gpu
def test_correct_batch_v1_edges(po, synth):
    """v1 correct(Tbm[N]) (k_rcc_fused_batch -> k_umeyama_from_partials) with O1Dn models around a warp and a block of rays and pose counts
    around the 64-pose blocks of the Umeyama kernel: Ncorr exact, statistics and Tdelta against the float64 reference."""
    sc = scene(po, synth, 1000)
    osc, Tsb = sc["osc"], sc["Tsb"]
    rng = np.random.default_rng(13)
    Tbm0 = synth.compose(sc["Tom"], sc["Tbo"])
    for n in (1, 33, 127, 128, 129):
        h = _o1dn(synth, sc, n)
        h.setInputData(sc["ranges"][:n].copy())
        D, dmask, _ = po.dataset_from_ranges(np.zeros((1, 3), np.float32), sc["dirs"][:n], sc["ranges"][:n], sc["range_min"], sc["range_max"])
        for N in (1, 64, 65):
            T = synth.transforms(N)
            T[:] = Tbm0
            T["t"] += rng.uniform(-0.02, 0.02, (N, 3)).astype(np.float32)
            Td, nc, st = h.correct(T)
            for p in range(N):
                sim = osc.simulate(T[p], Tsb, np.zeros((1, 3), np.float32), sc["dirs"][:n], sc["range_max"])
                s = p2l_f64(np.eye(4), D, dmask, sim["points"], sim["normals"], sim["hits"], 1.0)
                assert s["margin"] > GATE_MARGIN, (n, N, p)
                sb = stats_transform(tf_mat(Tsb), s)
                assert int(nc[p]) == sb["n"], (n, N, p)
                assert_stats(st[p], sb, f"n {n} N {N} pose {p}")
                Tref, S = umeyama_f64(sb)
                if sb["n"] > 0 and S[2] >= COND_MIN * S[0]:
                    assert_pose(Td[p], Tref, f"n {n} N {N} pose {p}")


def _multi(hs, Tbos, Tom, weights=None, iterations=5):
    import rmcl_b200
    return rmcl_b200.micp_correct_once(hs, np.stack(Tbos), Tom, iterations, 0.0, merge_weights=weights)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [2, 1])
def test_loop_multi_sensor_edges(po, synth, mode):
    """Several sensors in one k_icp_loop: four (B2_MAX_SENSORS) mixing ray casting and closest points, a fifth refused, strongly skewed pair
    counts (every sensor keeps at least one block, the blocks add up to the grid), merge weight 0 on one and on all sensors."""
    import rmcl_b200
    probe = _cpc(synth, {"Tsb": synth.scenario_tsb()}, np.zeros((1, 3), np.float32))
    G, cap, R = limits(probe)
    sc = scene(po, synth, 300000)
    Tom, Tbo, Tsb = sc["Tom"], sc["Tbo"], sc["Tsb"]
    Tbo2 = synth.compose(Tbo, synth.make_transform((0.02, -0.01, 0.0), (0, 0, 0.002)))

    def run(hs, Tbos, weights=None, what=""):
        for h in hs:
            h.setExecMode(mode)
        out = verify(lambda it: _multi(hs, Tbos, Tom, weights, it), lambda: [device_inputs(h, b, Tsb) for h, b in zip(hs, Tbos)], Tom, what, weights)
        g = geometry(hs[0])
        assert g["ns"] == len(hs) and sum(s["nblk"] for s in g["sensors"]) == g["grid"], g
        assert all(s["nblk"] >= 1 for s in g["sensors"] if s["n"] > 0), g
        return out, g

    four = [_o1dn(synth, sc, 20000), _cpc(synth, sc, sc["pts"][:50000]), _o1dn(synth, sc, 3000), _cpc(synth, sc, sc["pts"][50000:150000])]
    Tb4 = [Tbo, Tbo2, Tbo, Tbo2]
    for h, k in zip(four[::2], (20000, 3000)):
        h.setRanges(sc["ranges"][:k].copy())
    run(four, Tb4, [1.0, 0.5, 2.0, 1.0], "four sensors")
    run(four, Tb4, [1.0, 0.0, 1.0, 1.0], "weight 0 on one")
    out, _ = run(four, Tb4, [0.0] * 4, "weight 0 on all")
    assert np.abs(out[1]["t"]).max() == 0.0 and int(out[2]["n_meas"]) > 0            # nothing to fit: T_onew_oold stays the identity
    with pytest.raises(rmcl_b200.B2Error):
        _multi(four + [_cpc(synth, sc, sc["pts"][:100])], Tb4 + [Tbo2], Tom)
    # skewed: 1 pair next to ~300 000, 33 next to 2R + 1 (the big one is in the shared-memory tier, the small one in one block)
    for small, big in ((1, 300000), (33, 2 * R + 1)):
        hs = [_cpc(synth, sc, sc["pts"][-small:]), _cpc(synth, sc, sc["pts"][:big])]
        for order in (hs, hs[::-1]):
            _, g = run(order, [Tbo2, Tbo], None, f"skewed {small}/{big}")
            assert g["grid"] == G and min(s["nblk"] for s in g["sensors"]) == 1, g


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [2, 1])
def test_loop_empty_sensor(po, synth, mode):
    """A sensor without pairs (a ray-casting sensor with a zero-size model, a closest-point sensor with an empty dataset) before or after one
    with pairs: it takes no block of the loop and changes no bit of the result, which equals the call on the other sensor alone."""
    import rmcl_b200
    sc = scene(po, synth, 100000)
    Tom, Tbo, Tsb = sc["Tom"], sc["Tbo"], sc["Tsb"]
    full = _cpc(synth, sc, sc["pts"][:100000])
    zero_rcc = rmcl_b200.RCCB200O1Dn(gpu_map(NAME))
    zero_rcc.setTsb(Tsb); zero_rcc.setParams(1.0, 0.15)
    zero_rcc.setModel(synth.O1DnModel(0, 1, np.zeros(3, np.float32), np.zeros((0, 3), np.float32), sc["range_min"], sc["range_max"]))
    empty_cpc = _cpc(synth, sc, np.zeros((0, 3), np.float32))
    for h in (full, zero_rcc, empty_cpc):
        h.setExecMode(mode)
    alone = verify(lambda it: _multi([full], [Tbo], Tom, None, it), lambda: [device_inputs(full, Tbo, Tsb)], Tom, "alone")
    for empty in (zero_rcc, empty_cpc):
        for order in ([empty, full], [full, empty]):
            out = _multi(order, [Tbo, Tbo], Tom)
            assert out[0].tobytes() == alone[0].tobytes() and out[2].tobytes() == alone[2].tobytes(), order
            g = geometry(order[0])
            assert [s["nblk"] == 0 for s in g["sensors"]] == [h is empty for h in order], g
            assert rmcl_b200.load_library().b2_peek_cuda_error().decode() == ""
    # only sensors without pairs: nothing to do on the device, the pose stays
    out = _multi([zero_rcc, empty_cpc], [Tbo, Tbo], Tom)
    assert out[0]["t"].tobytes() == Tom["t"].tobytes() and int(out[2]["n_meas"]) == 0


@pytest.mark.gpu
def test_tile_schedule_at_its_limit(po, synth):
    """The find's tile schedule at B2_PERM_MAX_TILES tiles (368 640 rays, sorted by the loop kernel): the order stays a permutation, the result
    does not depend on it and matches the float64 reference.  One tile more (368 672 rays) switches the schedule off; that run matches too."""
    import rmcl_b200
    max_tiles = 11520                                                                 # B2_PERM_MAX_TILES (icp_loop.cuh)
    osc, Tsb = oracle_scene(NAME), synth.scenario_tsb()
    m = synth.SphericalModel(np.radians(-35.0), np.radians(60.0) / 359, 360, -np.pi, 2 * np.pi / 1024, 1024, 0.5, 120.0)
    assert m.size == 32 * max_tiles
    o, d = po.model_rays(m)
    sc = scene(po, synth, 1000)
    Tom, Tbo, Tgt = sc["Tom"], sc["Tbo"], sc["Tgt"]
    lib = rmcl_b200.load_library()

    def order(h, n_tiles):
        out, n = np.zeros(max(n_tiles, 1), np.uint16), C.c_uint32(0)
        assert lib.b2_rcc_debug_tile_perm(h._h, C.c_void_p(out.ctypes.data), C.c_uint32(len(out)), C.byref(n)) == 0
        return out, n.value

    def dataset(dirs):
        # scan from the true pose; pairs whose first-pass plane distance lies near the gate (0.7 .. 1.3 m) are masked, so that no pair comes
        # within the gate margin while the pose moves by a few centimetres
        ranges = synth.noisy_ranges(osc.simulate(Tgt, Tsb, o, dirs, m.range_max)["ranges"], m.range_max, seed=17)
        dp, dm, _ = po.dataset_from_ranges(o, dirs, ranges, m.range_min, m.range_max)
        sim = osc.simulate(synth.compose(Tom, Tbo), Tsb, o, dirs, m.range_max)
        sd = np.abs(np.einsum("ij,ij->i", sim["points"].astype(np.float64) - dp, sim["normals"].astype(np.float64)))
        dm[(sd > 0.7) & (sd < 1.3)] = 0
        return dp, dm

    h = rmcl_b200.RCCB200Spherical(gpu_map(NAME))
    h.setTsb(Tsb); h.setParams(1.0, 0.15); h.setModel(m)
    dp, dm = dataset(d)
    h.setDataset(dp, dm)
    first = verify(lambda it: h.correctOnce(Tom, Tbo, it, 0.0), lambda: [device_inputs(h, Tbo, Tsb)], Tom, "368 640 rays")   # the loop sorts the
    p1, n1 = order(h, max_tiles)                                                                                          # find's durations
    assert n1 == max_tiles and np.array_equal(np.sort(p1), np.arange(max_tiles)) and not np.array_equal(p1, np.arange(max_tiles))
    for _ in range(2):
        again = h.correctOnce(Tom, Tbo, 5, 0.0)                                        # finds in the sorted order
        assert again[0].tobytes() == first[0].tobytes() and again[2].tobytes() == first[2].tobytes()
        p, _ = order(h, max_tiles)
        assert np.array_equal(np.sort(p), np.arange(max_tiles))
    # one tile more: no schedule
    d2 = np.concatenate([d, d[:32]])
    h2 = rmcl_b200.RCCB200O1Dn(gpu_map(NAME))
    h2.setTsb(Tsb); h2.setParams(1.0, 0.15)
    h2.setModel(synth.O1DnModel(len(d2), 1, np.zeros(3, np.float32), d2, m.range_min, m.range_max))
    dp2, dm2 = dataset(d2)
    h2.setDataset(dp2, dm2)
    verify(lambda it: h2.correctOnce(Tom, Tbo, it, 0.0), lambda: [device_inputs(h2, Tbo, Tsb)], Tom, "368 672 rays")
    assert order(h2, 0)[1] == 0
