"""GPU tests of the Stein steps on a sharded particle set (b2_pf_stein_slice_*, PCDSensorUpdaterB200.steinBegin / steinScore / steinMove /
steinResult / steinUpdateSharded, SURVEY L14) against steinUpdate of the whole set, whose bits tests/test_gpu_pf_stein.py pins to the
host-compiled product.

W handles on one device play W ranks.  Per iteration every rank scores its range of J into its offset of one snapshot buffer (the
all-gather of the snapshots), then every rank moves its slice into its own buffer, and the buffers are copied back into the whole set (the
all-gather of the poses).

Tolerances: poses, bandwidth and n_ref exact (bytes); n_blocked summed over the ranks exact; the RMS steps from the summed FP64 sums
within 1e-6 relative (the slices' block partials are summed in another order than the whole grid's), exact for one rank."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import native
import test_gpu_pf_stein as G
from conftest import mesh

pytestmark = pytest.mark.gpu


def _updater(f, gmap):
    import rmcl_b200
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    up.setDistanceField(f)
    return up


def _prm():
    import rmcl_b200
    prm = rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.2
    return prm


def _ranks(n, m, W):
    from rmcl_b200.shard import shard_range
    return [(shard_range(n, r, W), shard_range(m, r, W)) for r in range(W)]


def _run_slices(ups, Pd, Tsb, B, cfg, in_place=False, counts=None):
    """len(ups) ranks on one device; Pd (n, 8) is left as it was.  -> (poses (n, 8), per-rank records)"""
    import rmcl_b200
    import torch
    n, W = Pd.shape[0], len(ups)
    m = n if cfg.n_ref == 0 or cfg.n_ref >= n else cfg.n_ref
    ranks = _ranks(n, m, W)
    for up, ((a, b), (ja, jb)) in zip(ups, ranks):
        up.steinBegin(n, a, b - a, ja, jb - ja, Tsb, B, cfg, _prm(), seed=1234, step=7)
    snap = torch.zeros((max(m, 1), 6), dtype=torch.float32, device=Pd.device)
    P_all = Pd.clone()
    for k in range(cfg.iterations):
        for up, (_, (ja, jb)) in zip(ups, ranks):
            c0 = rmcl_b200.kernel_launch_count()
            up.steinScore(P_all, k, snap[ja:])
            if counts is not None:
                counts.append(("score", jb - ja, rmcl_b200.kernel_launch_count() - c0))
        alls = [P_all.clone() for _ in ups] if in_place else [P_all] * W
        outs = []
        for up, ((a, b), _), Pr in zip(ups, ranks, alls):
            out = Pr[a:b] if in_place else torch.empty((b - a, 8), dtype=torch.float32, device=Pd.device)
            c0 = rmcl_b200.kernel_launch_count()
            up.steinMove(Pr, snap[:m], k, out)
            if counts is not None:
                counts.append(("move", b - a, rmcl_b200.kernel_launch_count() - c0))
            outs.append(out)
        P_all = torch.cat(outs) if outs else P_all
    return P_all, [up.steinResult() for up in ups]


def _rms(res):
    n_steps = sum(r["n_steps"] for r in res)
    f = lambda key: float(np.float32(np.sqrt(sum(r[key] for r in res) / n_steps))) if n_steps else 0.0
    return f("sum_step_t2"), f("sum_step_r2")


def _check(got, want, res, rec, W):
    assert got.cpu().numpy().tobytes() == want.cpu().numpy().tobytes(), f"W {W}"
    hb = np.array(rec["bandwidth"], np.float32).tobytes()
    assert all(np.array(r["bandwidth"], np.float32).tobytes() == hb and r["n_ref"] == rec["n_ref"] for r in res), W
    assert sum(r["n_blocked"] for r in res) == rec["n_blocked"], W
    rt, rr = _rms(res)
    for g, w in ((rt, rec["rms_step_t"]), (rr, rec["rms_step_r"])):
        assert abs(g - w) <= 1e-6 * abs(w), (W, g, w)
        if W == 1:
            assert np.float32(g) == np.float32(w)


_ROWS = [
    ("indoor:500000", 1, 0, 180, 10), ("indoor:500000", 33, 0, 1, 10), ("indoor:500000", 33, 4096, 0, 10), ("indoor:500000", 4097, 0, 180, 10),
    ("indoor:500000", 4097, 4096, 1000, 10), ("indoor:500000", 100_000, 4096, 180, 10), ("indoor:500000", 100_000, 0, 180, 1),
    ("building:1000000", 1, 4096, 1000, 10), ("building:1000000", 33, 4096, 180, 10), ("building:1000000", 4097, 0, 0, 10),
    ("building:1000000", 4097, 4096, 180, 1), ("building:1000000", 100_000, 4096, 1000, 1), ("building:1000000", 1_000_000, 4096, 180, 1)]


@pytest.mark.parametrize("name,n,n_ref,n_beams,iters", _ROWS)
def test_slices_on_one_device_equal_the_whole_set(name, n, n_ref, n_beams, iters):
    """W = 1, 2, 3, 8 ranks: the concatenated slices equal steinUpdate of the whole set byte for byte, and so do the bandwidth, n_ref and the
    summed n_blocked"""
    from rmcl_b200 import synth
    gmap, f, *_ = G._setup(name)
    P, B, Tsb = G._poses(name, n), G._beams(n_beams), synth.scenario_tsb()
    cfg = G._cfg(iters, n_ref)
    Pd = G._tensor(P)
    want = Pd.clone()
    rec = _updater(f, gmap).steinUpdate(want, Tsb, B, cfg, _prm(), seed=1234, step=7)
    for W in (1, 2, 3, 8):
        got, res = _run_slices([_updater(f, gmap) for _ in range(W)], Pd, Tsb, B, cfg)
        _check(got, want, res, rec, W)
    print(f"{name} n {n} n_ref {n_ref} beams {n_beams} x{iters}: blocked {rec['n_blocked']}, h {np.round(rec['bandwidth'], 4)}")


def test_in_place_move_and_launch_count():
    """an in-place move (poses_out = poses_all + first, each rank its own copy of the set) equals an out-of-place one; each rank-iteration
    launches score 1 (0 for an empty J range) and move 2 (bandwidth, move; 1 for an empty slice: the bandwidth always runs)"""
    from rmcl_b200 import synth
    gmap, f, *_ = G._setup("indoor:500000")
    n, W = 5, 8
    P, B, Tsb = G._poses("indoor:500000", n), G._beams(180), synth.scenario_tsb()
    cfg = G._cfg(3, 0)
    Pd = G._tensor(P)
    want = Pd.clone()
    rec = _updater(f, gmap).steinUpdate(want, Tsb, B, cfg, _prm(), seed=1234, step=7)
    counts = []
    got, res = _run_slices([_updater(f, gmap) for _ in range(W)], Pd, Tsb, B, cfg, in_place=True, counts=counts)
    _check(got, want, res, rec, W)
    got2, _ = _run_slices([_updater(f, gmap) for _ in range(W)], Pd, Tsb, B, cfg)
    assert got.cpu().numpy().tobytes() == got2.cpu().numpy().tobytes()
    assert len(counts) == 2 * W * cfg.iterations
    for kind, size, launched in counts:
        assert launched == (1 if kind == "score" else 2) - (0 if size else 1), (kind, size, launched)
    big = [_updater(f, gmap) for _ in range(2)]
    counts = []
    _run_slices(big, G._tensor(G._poses("indoor:500000", 4097)), Tsb, B, G._cfg(2, 4096), counts=counts)
    assert all(launched == (1 if kind == "score" else 2) for kind, _, launched in counts)


def test_refusals_leave_the_session_unchanged():
    """null arguments, ranges beyond n_all or m, iterations out of sequence, a move before its score and an iteration >= cfg.iterations are
    refused with nothing launched; the session then runs on and still equals steinUpdate.  n_all == 0: B2_OK everywhere."""
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    gmap, f, *_ = G._setup("indoor:500000")
    n = 300
    P, B, Tsb = G._poses("indoor:500000", n), G._beams(40), synth.scenario_tsb()
    cfg = G._cfg(2, 100)
    Pd = G._tensor(P)
    want = Pd.clone()
    rec = _updater(f, gmap).steinUpdate(want, Tsb, B, cfg, _prm(), seed=1234, step=7)
    up = _updater(f, gmap)
    lib = rmcl_b200.load_library()
    snap = torch.zeros((100, 6), dtype=torch.float32, device=Pd.device)
    out = torch.empty_like(Pd)
    with pytest.raises(rmcl_b200.B2Error):
        up.steinScore(Pd, 0, snap)                                   # no session
    up.steinBegin(n, 0, n, 0, 100, Tsb, B, cfg, _prm(), seed=1234, step=7)
    n0 = rmcl_b200.kernel_launch_count()

    def refused(call):
        with pytest.raises(rmcl_b200.B2Error) as e:
            call()
        assert e.value.code == -1

    refused(lambda: up.steinBegin(n, 1, n, 0, 100, Tsb, B, cfg, _prm()))             # slice beyond n_all
    refused(lambda: up.steinBegin(n, 0, n, 50, 51, Tsb, B, cfg, _prm()))             # J range beyond m
    refused(lambda: up.steinMove(Pd, snap, 0, out))                                  # move before score
    refused(lambda: up.steinScore(Pd, 1, snap))                                      # out of sequence
    refused(lambda: up.steinScore(None, 0, snap))                                    # null poses
    refused(lambda: up.steinScore(Pd, 0, None))                                      # null snapshot
    up.steinScore(Pd, 0, snap)
    refused(lambda: up.steinScore(Pd, 0, snap))                                      # score twice
    refused(lambda: up.steinMove(Pd, None, 0, out))                                  # null snapshot
    refused(lambda: up.steinMove(Pd, snap, 0, None))                                 # null output
    refused(lambda: up.steinMove(Pd, snap, 0, Pd[1:]))                               # output overlapping the set off the slice
    refused(lambda: up.steinMove(Pd, snap, 1, out))                                  # out of sequence
    assert lib.b2_pf_stein_slice_begin(up._h, None, n, 0, n, 0, 100, None, None, 0, None, None, C.c_uint64(0), 0) == -1      # null field
    assert rmcl_b200.kernel_launch_count() == n0 + 1
    up.steinMove(Pd, snap, 0, out)
    Pd.copy_(out)
    up.steinScore(Pd, 1, snap)
    up.steinMove(Pd, snap, 1, out)
    refused(lambda: up.steinScore(out, 2, snap))                                     # iteration >= cfg.iterations
    r = up.steinResult()
    assert out.cpu().numpy().tobytes() == want.cpu().numpy().tobytes()
    assert np.array(r["bandwidth"], np.float32).tobytes() == np.array(rec["bandwidth"], np.float32).tobytes()
    assert (r["n_ref"], r["n_blocked"]) == (rec["n_ref"], rec["n_blocked"]) and _rms([r]) == (rec["rms_step_t"], rec["rms_step_r"])
    # n_all == 0: every call B2_OK, nothing launched, a zeroed record
    n0 = rmcl_b200.kernel_launch_count()
    up.steinBegin(0, 0, 0, 0, 0, Tsb, B, cfg, _prm())
    for k in range(3):
        up.steinScore(None, k, None)
        up.steinMove(None, None, k, None)
    assert rmcl_b200.kernel_launch_count() == n0 and up.steinResult()["n_ref"] == 0


@pytest.mark.skipif("__import__('torch').cuda.device_count() < 2")
def test_field_on_another_device_is_refused():
    import rmcl_b200
    from rmcl_b200 import synth
    V, F = mesh("indoor:500000")
    f1 = rmcl_b200.DistanceField(rmcl_b200.Map(V, F, device=1), 0.05, 1.0)
    gmap, *_ = G._setup("indoor:500000")
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    up.setDistanceField(f1)
    with pytest.raises(rmcl_b200.B2Error):
        up.steinBegin(10, 0, 10, 0, 10, synth.scenario_tsb(), G._beams(4))


def test_world_size_one_nccl_equals_stein_update(tmp_path):
    """steinUpdateSharded in a one-rank NCCL group equals steinUpdate, and the handle's stream is restored"""
    import torch
    import torch.distributed as dist
    from rmcl_b200 import synth
    gmap, f, *_ = G._setup("building:1000000")
    P, B, Tsb = G._poses("building:1000000", 20_000), G._beams(180), synth.scenario_tsb()
    cfg = G._cfg(5, 4096)
    want = G._tensor(P)
    rec = _updater(f, gmap).steinUpdate(want, Tsb, B, cfg, _prm(), seed=1234, step=7)
    dist.init_process_group("nccl", store=dist.FileStore(str(tmp_path / "store"), 1), rank=0, world_size=1)
    try:
        up = _updater(f, gmap)
        Pl = G._tensor(P)
        res = up.steinUpdateSharded(Pl, Tsb, B, dist, cfg, _prm(), seed=1234, step=7)
        torch.cuda.synchronize()
        assert up._stream == 0
    finally:
        dist.destroy_process_group()
    assert Pl.cpu().numpy().tobytes() == want.cpu().numpy().tobytes()
    assert res == rec


def test_cpp_classes_match_stein_update(tmp_path):
    """tests/pf_stein_cpp/pf_stein_cpp.cpp, compiled here against include/rmcl_b200/rcc_b200.hpp: two ranks through steinBegin / steinScore /
    steinMove on one device equal the class's steinUpdate byte for byte, which equals the Python steinUpdate"""
    import rmcl_b200
    from rmcl_b200 import synth
    exe = native.adapter("pf_stein_cpp")
    V, F = synth.indoor(2000)
    V, F = np.ascontiguousarray(V, np.float32), np.ascontiguousarray(F, np.uint32)
    n, iters, n_ref = 3001, 4, 1000
    P, Tsb = G._poses("indoor:500000", n), synth.scenario_tsb()
    P["t"][:, :2] -= P["t"][:, :2].mean(0) - V[:, :2].mean(0)             # around the middle of the small indoor mesh
    B = G._beams(60)
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as fh:
        fh.write(np.array([len(V), len(F), n, len(B), iters, n_ref], np.uint32).tobytes())
        fh.write(np.array([0.05, 1.0, 0.2], np.float32).tobytes())
        fh.write(V.tobytes()); fh.write(F.tobytes()); fh.write(np.ascontiguousarray(Tsb).tobytes()); fh.write(P.tobytes()); fh.write(B.tobytes())
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "REFUSED" in r.stdout and "sequence" in r.stdout
    raw = np.fromfile(out, np.uint8)
    rec_cpp, poses_cpp = raw[:32], raw[32:32 + 32 * n]
    slice_recs, poses_sl = raw[32 + 32 * n:112 + 32 * n], raw[112 + 32 * n:]
    assert poses_sl.tobytes() == poses_cpp.tobytes()
    gmap = rmcl_b200.Map(V, F)
    f = rmcl_b200.DistanceField(gmap, 0.05, 1.0)
    Pd = G._tensor(P)
    res = _updater(f, gmap).steinUpdate(Pd, Tsb, B, G._cfg(iters, n_ref), _prm(), seed=1234, step=7)
    assert poses_cpp.tobytes() == Pd.cpu().numpy().tobytes()
    c = rec_cpp.view(np.float32)
    assert c[:3].tobytes() == np.array(res["bandwidth"], np.float32).tobytes() and rec_cpp[12:20].view(np.uint32).tolist() == [res["n_ref"], res["n_blocked"]]
    sr = slice_recs.reshape(2, 40)
    assert sum(int(s[16:20].view(np.uint32)[0]) for s in sr) == res["n_blocked"]
    moved = (G._host(Pd)["t"][:, :2] != P["t"][:, :2]).any(1).sum()
    assert moved > n // 2
