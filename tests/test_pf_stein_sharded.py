"""CPU tests of the Stein steps on a sharded particle set (b2_pf_stein_slice_*, shard.stein_update_sharded, SURVEY L14) through the
product's functions compiled for the host (tests/pf_stein_sharded_ref.py): W emulated rank sessions, each scoring its range of J and moving its
slice, against the emulated whole-set b2_pf_stein_update.

Tolerances.
  * poses, bandwidth, n_ref: exact (bytes).  Every rank computes the bandwidth over the whole set in est_grid_reduce's order, and each
    slice's move reads the same snapshot the whole-set move reads.
  * n_blocked summed over the ranks: exact (integer counts).
  * RMS steps from the summed step counts and FP64 sums: within 1e-6 relative of the whole-set record.  The slices' block partials are
    summed in another order than the whole grid's, which moves the FP64 sums by a few ulp; the square root and the rounding to float
    keep that far below 1e-6."""
import ctypes as C
import os
import socket
import sys

import numpy as np
import pytest

import pf_stein_ref as S
import pf_stein_sharded_ref as SR
import test_pf_stein as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_WALLS = {}


def _walls(name, d):
    """the field's mesh as the slice library's host-built BVH"""
    if name not in _WALLS:
        _WALLS[name] = SR.Walls(d["V"], d["F"])
    return _WALLS[name]


def _cfg(iterations, n_ref):
    return S.SteinConfig(iterations, n_ref, 0.02, 0.01, 0.05, 0.02, 0.05, 0.0)


def _slices(d, walls, P, B, Tsb, cfg, W, seed=1234, step=7):
    """W emulated ranks: rank r moves shard_range(n, r, W) and scores shard_range(m, r, W) of J.  Per iteration every rank scores, the
    snapshots are concatenated in rank order (the all-gather), then every rank moves its slice into its own buffer, and the buffers are
    concatenated (the next iteration's all-gather).  -> (poses, per-rank records)"""
    from rmcl_b200.shard import shard_range
    n = len(P)
    m = S.n_refs(n, cfg.n_ref)
    ranks = []
    for r in range(W):
        a, b = shard_range(n, r, W)
        ja, jb = shard_range(m, r, W)
        ranks.append(SR.Session(walls, d["g"], d["index"], d["bricks"], n, a, b - a, ja, jb - ja, Tsb, B, 0.2, cfg, seed, step))
    P_all = np.array(P, copy=True)
    for k in range(cfg.iterations):
        snap_all = np.concatenate([s.score(P_all, k) for s in ranks])
        assert len(snap_all) == m
        outs = []
        for s in ranks:
            out = np.empty(s.n_local, P.dtype)
            s.move(P_all, snap_all, k, out)
            outs.append(out)
        P_all = np.concatenate(outs)
    return P_all, [s.result() for s in ranks]


def _whole_rms(results):
    n_steps = sum(r["n_steps"] for r in results)
    rms = lambda key: float(np.float32(np.sqrt(sum(r[key] for r in results) / n_steps))) if n_steps else 0.0
    return rms("sum_step_t2"), rms("sum_step_r2")


_CASES = [(n, kind, nb, it) for n in (1, 33) for kind in ("all", "4096", "ge") for nb in (0, 1, 180) for it in (1, 10)]
_CASES += [(4097, kind, nb, 1) for kind in ("all", "4096", "ge") for nb in (0, 1, 180)] + [(4097, "4096", 180, 10)]


@pytest.mark.parametrize("n,n_ref_kind,n_beams,iters", _CASES)
def test_slices_concatenate_to_the_whole_set(n, n_ref_kind, n_beams, iters):
    """for W = 1 ... 7 ranks (W > n leaves slices and J ranges empty; n = 33 and 4097 give unequal slices) the slices after `iters`
    iterations equal the whole-set update byte for byte; every rank's bandwidth is the whole's; n_blocked sums exactly"""
    d = T._field("indoor")
    n_ref = {"all": 0, "4096": 4096, "ge": n + 5}[n_ref_kind]
    P, B, Tsb = T._poses(n), T._beams(n_beams), T._tsb()
    cfg = _cfg(iters, n_ref)
    want, rec = d["scene"].update(d["g"], d["index"], d["bricks"], P, Tsb, B, 0.2, cfg, 1234, 7)
    hb = np.array(rec.bandwidth, np.float32).tobytes()
    for W in range(1, 8):
        got, res = _slices(d, _walls("indoor", d), P, B, Tsb, cfg, W)
        assert got.tobytes() == want.tobytes(), f"W {W}: {np.flatnonzero((got.view(np.uint32).reshape(n, 8) != want.view(np.uint32).reshape(n, 8)).any(1))[:5]}"
        assert all(np.array(r["bandwidth"], np.float32).tobytes() == hb and r["n_ref"] == rec.n_ref for r in res), W
        assert sum(r["n_blocked"] for r in res) == rec.n_blocked, W
        rt, rr = _whole_rms(res)
        for got_rms, want_rms in ((rt, rec.rms_step_t), (rr, rec.rms_step_r)):
            assert abs(got_rms - want_rms) <= 1e-6 * abs(want_rms), (W, got_rms, want_rms)
        if W == 1:
            assert (rt, rr) == (np.float32(rec.rms_step_t), np.float32(rec.rms_step_r))
    print(f"n {n} n_ref {n_ref} beams {n_beams} x{iters}: blocked {rec.n_blocked}, h {np.round(rec.bandwidth[:], 4)}")


# ---------------------------------------------------------------- gloo --------------------------------------------------------------------
def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch
    import torch.distributed as dist
    import pf_stein_sharded_ref as SR
    import test_pf_stein as T
    from rmcl_b200 import synth
    from rmcl_b200.shard import stein_update_sharded
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        d = T._field("indoor")
        walls = SR.Walls(d["V"], d["F"])
        n_local = 20
        P = T._poses(world * n_local)
        B, Tsb = T._beams(30), T._tsb()
        cfg = _cfg(4, 50)
        sess = {}

        def begin(n_all, first, n, j_first, j_count):
            sess["s"] = SR.Session(walls, d["g"], d["index"], d["bricks"], n_all, first, n, j_first, j_count, Tsb, B, 0.2, cfg, 99, 3)

        def score(P_all, k, snap):
            rows = sess["s"].score(P_all.numpy().view(synth.TRANSFORM_DTYPE).reshape(-1), k)
            snap[: len(rows)] = torch.from_numpy(rows)

        def move(P_all, snap_all, k, out):
            sess["s"].move(P_all.numpy().view(synth.TRANSFORM_DTYPE).reshape(-1), snap_all.numpy(), k, out.numpy().view(synth.TRANSFORM_DTYPE).reshape(-1))

        Pl = torch.from_numpy(P[rank * n_local:(rank + 1) * n_local].view(np.float32).reshape(-1, 8).copy())
        res = stein_update_sharded(begin, score, move, lambda: sess["s"].result(), Pl, dist, cfg.iterations, cfg.n_ref)
        outs = [torch.empty_like(Pl) for _ in range(world)]
        dist.all_gather(outs, Pl)
        if rank == 0:
            want, rec = d["scene"].update(d["g"], d["index"], d["bricks"], P, Tsb, B, 0.2, cfg, 99, 3)
            got = torch.cat(outs).numpy().view(synth.TRANSFORM_DTYPE).reshape(-1)
            ok = (got.tobytes() == want.tobytes() and not np.array_equal(got["t"], P["t"])
                  and np.array(res["bandwidth"], np.float32).tobytes() == np.array(rec.bandwidth, np.float32).tobytes()
                  and (res["n_ref"], res["n_blocked"]) == (rec.n_ref, rec.n_blocked)
                  and abs(res["rms_step_t"] - rec.rms_step_t) <= 1e-6 * rec.rms_step_t and abs(res["rms_step_r"] - rec.rms_step_r) <= 1e-6 * rec.rms_step_r)
            q.put(("ok", ok))
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_stein_update_sharded_over_gloo_equals_the_whole(world):
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    tag, ok = q.get(timeout=5)
    assert tag == "ok" and ok


# ---------------------------------------------------------------- ABI ---------------------------------------------------------------------
def test_abi_records_exports_and_null_handle():
    import rmcl_b200
    from rmcl_b200 import api
    assert C.sizeof(api._SteinSliceResult) == 40 and C.sizeof(SR.SteinSliceResult) == 40
    hdr = open(os.path.join(ROOT, "include", "rmcl_b200.h")).read()
    assert "b2_stein_ref_is_24_bytes[sizeof(b2_stein_ref) == 24" in hdr and "b2_stein_slice_result_is_40_bytes[sizeof(b2_stein_slice_result) == 40" in hdr
    names = ["b2_pf_stein_slice_begin", "b2_pf_stein_slice_score", "b2_pf_stein_slice_move", "b2_pf_stein_slice_result"]
    assert all(x in api.EXPORTS for x in names)
    for meth in ("steinBegin", "steinScore", "steinMove", "steinResult", "steinUpdateSharded"):
        assert callable(getattr(rmcl_b200.PCDSensorUpdaterB200, meth))
    if not os.path.exists(rmcl_b200.lib_path()):
        pytest.skip("library not built")
    lib = rmcl_b200.load_library()
    r = SR.SteinSliceResult()
    assert lib.b2_pf_stein_slice_begin(None, None, 0, 0, 0, 0, 0, None, None, 0, None, None, C.c_uint64(0), 0) == -1
    assert lib.b2_pf_stein_slice_score(None, None, 0, None) == -1
    assert lib.b2_pf_stein_slice_move(None, None, None, 0, None) == -1
    assert lib.b2_pf_stein_slice_result(None, C.byref(r)) == -1
