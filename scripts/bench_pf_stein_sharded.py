"""Stein variational steps on a particle set sharded over GPUs (b2_pf_stein_slice_*, PCDSensorUpdaterB200.steinUpdateSharded).

Workload: building:1000000 with its field (h 0.05 m, trunc 1 m), 180 beams of a C3 scan, n_all = 1 000 000 particles, n_ref 4096, on a
spread set (uniform over the building) and a converged one (N(true pose, 0.05 m, 0.02 rad)), as in bench_pf_stein.py.

  one GPU (always): for W in 1, 2, 4, 8, the device time (CUDA events) of one rank's iteration, steinScore of its range of J
      (shard_range(m, 0, W)) plus steinMove of its slice of n_all / W particles, median of --reps; alternated call by call with the
      whole-set iteration (the one-rank session, what steinUpdate runs per iteration).  The exchange per rank and iteration is computed from
      the shapes: 32 n_all + 24 W ceil(m / W) bytes gathered (the poses and the padded snapshots), of which the other ranks' share crosses
      the link.  The time of the exchange is not measured in this mode.
  torchrun on N GPUs (WORLD_SIZE set): the full iteration on every rank, both all-gathers included (steinUpdateSharded of --iters
      iterations, host clock around a device synchronise, over --iters), p50 over --reps per rank, and the max over the ranks.

The card name, power limit and maximum SM clock come from the same run.  Writes one JSON line to stdout (rank 0; a table to stderr) and
nothing into the tree.

    python scripts/bench_pf_stein_sharded.py [--reps 50]
    python -m torch.distributed.run --nproc-per-node N scripts/bench_pf_stein_sharded.py [--reps 20]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_micp_chain import card  # noqa: E402
from bench_pf_stein import _max_sm_clock_mhz  # noqa: E402

N_ALL, N_REF, N_BEAMS = 1_000_000, 4096, 180


def _workload(torch, device):
    import rmcl_b200
    from rmcl_b200 import synth
    gmap = rmcl_b200.Map(*synth.building(1_000_000), device=device)
    f = rmcl_b200.DistanceField(gmap, 0.05, 1.0)
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gmap)
    sm = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(sm); h.find(Tgt)
    beams = synth.pf_beams(h.modelView()["points"], N_BEAMS)
    prm = rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.2
    yaw_gt = 2 * np.arctan2(float(Tgt["R"][2]), float(Tgt["R"][3]))
    P, _ = synth.pf_particles(N_ALL)
    rng = np.random.default_rng(3)
    Q = synth.transforms(N_ALL)
    Q["t"] = np.asarray(Tgt["t"], np.float32)
    Q["t"][:, :2] += rng.normal(0, 0.05, (N_ALL, 2)).astype(np.float32)
    yaw = yaw_gt + rng.normal(0, 0.02, N_ALL)
    Q["R"][:, 2], Q["R"][:, 3] = np.sin(yaw / 2), np.cos(yaw / 2)
    return gmap, f, Tsb, beams, prm, {"spread": P, "converged": Q}


def _exchange_bytes(W):
    j_len = -(-N_REF // W)
    return {"poses_gathered": 32 * N_ALL, "snapshot_gathered": 24 * W * j_len, "received_from_other_ranks": 32 * (N_ALL - N_ALL // W) + 24 * (W - 1) * j_len}


def one_gpu(args):
    import torch
    import rmcl_b200
    from rmcl_b200.shard import shard_range
    stream = torch.cuda.current_stream()
    info = card(torch)
    mhz = _max_sm_clock_mhz(torch)
    info["max_sm_clock_mhz"] = mhz if mhz else "not measured"
    print(info, file=sys.stderr, flush=True)
    gmap, f, Tsb, beams, prm, sets = _workload(torch, 0)
    cfg = rmcl_b200.SteinConfig.defaults()
    cfg.n_ref = N_REF
    cfg.iterations = args.warmup + args.reps
    res = {"card": info, "mode": "one GPU, per-rank iteration without the exchange", "n_all": N_ALL, "n_ref": N_REF, "beams": N_BEAMS,
           "multi_gpu_iteration_ms": "not measured (one GPU)", "runs": []}
    for label, P in sets.items():
        P0 = torch.from_numpy(P.view(np.float32).reshape(-1, 8).copy()).cuda()
        for W in (1, 2, 4, 8):
            n_local = N_ALL // W
            ja, jb = shard_range(N_REF, 0, W)
            ups = {}
            for key, (nl, j0, j1) in {"whole": (N_ALL, 0, N_REF), "rank": (n_local, ja, jb)}.items():
                up = rmcl_b200.PCDSensorUpdaterB200(gmap)
                up.setStream(stream.cuda_stream)
                up.setDistanceField(f)
                up.steinBegin(N_ALL, 0, nl, j0, j1 - j0, Tsb, beams, cfg, prm, seed=1)
                ups[key] = (up, torch.empty((nl, 8), dtype=torch.float32, device="cuda"))
            snap = torch.zeros((N_REF, 6), dtype=torch.float32, device="cuda")
            times = {"whole": [], "rank": []}
            for k in range(cfg.iterations):
                for key in ("whole", "rank") if k % 2 == 0 else ("rank", "whole"):
                    up, out = ups[key]
                    j0 = 0 if key == "whole" else ja
                    torch.cuda.synchronize()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    up.steinScore(P0, k, snap[j0:])
                    up.steinMove(P0, snap, k, out)
                    b.record(stream)
                    torch.cuda.synchronize()
                    if k >= args.warmup:
                        times[key].append(a.elapsed_time(b))
            row = {"set": label, "W": W, "n_local": n_local, "j_count": jb - ja, "whole_iteration_ms": round(float(np.median(times["whole"])), 4),
                   "rank_iteration_ms": round(float(np.median(times["rank"])), 4), "exchange_bytes_per_rank_iteration": _exchange_bytes(W)}
            row["speedup_vs_whole"] = round(row["whole_iteration_ms"] / row["rank_iteration_ms"], 2)
            res["runs"].append(row)
            print(row, file=sys.stderr, flush=True)
    print(json.dumps(res))


def multi_gpu(args):
    import torch
    import torch.distributed as dist
    import rmcl_b200
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    try:
        info = card(torch)
        gmap, f, Tsb, beams, prm, sets = _workload(torch, local)
        up = rmcl_b200.PCDSensorUpdaterB200(gmap)
        up.setDistanceField(f)
        cfg = rmcl_b200.SteinConfig.defaults()
        cfg.n_ref, cfg.iterations = N_REF, args.iters
        n_local = N_ALL // world
        runs = []
        for label, P in sets.items():
            P0 = torch.from_numpy(P[rank * n_local:(rank + 1) * n_local].view(np.float32).reshape(-1, 8).copy()).cuda()
            Pl = P0.clone()
            per_it = []
            for r in range(args.warmup + args.reps):
                Pl.copy_(P0)
                torch.cuda.synchronize(); dist.barrier()
                t0 = time.perf_counter()
                up.steinUpdateSharded(Pl, Tsb, beams, dist, cfg, prm, seed=1)
                torch.cuda.synchronize()
                if r >= args.warmup:
                    per_it.append((time.perf_counter() - t0) * 1e3 / args.iters)
            p50 = torch.tensor([float(np.median(per_it))], dtype=torch.float64, device="cuda")
            allp = [torch.zeros_like(p50) for _ in range(world)]
            dist.all_gather(allp, p50)
            runs.append({"set": label, "iteration_ms_p50_per_rank": [round(float(x), 4) for x in allp], "iteration_ms_max_over_ranks":
                         round(max(float(x) for x in allp), 4), "exchange_bytes_per_rank_iteration": _exchange_bytes(world)})
        if rank == 0:
            mhz = _max_sm_clock_mhz(torch)
            info["max_sm_clock_mhz"] = mhz if mhz else "not measured"
            line = {"card": info, "mode": f"torchrun, {world} GPUs, full iteration with both all-gathers (host clock over {args.iters} iterations)",
                    "world": world, "n_all": n_local * world, "n_ref": N_REF, "beams": N_BEAMS, "runs": runs}
            print(line, file=sys.stderr, flush=True)
            print(json.dumps(line))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10, help="iterations per steinUpdateSharded call (torchrun mode)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    multi_gpu(args) if "WORLD_SIZE" in os.environ else one_gpu(args)


if __name__ == "__main__":
    main()
