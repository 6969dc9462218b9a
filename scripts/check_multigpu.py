"""Multi-GPU correctness on hardware (VERDICT r01 item 9): run under torchrun on N >= 2 GPUs of one node.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 scripts/check_multigpu.py

Checks, with particles sharded contiguously over the ranks and the map replicated:
  1. sensor update of the shards == the single-GPU update of the whole set (gathered on rank 0, compared byte for byte);
  2. Gladiator resampling: all-gather variant == peer-memory (CUDA IPC over NVLink) variant on every rank, and their concatenation ==
     rank 0's single-GPU resampling of the gathered set; exchanged bytes of both variants;
  3. particle set initialisation (uniform and Gaussian): each rank's shard (first = rank * n) gathered == rank 0's initialisation of the
     whole set, byte for byte;
  4. Stein steps: steinUpdateSharded over NCCL (3 iterations, n_ref 4096) gathered == rank 0's steinUpdate of the gathered set, byte for
     byte, with the same bandwidth, n_ref and n_blocked.
Prints one JSON line on rank 0; exit code 1 on any mismatch."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
import rmcl_b200
from rmcl_b200 import synth
from rmcl_b200.shard import shard_range


def main():
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    n_per = int(os.environ.get("B2_CHECK_PARTICLES", "50000"))
    V, F = synth.building(200_000)
    gmap = rmcl_b200.Map(V, F, device=local)
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gmap)
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(m); h.find(Tgt)
    beams = synth.pf_beams(h.modelView()["points"], 60)
    P, A = synth.pf_particles(n_per * world, seed=3)
    b, e = shard_range(len(P), rank, world)
    dev = torch.device("cuda", local)
    Pd = torch.from_numpy(P[b:e].view(np.float32).reshape(-1, 8).copy()).to(dev)
    Ad = torch.from_numpy(A[b:e].view(np.float32).reshape(-1, 9).copy()).to(dev)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    prm = rmcl_b200.PFParams.defaults()
    up.update(Pd, Ad, Tsb, beams, prm)
    torch.cuda.synchronize()
    # 1. shards == whole
    A_all = torch.empty((world * n_per, 9), dtype=torch.float32, device=dev)
    dist.all_gather_into_tensor(A_all, Ad)
    ok_update = True
    if rank == 0:
        Pw = torch.from_numpy(P.view(np.float32).reshape(-1, 8).copy()).to(dev)
        Aw = torch.from_numpy(A.view(np.float32).reshape(-1, 9).copy()).to(dev)
        up.update(Pw, Aw, Tsb, beams, prm)
        torch.cuda.synchronize()
        ok_update = bool(torch.equal(Aw, A_all))
    # 2. resampling, both exchange variants
    cfg = rmcl_b200.GladiatorConfig.defaults()
    torch.cuda.synchronize(); dist.barrier()
    t0 = time.perf_counter()
    Pg, Ag = up.resampleSharded(Pd, Ad, dist, cfg, seed=99, step=1)
    torch.cuda.synchronize(); dist.barrier()
    t_allgather = time.perf_counter() - t0
    p2p_err, Pp, Ap, traffic, t_p2p = None, None, None, 0, None
    try:
        up.p2pConnect(dist, n_per)
        up.resampleShardedP2P(Pd, Ad, dist, cfg, seed=99, step=1)                 # warm-up (maps, first touch)
        torch.cuda.synchronize(); dist.barrier()
        t0 = time.perf_counter()
        Pp, Ap, traffic = up.resampleShardedP2P(Pd, Ad, dist, cfg, seed=99, step=1, want_traffic=True)
        torch.cuda.synchronize(); dist.barrier()
        t_p2p = time.perf_counter() - t0
    except rmcl_b200.B2Error as ex:
        p2p_err = str(ex)
    same_variants = p2p_err is None and bool(torch.equal(Pp, Pg) and torch.equal(Ap, Ag))
    flags = torch.tensor([int(same_variants), traffic], dtype=torch.int64, device=dev)
    allf = [torch.zeros_like(flags) for _ in range(world)]
    dist.all_gather(allf, flags)
    Pn_all = torch.empty((world * n_per, 8), dtype=torch.float32, device=dev)
    An_all = torch.empty((world * n_per, 9), dtype=torch.float32, device=dev)
    dist.all_gather_into_tensor(Pn_all, Pg); dist.all_gather_into_tensor(An_all, Ag)
    P_all = torch.empty((world * n_per, 8), dtype=torch.float32, device=dev)
    dist.all_gather_into_tensor(P_all, Pd)
    # 3. initialisation: every rank initialises its shard (first = rank * n_per), the gathered set == one initialisation of the whole set
    bb_min, bb_max = [1.0, 1.0, 0.5, 0.0, 0.0, -np.pi], [59.0, 39.0, 0.5, 0.0, 0.0, np.pi]
    cov = np.diag([0.25, 0.25, 0.0, 0.0, 0.0, 0.0685])
    Pi, Ai = torch.empty_like(Pd), torch.empty_like(Ad)
    Pi_all, Ai_all = torch.empty_like(P_all), torch.empty_like(A_all)
    gathered = {}
    for kind in ("uniform", "gaussian"):
        if kind == "uniform":
            up.initSamplesUniform(Pi, Ai, bb_min, bb_max, seed=17, first=rank * n_per)
        else:
            up.initSamples(Pi, Ai, Tgt, cov, seed=17, first=rank * n_per)
        dist.all_gather_into_tensor(Pi_all, Pi); dist.all_gather_into_tensor(Ai_all, Ai)
        gathered[kind] = (Pi_all.clone(), Ai_all.clone())
    # 4. Stein steps on the sharded set: all-gathers of the poses and of J's snapshot per iteration, each rank moving its own shard
    us = rmcl_b200.PCDSensorUpdaterB200(gmap)
    us.setDistanceField(rmcl_b200.DistanceField(gmap, 0.05, 1.0))
    scfg = rmcl_b200.SteinConfig.defaults()
    scfg.iterations = 3
    sprm = rmcl_b200.PFParams.defaults()
    sprm.dist_sigma = 0.2
    Ps = Pd.clone()
    torch.cuda.synchronize(); dist.barrier()
    t0 = time.perf_counter()
    sres = us.steinUpdateSharded(Ps, Tsb, beams, dist, scfg, sprm, seed=5, step=2)
    torch.cuda.synchronize(); dist.barrier()
    t_stein = time.perf_counter() - t0
    Ps_all = torch.empty_like(P_all)
    dist.all_gather_into_tensor(Ps_all, Ps)
    rc = 0
    if rank == 0:
        Pw = P_all.clone()
        wres = us.steinUpdate(Pw, Tsb, beams, scfg, sprm, seed=5, step=2)
        torch.cuda.synchronize()
        ok_stein = (bool(torch.equal(Pw.view(torch.int32), Ps_all.view(torch.int32))) and wres["bandwidth"] == sres["bandwidth"]
                    and (wres["n_ref"], wres["n_blocked"]) == (sres["n_ref"], sres["n_blocked"]) and not torch.equal(Pw, P_all))
        ok_init = True
        for kind, (Pg_i, Ag_i) in gathered.items():
            Pw, Aw = torch.empty_like(P_all), torch.empty_like(A_all)
            if kind == "uniform":
                up.initSamplesUniform(Pw, Aw, bb_min, bb_max, seed=17)
            else:
                up.initSamples(Pw, Aw, Tgt, cov, seed=17)
            torch.cuda.synchronize()
            ok_init = ok_init and bool(torch.equal(Pw.view(torch.int32), Pg_i.view(torch.int32)) and torch.equal(Aw.view(torch.int32), Ag_i.view(torch.int32)))
        Pr, Ar = torch.empty_like(P_all), torch.empty_like(A_all)
        up.resample(P_all, A_all, Pr, Ar, cfg, seed=99, step=1)
        torch.cuda.synchronize()
        ok_resample = bool(torch.equal(Pr, Pn_all) and torch.equal(Ar, An_all))
        changed = float((Ar[:, 0] != A_all[:, 0]).float().mean())
        line = {"world": world, "particles_per_rank": n_per, "sensor_update_shards_equal_whole": ok_update, "resample_sharded_equals_single_gpu": ok_resample,
                "init_shards_equal_whole": ok_init, "stein_sharded_equals_single_gpu": ok_stein, "stein_sharded_wall_ms": t_stein * 1e3,
                "p2p_equals_allgather_on_every_rank": [bool(int(f[0])) for f in allf] if p2p_err is None else None, "p2p_error": p2p_err,
                "fraction_of_slots_replaced": changed, "checksum": hex(int(torch.from_numpy(Pn_all.cpu().numpy().view(np.uint32).astype(np.uint64)).sum().item()) & 0xffffffffffff),
                "exchange_bytes": {"allgather_received_per_rank": (world - 1) * n_per * 68, "p2p_read_per_rank": [int(f[1]) for f in allf]},
                "wall_ms": {"allgather_variant": t_allgather * 1e3, "p2p_variant": None if t_p2p is None else t_p2p * 1e3}}
        print(json.dumps(line))
        if not (ok_update and ok_resample and ok_init and ok_stein and (p2p_err is not None or all(int(f[0]) for f in allf))):
            rc = 1
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(rc)


if __name__ == "__main__":
    main()
