"""Residual resampling on the device (b2_pf_resample_residual) against the reference's path, in three cases:

  50000->1000000    : the node's defaults, a 50 000-particle set grown into the whole max_particles buffer;
  1000000->1000000  : a full set resampled into the same size;
  dominant          : one particle holds 99 % of the weight among 1 000 000 (the others share 1 %), into 1 000 000 slots.

  device : host wall clock around one synchronised resampleResidual call, median over --reps (>= 50); in a separate profiled run, the
           device time per call of the residual kernels and the scan (torch.profiler, CUDA activities); the number of draws and of chunks
           (one host read-back each).
  host   : what the node's residual path costs on the b200 backend (prepareMemory("cpu"), ResidualResamplerCPU::update, the set back to
           the device): download of the input set, the C restatement's loop of tests/pf_residual_ref (single thread, as the reference's
           loop is), upload of the filled slots.  Median over --host-reps.

The card name and power limit come from the same run.  Writes one JSON line to stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pf_residual.py [--reps 50] [--host-reps 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import pf_residual_ref  # noqa: E402  (the host loop)
from bench_micp_chain import card  # noqa: E402

KERNELS = ("k_pf_residual_stats", "k_pf_residual_counts", "DeviceScan", "k_pf_residual_find", "k_pf_residual_expand")
CASES = (("50000->1000000", 50_000, 1_000_000, "uniform"), ("1000000->1000000", 1_000_000, 1_000_000, "uniform"),
         ("dominant", 1_000_000, 1_000_000, "dominant"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.reps < 50:
        raise SystemExit("--reps must be at least 50")

    import torch
    import rmcl_b200
    from rmcl_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    stream = torch.cuda.current_stream()
    V, F = synth.cube(3)
    up = rmcl_b200.PCDSensorUpdaterB200(rmcl_b200.Map(V, F, device=0))
    up.setStream(stream.cuda_stream)
    cfg = rmcl_b200.GladiatorConfig.defaults()
    print(f"{card(torch)}", file=sys.stderr, flush=True)
    res = {}
    for name, n, M, kind in CASES:
        P = torch.empty((n, 8), dtype=torch.float32, device="cuda")
        A = torch.empty((n, 9), dtype=torch.float32, device="cuda")
        up.initSamples(P, A, synth.make_transform((10.0, -3.0, 0.0), (0.0, 0.0, 0.8)), np.diag([0.25, 0.25, 0.0, 0.0, 0.0, 0.07]), 1)
        g = torch.Generator("cuda").manual_seed(2)
        if kind == "uniform":
            A[:, 0] = torch.rand(n, device="cuda", generator=g)                                  # likelihoods in [0, 1)
        else:
            A[:, 0] = torch.rand(n, device="cuda", generator=g) * (0.02 / n)                     # mean 0.01 / n: 1 % of the weight
            A[n // 3, 0] = 0.99
        Pn = torch.empty((M, 8), dtype=torch.float32, device="cuda")
        An = torch.empty((M, 9), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        for _ in range(args.warmup):
            r = up.resampleResidual(P, A, Pn, An, cfg, seed=1, step=0)
        wall = []
        for step in range(args.reps):
            t0 = time.perf_counter()
            r = up.resampleResidual(P, A, Pn, An, cfg, seed=1, step=step)
            wall.append(time.perf_counter() - t0)
        call_us = float(np.median(wall)) * 1e6
        draws = [int(up.resampleResidual(P, A, Pn, An, cfg, seed=1, step=s)["draws"]) for s in range(8)]
        chunks = [pf_residual_ref.chunks(n, M, d) for d in draws]
        from torch.profiler import ProfilerActivity, profile
        n_prof = 20
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for step in range(n_prof):
                up.resampleResidual(P, A, Pn, An, cfg, seed=1, step=step)
        kern = {k: 0.0 for k in KERNELS}
        for e in prof.key_averages():
            for k in KERNELS:
                if k in e.key:
                    kern[k] += e.device_time_total / n_prof                           # us per call
        kern_us = sum(kern.values())
        hw = []
        for _ in range(args.host_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            hp = P.cpu().numpy().view(synth.TRANSFORM_DTYPE).reshape(-1)            # prepareMemory("cpu")
            ha = A.cpu().numpy().view(synth.PARTICLE_ATTR_DTYPE).reshape(-1)
            h = pf_residual_ref.resample(hp, ha, M, cfg, 1, 0)                        # the host loop
            k = h["n_particles"]
            Pn[:k].copy_(torch.from_numpy(h["P"][:k].view(np.float32).reshape(k, 8)))    # prepareMemory("gpu")
            An[:k].copy_(torch.from_numpy(h["A"][:k].view(np.float32).reshape(k, 9)))
            torch.cuda.synchronize()
            hw.append(time.perf_counter() - t0)
        host_us = float(np.median(hw)) * 1e6
        res[name] = {"particles": n, "slots": M, "n_particles": int(r["n_particles"]), "draws": draws, "chunks": chunks,
                     "call_us": call_us, "call_us_spread": [float(np.min(wall)) * 1e6, float(np.max(wall)) * 1e6],
                     "kernel_us": kern, "kernel_us_total": kern_us, "reference_copy_loop_copy_us": host_us, "speedup": host_us / call_us}
        print(f"{name:>18s}  call {call_us:9.1f} us  kernels {kern_us:8.1f} us  draws {min(draws)}..{max(draws)}  chunks {min(chunks)}..{max(chunks)}  "
              f"reference {host_us / 1e3:10.2f} ms", file=sys.stderr, flush=True)
        del P, A, Pn, An
    out = {"workload": "resampleResidual (initSamples with rviz's covariance; likelihoods uniform in [0, 1), or one particle with 99 % of the weight)",
           "reps": args.reps, "host_reps": args.host_reps, **card(torch), "results": res}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
