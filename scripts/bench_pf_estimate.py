"""The particle set's pose estimate on the device (b2_pf_estimate_stats) against the reference's path, at 50 000 (the node's default
max_induction_particles), 1 000 000 and 10 000 000 particles, the whole set being the induction slice.

  device : host wall clock around one synchronised estimateStats call (two kernels, the 440-byte copy, the synchronise), median over --reps
           (>= 50); and, in a separate profiled run, the device time of k_pf_estimate_moments and k_pf_estimate_cov (torch.profiler, CUDA
           activities, mean per call).  Read bandwidth: two passes of 36 B per particle (the 32 B pose and the 4 B likelihood.mean) over the
           kernel time, against the H100 SXM's 3.35 TB/s; the attributes are 36-byte records, so each 4-byte read touches its own 32-byte
           sector and the bytes moved are about 68 per particle and pass.
  host   : what RmclNode::estimateStats (rmcl_ros/src/nodes/rmcl_localization.cpp:642-731) with prepareMemory (:396-430) costs: the copy of the
           whole set to the host, the host loop (the float64 numpy restatement of tests/pf_estimate_ref), and the copy back to the device for
           the next GPU step.  Host wall clock ending in a synchronise, median over --host-reps.

The card name and power limit come from the same run.  Writes one JSON line to stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pf_estimate.py [--reps 50] [--host-reps 3]
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

import pf_estimate_ref  # noqa: E402  (the host loop)
from bench_micp_chain import card  # noqa: E402

HBM_TBPS = 3.35                                   # H100 SXM data sheet
KERNELS = ("k_pf_estimate_moments", "k_pf_estimate_cov")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sizes", default="50000,1000000,10000000")
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
    print(f"{card(torch)}", file=sys.stderr, flush=True)
    res = {}
    for n in (int(x) for x in args.sizes.split(",")):
        P = torch.empty((n, 8), dtype=torch.float32, device="cuda")
        A = torch.empty((n, 9), dtype=torch.float32, device="cuda")
        up.initSamples(P, A, synth.make_transform((10.0, -3.0, 0.0), (0.0, 0.0, 0.8)), np.diag([0.25, 0.25, 0.0, 0.0, 0.0, 0.07]), 1)
        A[:, 0] = torch.rand(n, device="cuda", generator=torch.Generator("cuda").manual_seed(2))         # likelihoods in [0, 1)
        torch.cuda.synchronize()
        for _ in range(args.warmup):
            up.estimateStats(P, A, n)
        wall = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            up.estimateStats(P, A, n)
            wall.append(time.perf_counter() - t0)
        call_us = float(np.median(wall)) * 1e6
        from torch.profiler import ProfilerActivity, profile
        n_prof = 20
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_prof):
                up.estimateStats(P, A, n)
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
            pf_estimate_ref.estimate_np(hp, ha)                                       # the host loop
            P.copy_(torch.from_numpy(hp.view(np.float32).reshape(n, 8)))              # prepareMemory("gpu")
            A.copy_(torch.from_numpy(ha.view(np.float32).reshape(n, 9)))
            torch.cuda.synchronize()
            hw.append(time.perf_counter() - t0)
        host_us = float(np.median(hw)) * 1e6
        gbps = 2 * 36.0 * n / (kern_us * 1e-6) / 1e9 if kern_us > 0 else float("nan")
        res[str(n)] = {"particles": n, "call_us": call_us, "call_us_spread": [float(np.min(wall)) * 1e6, float(np.max(wall)) * 1e6],
                       "kernel_us": kern, "read_GBps_36B": gbps, "fraction_of_hbm_peak": gbps / (HBM_TBPS * 1e3),
                       "floor_us_36B": 2 * 36.0 * n / (HBM_TBPS * 1e12) * 1e6, "floor_us_68B": 2 * 68.0 * n / (HBM_TBPS * 1e12) * 1e6,
                       "reference_copy_loop_copy_us": host_us, "speedup": host_us / call_us}
        print(f"{n:>10d}  call {call_us:9.1f} us  kernels {kern[KERNELS[0]]:8.1f} + {kern[KERNELS[1]]:8.1f} us  {gbps:7.0f} GB/s "
              f"({gbps / (HBM_TBPS * 1e3) * 100:4.1f}% of {HBM_TBPS} TB/s at 36 B)  reference {host_us / 1e3:10.2f} ms", file=sys.stderr, flush=True)
        del P, A
    out = {"workload": "estimateStats over the whole set (initSamples with rviz's covariance, likelihoods uniform in [0, 1))",
           "reps": args.reps, "host_reps": args.host_reps, "hbm_peak_TBps": HBM_TBPS, **card(torch), "results": res}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
