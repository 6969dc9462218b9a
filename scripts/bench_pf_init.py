"""Particle set initialisation on the device (b2_pf_init_uniform / b2_pf_init_gaussian) against the reference's path, at 50 000 (the node's
default), 1 000 000 and 10 000 000 particles.

  device : CUDA events around one initialiser call on the handle's stream, after a warm-up; median over --reps (>= 50).  The achieved write
           bandwidth is 68 B per particle (32 B pose + 36 B attributes, nothing is read) over that time, against the H100 SXM's 3.35 TB/s.
  host   : what RmclNode::initSamplesUniform / initSamples (rmcl_ros/src/nodes/rmcl_localization.cpp:165-342) and prepareMemory (:396-430) do:
           a sequential loop over the particles on one host core (the C restatement of tests/pf_init_ref with one OpenMP thread; Philox in
           place of std::mt19937), then the copy of the set from pageable host memory to the device.  Host wall clock, ending in a
           synchronise; median over --host-reps.

The card name and power limit come from the same run.  Writes one JSON line to stdout (a table to stderr) and nothing into the tree; the
host reference is compiled into the system temporary directory.

    python scripts/bench_pf_init.py [--reps 50] [--host-reps 5]
"""
import argparse
import json
import os
import sys
import time

os.environ["OMP_NUM_THREADS"] = "1"              # the host loop of the reference is sequential

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import pf_init_ref  # noqa: E402  (the host loop)
from bench_micp_chain import card  # noqa: E402

HBM_TBPS = 3.35                                   # H100 SXM data sheet
BOX_MIN = [-50.0, -50.0, 0.0, 0.0, 0.0, -np.pi]   # the node's default box (rmcl_localization.hpp:153-154)
BOX_MAX = [50.0, 50.0, 0.0, 0.0, 0.0, np.pi]
RVIZ_COV = np.diag([0.25, 0.25, 0.0, 0.0, 0.0, 0.06853891909122467])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--host-reps", type=int, default=5)
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
    pose = synth.make_transform((10.0, -3.0, 0.0), (0.0, 0.0, 0.8))
    kinds = {
        "uniform": (lambda P, A, s: up.initSamplesUniform(P, A, BOX_MIN, BOX_MAX, s),
                    lambda n, s: pf_init_ref.init_uniform(0, n, BOX_MIN, BOX_MAX, s)),
        "gaussian": (lambda P, A, s: up.initSamples(P, A, pose, RVIZ_COV, s),
                     lambda n, s: pf_init_ref.init_gaussian(0, n, pose, RVIZ_COV, s)),
    }
    print(f"{card(torch)}", file=sys.stderr, flush=True)
    res = {}
    for n in (int(x) for x in args.sizes.split(",")):
        P = torch.empty((n, 8), dtype=torch.float32, device="cuda")
        A = torch.empty((n, 9), dtype=torch.float32, device="cuda")
        for kind, (dev_fn, host_fn) in kinds.items():
            for i in range(args.warmup):
                dev_fn(P, A, i)
            ms = []
            for i in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                dev_fn(P, A, 1000 + i)
                b.record(stream)
                b.synchronize()
                ms.append(a.elapsed_time(b))
            dev_us = float(np.median(ms)) * 1e3
            wall = []
            for i in range(args.host_reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                hp, ha = host_fn(n, 2000 + i)
                P.view(torch.uint8).reshape(-1).copy_(torch.from_numpy(hp.view(np.uint8)))
                A.view(torch.uint8).reshape(-1).copy_(torch.from_numpy(ha.view(np.uint8)))
                torch.cuda.synchronize()
                wall.append(time.perf_counter() - t0)
            host_us = float(np.median(wall)) * 1e6
            gbps = 68.0 * n / (dev_us * 1e-6) / 1e9
            res[f"{kind}_{n}"] = {"particles": n, "device_us": dev_us, "device_us_spread": [float(np.min(ms)) * 1e3, float(np.max(ms)) * 1e3],
                                  "write_GBps": gbps, "fraction_of_hbm_peak": gbps / (HBM_TBPS * 1e3), "floor_us": 68.0 * n / (HBM_TBPS * 1e12) * 1e6,
                                  "host_loop_plus_copy_us": host_us, "speedup": host_us / dev_us}
            print(f"{kind:9s} {n:>10d}  {dev_us:10.1f} us  {gbps:8.0f} GB/s ({gbps / (HBM_TBPS * 1e3) * 100:4.1f}% of {HBM_TBPS} TB/s)  "
                  f"host {host_us / 1e3:10.2f} ms", file=sys.stderr, flush=True)
        del P, A
    out = {"workload": "particle set initialisation: global uniform over the node's default box, and rviz's /initialpose covariance",
           "reps": args.reps, "host_reps": args.host_reps, "hbm_peak_TBps": HBM_TBPS, **card(torch), "results": res}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
