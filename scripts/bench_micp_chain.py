"""Chained MICP-L corrections: N host-fed b2_micp_correct_once calls against one b2_micp_correct(N), on the C2 workload of bench.py.

  (a) host : N synchronous correctOnce calls; after each the host reads Tom_new, computes the convergence progress
             (micp_localization.cpp:988-1007, the C restatement of tests/chain_ref) and enqueues the next step -- what a caller had to do before
  (b) chain: one b2_micp_correct(N): the steps follow each other on the device, one copy to the host at the end

for N = 1, 3, 10.  Reported per correction: host wall time (call to result on the host) and device time (CUDA events around the whole
sequence on the handle's stream), median over --reps repetitions, L2 flushed before each repetition (256 MiB write, as in bench.py).  The
card name and power limit come from the same run.  Writes one JSON line to stdout and nothing into the tree.

    python scripts/bench_micp_chain.py [--faces 1000000] [--reps 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (the C2 inputs: ITERATIONS, MAX_DIST, ADAPTIVE_MIN, rank_pose)
import chain_ref  # noqa: E402  (the host-side progress of the host-fed path)


def card(torch):
    out = {"device": torch.cuda.get_device_name(0), "power_limit_w": "not measured"}
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        if r.returncode == 0 and r.stdout.strip():
            out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, subprocess.SubprocessError):
        pass
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--faces", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch
    import rmcl_b200
    from rmcl_b200 import synth
    from oracle import pyoracle
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    stream = torch.cuda.current_stream()
    V, F = synth.building(args.faces)
    gmap = rmcl_b200.Map(V, F, device=0)
    m = synth.c2_sensor()
    Tsb, Tgt, I = synth.scenario_tsb(), synth.building_gt_pose(), synth.make_transform()
    h = rmcl_b200.RCCB200Spherical(gmap)
    h.setStream(stream.cuda_stream)
    h.setTsb(Tsb)
    h.setModel(m)
    h.setParams(bench.MAX_DIST, bench.ADAPTIVE_MIN)
    h.find(Tgt)
    h.setRanges(synth.noisy_ranges(h.modelView()["ranges"], m.range_max))
    valid = int(h.datasetView()["mask"].astype(bool).sum())
    Tom0 = bench.rank_pose(synth, 0)
    Tbo = np.stack([I])
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    its = bench.ITERATIONS

    def host_fed(n):
        T, cp = Tom0, 0.0
        for _ in range(n):
            Tn, Td, Cm = rmcl_b200.micp_correct_once([h], Tbo, T, its, cp)
            cp = chain_ref.oracle_progress(pyoracle, T, Td, int(Cm["n_meas"]), valid, True)
            T = Tn
        return T, cp

    def chained(n):
        T, cp, _ = rmcl_b200.micp_correct([h], Tbo, Tom0, n_corrections=n, iterations=its)
        return T, cp

    res = {}
    for n in (1, 3, 10):
        for name, fn in (("host", host_fed), ("chain", chained)):
            for _ in range(args.warmup):
                fn(n)
            wall, dev = [], []
            for _ in range(args.reps):
                flush.fill_(1)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                a.record(stream)
                fn(n)
                b.record(stream)
                t1 = time.perf_counter()
                b.synchronize()
                wall.append((t1 - t0) / n * 1e6)
                dev.append(a.elapsed_time(b) / n * 1e3)
            res[f"{name}_N{n}"] = {"host_wall_us_per_correction": float(np.median(wall)), "device_us_per_correction": float(np.median(dev)),
                                   "host_wall_us_spread": [float(np.min(wall)), float(np.max(wall))]}
        # both paths compute the same chain (the host-fed one feeds the chain's own progress formula)
        Ta, cpa = host_fed(n)
        Tb, cpb = chained(n)
        res[f"same_result_N{n}"] = bool(Ta.tobytes() == Tb.tobytes() and np.float32(cpa) == np.float32(cpb))
    out = {"workload": "C2 (128x1024 spherical scan, building mesh), chained correctOnce, %d inner iterations" % its, "faces": args.faces,
           "reps": args.reps, "l2": "flushed before each repetition (256 MiB write)", **card(torch), "results": res}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
