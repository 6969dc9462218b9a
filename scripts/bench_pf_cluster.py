"""The filter's pose hypotheses on the device (b2_pf_cluster_stats) at n = 1 000 000 particles on building:1000000, for three sets weighted by
one sensor update (180 beams from the true pose):

  spread    : initSamplesUniform over the whole storey (60 x 40 m, all headings), as after a global initialisation;
  bimodal   : 60 % of the particles from initSamples about the true pose, 40 % about a second pose 12 m away (sigma 0.3 m, 5 deg each);
  converged : initSamples about the true pose with sigma 0.3 m in x, y and 5 deg in yaw, as once the filter tracks.

  call      : host wall clock around one synchronised estimateClusters call (default config, labels written), median over --reps (>= 50),
              with bins, n_clusters, rounds and the weight of the best hypothesis;
  kernel_us : in a separate profiled run, the device time per call of every kernel, memset and copy of the call (torch.profiler, CUDA
              activities);
  stats     : estimateStats on the same set in the same run, measured the same two ways.

The card name and power limit come from the same run.  Writes one JSON line to stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pf_cluster.py [--reps 50]
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_micp_chain import card  # noqa: E402


def _measure(torch, fn, reps, warmup):
    """-> (median wall us of one synchronised call, (min, max), device us per call by activity name)"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(warmup):
        fn()
    wall = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        wall.append(time.perf_counter() - t0)
    n_prof = 20
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            fn()
    kern = {e.key: e.device_time_total / n_prof for e in prof.key_averages() if e.device_time_total > 0}
    return float(np.median(wall)) * 1e6, [float(np.min(wall)) * 1e6, float(np.max(wall)) * 1e6], kern


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
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
    print(card(torch), file=sys.stderr, flush=True)
    V, F = synth.building(1_000_000)
    gm = rmcl_b200.Map(V, F, device=0)
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gm)
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(m); h.find(Tgt)
    beams = synth.pf_beams(h.modelView()["points"], 180)
    up = rmcl_b200.PCDSensorUpdaterB200(gm)
    up.setStream(stream.cuda_stream)
    prm, cfg = rmcl_b200.PFParams.defaults(), rmcl_b200.ClusterConfig.defaults()
    n = 1_000_000
    gx, gy, gz = (float(v) for v in Tgt["t"])
    second = synth.make_transform((gx - 12.0, gy, gz), (0.0, 0.0, math.radians(-120.0)))
    cov = np.diag([0.09, 0.09, 0.0, 0.0, 0.0, math.radians(5.0) ** 2])
    lo, hi = V.min(0).astype(np.float64), V.max(0).astype(np.float64)
    P = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    A = torch.empty((n, 9), dtype=torch.float32, device="cuda")
    labels = torch.empty((n,), dtype=torch.int32, device="cuda")
    res = {}
    for name in ("spread", "bimodal", "converged"):
        if name == "spread":
            up.initSamplesUniform(P, A, [lo[0], lo[1], gz, 0.0, 0.0, -np.pi], [hi[0], hi[1], gz, 0.0, 0.0, np.pi], 1)
        else:
            n_a = n * 6 // 10 if name == "bimodal" else n
            up.initSamples(P[:n_a], A[:n_a], Tgt, cov, 1)
            if n_a < n:
                up.initSamples(P[n_a:], A[n_a:], second, cov, 2)
        up.update(P, A, Tsb, beams, prm)
        torch.cuda.synchronize()
        out = {}

        def clusters():
            out["r"], out["recs"] = up.estimateClusters(P, A, cfg, labels)

        call_us, spread, kern = _measure(torch, clusters, args.reps, args.warmup)
        s_call_us, s_spread, s_kern = _measure(torch, lambda: up.estimateStats(P, A, max_induction_particles=n), args.reps, args.warmup)
        r, recs = out["r"], out["recs"]
        res[name] = {"n": n, "bins": int(r["bins"]), "n_clusters": int(r["n_clusters"]), "n_clustered": int(r["n_clustered"]), "rounds": int(r["rounds"]),
                     "best_weight": float(recs["weight"][0]) if len(recs) else None, "call_us": call_us, "call_us_spread": spread, "kernel_us": kern,
                     "kernel_us_total": sum(kern.values()), "stats_call_us": s_call_us, "stats_call_us_spread": s_spread, "stats_kernel_us": s_kern,
                     "stats_kernel_us_total": sum(s_kern.values())}
        print(f"{name:>10s}  call {call_us:9.1f} us  device {sum(kern.values()):8.1f} us  bins {int(r['bins']):7d}  clusters {int(r['n_clusters']):6d}  rounds {int(r['rounds'])}  "
              f"best weight {res[name]['best_weight']}  |  estimateStats call {s_call_us:8.1f} us  device {sum(s_kern.values()):7.1f} us", file=sys.stderr, flush=True)
        for key, v in sorted(kern.items(), key=lambda kv: -kv[1]):
            print(f"{'':>12s}{v:8.1f} us  {key[:110]}", file=sys.stderr, flush=True)
    print(json.dumps({"workload": "estimateClusters at n = 1 000 000 on building:1000000 (default config, labels written; sets weighted by one 180-beam sensor update)",
                      "reps": args.reps, **card(torch), "results": res}))


if __name__ == "__main__":
    main()
