"""KLD-sampling on the device (b2_pf_resample_kld) at n_max = 1 000 000 slots on building:1000000, for two sets of 1 000 000 particles
weighted by one sensor update (180 beams from the true pose):

  spread    : initSamplesUniform over the whole storey (60 x 40 m, all headings), as after a global initialisation;
  converged : initSamples about the true pose with sigma 0.3 m in x, y and 5 deg in yaw, as once the filter tracks.

  call      : host wall clock around one synchronised resampleKLD call, median over --reps (>= 50), with n_particles, bins and the number
              of chunks (one host read-back each);
  kernel_us : in a separate profiled run, the device time per call of each kernel, the scans and the hash-set memsets (torch.profiler,
              CUDA activities);
  update    : the sensor update (180 beams) of the first n_particles of the resampled set against the whole n_max set, CUDA events,
              median over --reps: the saving the smaller set buys on every later cycle.

The card name and power limit come from the same run.  Writes one JSON line to stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pf_kld.py [--reps 50]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import pf_kld_ref  # noqa: E402  (the chunk schedule)
from bench_micp_chain import card  # noqa: E402

KERNELS = ("k_pf_residual_stats", "k_pf_kld_weights", "k_pf_kld_draw", "k_pf_kld_flags", "DeviceScan", "k_pf_kld_stop", "k_pf_kld_expand", "Memset")


def _events(torch, stream, fn, reps):
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream); fn(); b.record(stream)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


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
    info = card(torch)
    print(info, file=sys.stderr, flush=True)
    V, F = synth.building(1_000_000)
    gm = rmcl_b200.Map(V, F, device=0)
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gm)
    m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(m); h.find(Tgt)
    beams = synth.pf_beams(h.modelView()["points"], 180)
    up = rmcl_b200.PCDSensorUpdaterB200(gm)
    up.setStream(stream.cuda_stream)
    prm, glad, kld = rmcl_b200.PFParams.defaults(), rmcl_b200.GladiatorConfig.defaults(), rmcl_b200.KLDConfig.defaults()
    n_max = 1_000_000
    gx, gy, gz = (float(v) for v in Tgt["t"])
    lo, hi = V.min(0).astype(np.float64), V.max(0).astype(np.float64)
    P = torch.empty((n_max, 8), dtype=torch.float32, device="cuda")
    A = torch.empty((n_max, 9), dtype=torch.float32, device="cuda")
    Pn = torch.empty((n_max, 8), dtype=torch.float32, device="cuda")
    An = torch.empty((n_max, 9), dtype=torch.float32, device="cuda")
    res = {}
    for name in ("spread", "converged"):
        if name == "spread":
            up.initSamplesUniform(P, A, [lo[0], lo[1], gz, 0.0, 0.0, -np.pi], [hi[0], hi[1], gz, 0.0, 0.0, np.pi], 1)
        else:
            up.initSamples(P, A, Tgt, np.diag([0.09, 0.09, 0.0, 0.0, 0.0, math.radians(5.0) ** 2]), 1)
        up.update(P, A, Tsb, beams, prm)
        torch.cuda.synchronize()
        for _ in range(args.warmup):
            r = up.resampleKLD(P, A, Pn, An, kld, glad, seed=1, step=0)
        wall = []
        for step in range(args.reps):
            t0 = time.perf_counter()
            r = up.resampleKLD(P, A, Pn, An, kld, glad, seed=1, step=step)
            wall.append(time.perf_counter() - t0)
        call_us = float(np.median(wall)) * 1e6
        k, bins = int(r["n_particles"]), int(r["bins"])
        chunks = pf_kld_ref.chunks(kld.n_min, n_max, k)
        from torch.profiler import ProfilerActivity, profile
        n_prof = 20
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for step in range(n_prof):
                up.resampleKLD(P, A, Pn, An, kld, glad, seed=1, step=step)
        kern = {key: 0.0 for key in KERNELS}
        for e in prof.key_averages():
            for key in KERNELS:
                if key in e.key:
                    kern[key] += e.device_time_total / n_prof                       # us per call
        kern_us = sum(kern.values())
        # the next cycle's sensor update, on the resampled set (n_particles) and on the whole buffer (n_max)
        Pk, Ak = Pn[:k].clone(), An[:k].clone()
        Pf, Af = Pn.clone(), An.clone()
        up.update(Pk, Ak, Tsb, beams, prm); up.update(Pf, Af, Tsb, beams, prm)
        upd_k = _events(torch, stream, lambda: up.update(Pk, Ak, Tsb, beams, prm), args.reps)
        upd_full = _events(torch, stream, lambda: up.update(Pf, Af, Tsb, beams, prm), args.reps)
        res[name] = {"n_max": n_max, "n_particles": k, "bins": bins, "chunks": chunks, "call_us": call_us,
                     "call_us_spread": [float(np.min(wall)) * 1e6, float(np.max(wall)) * 1e6], "kernel_us": kern, "kernel_us_total": kern_us,
                     "update_ms_at_n_particles": upd_k, "update_ms_at_n_max": upd_full}
        print(f"{name:>10s}  call {call_us:9.1f} us  kernels {kern_us:8.1f} us  n_particles {k:8d}  bins {bins:7d}  chunks {chunks}  "
              f"update {upd_k:7.3f} ms at n_particles vs {upd_full:7.3f} ms at n_max", file=sys.stderr, flush=True)
        del Pk, Ak, Pf, Af
    out = {"workload": "resampleKLD at n_max = 1 000 000 on building:1000000 (suggested config; sets weighted by one 180-beam sensor update)",
           "reps": args.reps, **card(torch), "results": res}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
