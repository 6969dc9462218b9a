"""The MICP-L pose covariance on the device (b2_micp_pose_covariance) after a correction, beside the correction itself:

  c2_building : C2 (128 x 1024 spherical) over building:1000000 at the bench pose, 1 cm range noise;
  c4_indoor   : C4 (640 x 480 depth camera) over indoor:500000.

  call      : host wall clock around one synchronised micp_pose_covariance call, median over --reps (>= 50);
  kernel_us : in a separate profiled run, the device time per call of every kernel and copy of the call (torch.profiler, CUDA activities);
  bytes     : 38 B per correspondence read by k_micp_information (two mask bytes and three float triples), over its kernel time, against the
              H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s (the buffers are likely still in L2 after the correction);
  correct   : micp_correct_once (5 iterations) on the same handle, measured the same two ways.

The card name and power limit come from the same run.  Writes one JSON line to stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_micp_cov.py [--reps 50]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_micp_chain import card  # noqa: E402
from bench_pf_cluster import _measure  # noqa: E402

BYTES_PER_PAIR = 38
HBM_BPS = 3.35e12


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
    print(card(torch), file=sys.stderr, flush=True)
    cases = {
        "c2_building": (synth.building(1_000_000), synth.c2_sensor(), rmcl_b200.RCCB200Spherical, synth.building_gt_pose()),
        "c4_indoor": (synth.indoor(500_000), synth.c4_sensor(), rmcl_b200.RCCB200Pinhole, synth.indoor_gt_pose()),
    }
    res = {}
    I = np.stack([synth.make_transform()])
    for name, ((V, F), m, cls, Tgt) in cases.items():
        gm = rmcl_b200.Map(V, F, device=0)
        h = cls(gm)
        Tsb = synth.scenario_tsb()
        h.setTsb(Tsb); h.setModel(m); h.setParams(1.0, 0.15)
        h.find(Tgt)
        mv = h.modelView()
        r = np.where(mv["hits"] > 0, mv["ranges"], np.float32(m.range_max + 1.0)).astype(np.float32)
        h.setRanges(synth.noisy_ranges(r, m.range_max, seed=3))
        Tom = synth.compose(Tgt, synth.scenario_pose_offset())
        _, Td, _ = rmcl_b200.micp_correct_once([h], I, Tom, 5, 0.0)
        torch.cuda.synchronize()
        out = {}

        def cov():
            out["rec"] = rmcl_b200.micp_pose_covariance([h], I, Td, 0.0)

        call_us, spread, kern = _measure(torch, cov, args.reps, args.warmup)
        c_call_us, c_spread, c_kern = _measure(torch, lambda: rmcl_b200.micp_correct_once([h], I, Tom, 5, 0.0), args.reps, args.warmup)
        rec = out["rec"]
        k_us = next((v for k, v in kern.items() if "k_micp_information" in k), None)
        n_corr = int(np.asarray(mv["hits"]).size)
        gbps = BYTES_PER_PAIR * n_corr / (k_us * 1e-6) / 1e9 if k_us else None
        res[name] = {"correspondences": n_corr, "pairs": int(rec["n_pairs"][0]), "n_degenerate": int(rec["n_degenerate"]),
                     "call_us": call_us, "call_us_spread": spread, "kernel_us": kern, "kernel_us_total": sum(kern.values()),
                     "k_micp_information_us": k_us, "read_GBps": gbps, "share_of_hbm": gbps * 1e9 / HBM_BPS if gbps else None,
                     "correct_once_call_us": c_call_us, "correct_once_call_us_spread": c_spread, "correct_once_kernel_us_total": sum(c_kern.values())}
        print(f"{name:>12s}  call {call_us:8.1f} us  kernel {k_us or 0:7.1f} us  {gbps or 0:7.1f} GB/s ({BYTES_PER_PAIR} B x {n_corr})  pairs {int(rec['n_pairs'][0])}  |  "
              f"correctOnce call {c_call_us:8.1f} us  device {sum(c_kern.values()):8.1f} us", file=sys.stderr, flush=True)
        for key, v in sorted(kern.items(), key=lambda kv: -kv[1]):
            print(f"{'':>14s}{v:8.1f} us  {key[:110]}", file=sys.stderr, flush=True)
    print(json.dumps({"workload": "micp_pose_covariance after micp_correct_once (5 iterations): C2 on building:1000000, C4 on indoor:500000",
                      "reps": args.reps, **card(torch), "results": res}))


if __name__ == "__main__":
    main()
