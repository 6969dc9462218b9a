"""Branch-and-bound global search (b2_pf_global_search_bnb, PCDSensorUpdaterB200.globalSearchBnB) against the exhaustive one
(b2_pf_global_search) on the same inputs.

On building:1000000 with its field (h 0.05 m, trunc 1 m), a C3 scan at the building's true pose with 64 and 180 beams, with and without the
surface rule, over two grids of the whole 60 x 40 m floor: 0.25 m x 72 headings (2.75 M candidates) and 0.05 m x 360 headings (3.5e8); and,
for the new call only, 200 x 200 x 32768 cells at 0.25 m (1.3e9 candidates, above the exhaustive call's 2^30).  Per workload:
  call   : device time (CUDA events on the handle's stream) of each call, median of --reps, the two calls alternating after a warm-up of each;
  kernels: per-kernel device time (the pyramid build, the bound, the leaves, the peaks; the exhaustive call's score kernel) from
           torch.profiler in a separate run;
  search : nodes bounded per tree level and leaves scored as fractions of the candidates, the passes, s* and tau;
  equal  : whether the new call's records equal the exhaustive call's byte for byte (min_ratio 0).
The card name and power limit come from the same run.  Writes one JSON line to stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pf_global_search_bnb.py [--reps 5] [--no-fine] [--no-huge]
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

KERNELS = ("k_pf_bnb_pyr", "k_pf_bnb_bound", "k_pf_bnb_leaves", "k_pf_bnb_peaks", "k_pf_search_score", "k_pf_search_peaks")


def _kernel_ms(torch, fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {k: 0.0 for k in KERNELS}
    for e in prof.events():
        for k in KERNELS:
            if k in e.name and e.device_type.name == "CUDA":
                tot[k] += (e.device_time if hasattr(e, "device_time") else e.cuda_time) / 1e3
    return {k: round(v, 3) for k, v in tot.items() if v}


def _time(torch, stream, fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    out = fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-fine", action="store_true", help="leave out the 0.05 m x 360 grid")
    ap.add_argument("--no-huge", action="store_true", help="leave out the grid above 2^30 candidates")
    args = ap.parse_args()
    import torch
    import rmcl_b200
    from rmcl_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_pf_global_search_bnb: no GPU")
    V, F = synth.building(1_000_000)
    gmap = rmcl_b200.Map(V, F, device=0)
    field = rmcl_b200.DistanceField(gmap, 0.05, 1.0)
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gmap)
    h.setTsb(Tsb)
    h.setModel(synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0))
    h.find(Tgt)
    points = h.modelView()["points"]
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    stream = torch.cuda.current_stream()
    up.setStream(stream.cuda_stream)
    prm = rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.2
    surface = rmcl_b200.SurfaceConfig(0.5, 1.0, 0.5, 0.6, 0)
    grids = [("0.25m x 72", rmcl_b200.SearchConfig.defaults((0.05, 0.2), (59.9, 39.9), 0.5, 0.25))]
    if not args.no_fine:
        fine = rmcl_b200.SearchConfig.defaults((0.05, 0.2), (59.9, 39.9), 0.5, 0.05)
        fine.n_yaw = 360
        grids.append(("0.05m x 360", fine))
    huge = rmcl_b200.SearchConfig(5.0, 5.0, 0.5, 0.25, 200, 200, 32768, 8, 1.0, np.radians(30.0))
    rows = []
    for name, cfg in grids + ([] if args.no_huge else [("200x200 x 32768", huge)]):
        n_cand = cfg.nx * cfg.ny * cfg.n_yaw
        for n_beams in (64, 180):
            B = synth.pf_beams(points, n_beams)
            for surf in (None, surface):
                exh = n_cand <= 1 << 30
                call_x = lambda: up.globalSearch(field, Tsb, B, cfg, surf, prm)                 # noqa: E731
                call_b = lambda: up.globalSearchBnB(field, Tsb, B, cfg, surf, prm, 0.0)         # noqa: E731
                res_b, recs_b = call_b()
                equal = None
                if exh:
                    res_x, recs_x = call_x()
                    equal = recs_b.tobytes() == recs_x.tobytes() and res_b["n_records"] == res_x["n_records"]
                tb, tx = [], []
                for _ in range(args.reps):
                    tb.append(_time(torch, stream, call_b)[0])
                    if exh:
                        tx.append(_time(torch, stream, call_x)[0])
                kb = _kernel_ms(torch, call_b)
                kx = _kernel_ms(torch, call_x) if exh else None
                ms_b = float(np.median(tb))
                ms_x = float(np.median(tx)) if exh else None
                d = res_b["depth"]
                rows.append({"grid": name, "cells": [cfg.nx, cfg.ny, cfg.n_yaw], "candidates": n_cand, "beams": n_beams, "surface": surf is not None,
                             "bnb_ms": round(ms_b, 3), "exhaustive_ms": None if ms_x is None else round(ms_x, 3),
                             "speedup": None if ms_x is None else round(ms_x / ms_b, 2), "records_equal": equal,
                             "bnb_kernel_ms": kb, "exhaustive_kernel_ms": kx, "passes": res_b["n_passes"], "depth": d,
                             "bounded_per_level_frac": [res_b["n_level"][lv] / n_cand for lv in range(d, 0, -1)],
                             "leaves_frac": res_b["n_leaves"] / n_cand, "bounded_per_pass": res_b["n_bounded_pass"],
                             "best_score": res_b["best_score"], "threshold": res_b["threshold"], "n_records": res_b["n_records"]})
                r = rows[-1]
                print(f"{name:16s} beams {n_beams:4d} surface {int(r['surface'])}: bnb {ms_b:9.2f} ms  exhaustive {ms_x}  equal {equal}  passes {r['passes']}  "
                      f"leaves {r['leaves_frac']:.2e}  levels {[f'{v:.1e}' for v in r['bounded_per_level_frac']]}  kernels {kb}", file=sys.stderr)
    print(json.dumps({"bench": "pf_global_search_bnb", **card(torch), "map": "building:1000000", "field": {"h": 0.05, "trunc": 1.0},
                      "reps": args.reps, "rows": rows}))


if __name__ == "__main__":
    main()
