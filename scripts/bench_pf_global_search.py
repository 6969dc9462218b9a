"""Global search of the pose over the whole map (b2_pf_global_search, PCDSensorUpdaterB200.globalSearch).

On building:1000000 with its field (h 0.05 m, trunc 1 m), the whole 60 x 40 m floor at 0.25 m x 72 headings (2.75 M candidates, the grid
through the true pose), with and without the surface rule, and 64 and 180 beams of a C3 scan at the building's true pose:
  call   : device time (CUDA events on the handle's stream) of one globalSearch, median of --reps after a warm-up call;
  kernels: per-kernel device time (k_pf_search_cells, k_pf_search_score, k_pf_search_peaks) from torch.profiler, in a separate run;
  rates  : candidates per second and beam lookups (candidates x beams) per second of the call and of the score kernel.
Also reports where record 0 lies against the true pose: at this pose the scan sees one 5 m bay, which fits the bays around it as well,
so record 0 names one of the bays that share the top score (tests/test_gpu_pf_search.py localises a pose whose beams reach the outer
walls).  The card name and power limit come from the same run.  Writes one JSON line to
stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pf_global_search.py [--reps 20]
"""
import argparse
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_micp_chain import card  # noqa: E402
from bench_pf_surface import _events  # noqa: E402

KERNELS = ("k_pf_search_cells", "k_pf_search_score", "k_pf_search_peaks")


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
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import torch
    import rmcl_b200
    from rmcl_b200 import synth
    if not torch.cuda.is_available():
        raise SystemExit("bench_pf_global_search: no GPU")
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
    cfg = rmcl_b200.SearchConfig.defaults((0.05, 0.2), (59.9, 39.9), 0.5, 0.25)      # the grid holds the true pose (31.3, 21.7)
    surface = rmcl_b200.SurfaceConfig(0.5, 1.0, 0.5, 0.6, 0)
    n_cand = cfg.nx * cfg.ny * cfg.n_yaw
    yaw_gt = 2 * math.atan2(float(Tgt["R"][2]), float(Tgt["R"][3]))
    rows = []
    for n_beams in (64, 180):
        B = synth.pf_beams(points, n_beams)
        for surf in (None, surface):
            call = lambda: up.globalSearch(field, Tsb, B, cfg, surf, prm)      # noqa: E731
            res, recs = call()                                                 # warm-up
            ms = _events(torch, stream, call, args.reps)
            kern = _kernel_ms(torch, call)
            r0 = recs[0]
            err_t = math.hypot(float(r0["pose"]["t"][0]) - float(Tgt["t"][0]), float(r0["pose"]["t"][1]) - float(Tgt["t"][1]))
            err_y = abs((2 * math.atan2(float(r0["pose"]["R"][2]), float(r0["pose"]["R"][3])) - yaw_gt + math.pi) % (2 * math.pi) - math.pi)
            rows.append({"beams": n_beams, "surface": surf is not None, "candidates": n_cand, "call_ms": round(ms, 3),
                         "kernel_ms": {k: round(v, 3) for k, v in kern.items()},
                         "candidates_per_s": n_cand / (ms * 1e-3), "lookups_per_s": n_cand * n_beams / (ms * 1e-3),
                         "score_kernel_lookups_per_s": n_cand * n_beams / (kern["k_pf_search_score"] * 1e-3) if kern["k_pf_search_score"] else None,
                         "n_valid": res["n_valid"], "n_peaks": res["n_peaks"], "record0_error_m": round(err_t, 4),
                         "record0_error_deg": round(math.degrees(err_y), 3)})
            r = rows[-1]
            print(f"beams {n_beams:4d} surface {int(r['surface'])}: call {ms:8.3f} ms  {r['candidates_per_s']:.3e} cand/s  {r['lookups_per_s']:.3e} lookups/s  "
                  f"kernels {r['kernel_ms']}  peaks {res['n_peaks']}  record 0 off by {err_t:.3f} m {math.degrees(err_y):.2f} deg", file=sys.stderr)
    print(json.dumps({"bench": "pf_global_search", **card(torch), "map": "building:1000000", "grid": [cfg.nx, cfg.ny, cfg.n_yaw], "step_m": cfg.step,
                      "reps": args.reps, "rows": rows}))


if __name__ == "__main__":
    main()
