"""The truncated distance field (b2_dfield_*, rmcl_b200.DistanceField) and the particle filter's sensor update from it
(b2_pf_sensor_update_field, PCDSensorUpdaterB200.setDistanceField).

  build  : wall time of b2_dfield_create (classify, scan, fill, synchronise; the handle's build_ms), bricks allocated and bytes resident, on
           building:1000000 and on a synth.terrain of about 1M triangles, for h in {0.05, 0.1} m and trunc in {1, 6} m (box: the map's
           grown by trunc);
  query  : b2_dfield_query of 10^6 random points in the building's field box, device tensors: device time (CUDA events) and the whole
           synchronised call, medians of --reps >= 50 after warm-up;
  update : C3, 100 000 particles spread over building:1000000 x 180 beams of a scan, device particles: ray casting (correspondence 0),
           closest point (1) and the field (h 0.05 / trunc 1 and h 0.1 / trunc 6): device time (CUDA events) and the whole synchronised
           update() (host clock), medians of --reps >= 50 after warm-up.
The card name and power limit come from the same run.  Writes one JSON line to stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pf_dfield.py [--reps 50]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_micp_chain import card  # noqa: E402
from bench_pf_surface import _events  # noqa: E402


def _wall(torch, fn, reps):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(out))


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
    res = {"card": info, "build": [], "query": {}, "update": {}}

    maps = {"building:1000000": rmcl_b200.Map(*synth.building(1_000_000)), "terrain": rmcl_b200.Map(*synth.terrain(1_000_000))}
    for name, m in maps.items():
        for h in (0.05, 0.1):
            for trunc in (1.0, 6.0):
                f = rmcl_b200.DistanceField(m, h, trunc)
                i = f.info()
                row = {"map": name, "h": h, "trunc": trunc, "build_ms": round(i["build_ms"], 2), "bricks": i["bricks_allocated"],
                       "bricks_total": i["bricks_total"], "mib": round(i["bytes"] / 2 ** 20, 1)}
                res["build"].append(row)
                print(row, file=sys.stderr, flush=True)
                f.close()
                torch.cuda.synchronize()

    gmap = maps["building:1000000"]
    f = rmcl_b200.DistanceField(gmap, 0.05, 1.0)
    i = f.info()
    lo = np.asarray(i["origin"], np.float64)
    hi = lo + (np.asarray(i["dims"]) - 1) * i["resolution"]
    pts = torch.from_numpy(np.random.default_rng(1).uniform(lo, hi, (1_000_000, 3)).astype(np.float32)).cuda()
    for _ in range(args.warmup):
        f.query(pts)
    dev = _events(torch, stream, lambda: f.query(pts), args.reps)
    wall = _wall(torch, lambda: f.query(pts), args.reps)
    res["query"] = {"n": 1_000_000, "device_ms": round(dev, 4), "call_ms": round(wall, 4), "g_queries_per_s": round(1e6 / dev / 1e6, 2)}
    print("query", res["query"], file=sys.stderr, flush=True)

    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gmap)
    sm = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(sm); h.find(Tgt)
    beams = synth.pf_beams(h.modelView()["points"], 180)
    P, A = synth.pf_particles(100_000)
    Pd = torch.from_numpy(P.view(np.float32).reshape(-1, 8).copy()).cuda()
    A0 = torch.from_numpy(A.view(np.float32).reshape(-1, 9).copy()).cuda()
    Ad = A0.clone()
    fields = {"field_h0.05_t1": f, "field_h0.1_t6": rmcl_b200.DistanceField(gmap, 0.1, 6.0)}
    arms = [("ray_casting", 0, None), ("closest_point", 1, None)] + [(k, 0, v) for k, v in fields.items()]
    for label, corr, fld in arms:
        up = rmcl_b200.PCDSensorUpdaterB200(gmap)
        up.setStream(stream.cuda_stream)
        up.setDistanceField(fld)
        prm = rmcl_b200.PFParams.defaults(correspondence_type=corr)

        def run():
            Ad.copy_(A0)
            up.update(Pd, Ad, Tsb, beams, prm)
        for _ in range(args.warmup):
            run()
        dev = _events(torch, stream, lambda: up.update(Pd, Ad, Tsb, beams, prm), args.reps, setup=lambda: Ad.copy_(A0))
        wall = _wall(torch, lambda: up.update(Pd, Ad, Tsb, beams, prm), args.reps)
        res["update"][label] = {"device_ms": round(dev, 3), "call_ms": round(wall, 3), "g_beams_per_s": round(100_000 * 180 / dev / 1e6, 2)}
        print(label, res["update"][label], file=sys.stderr, flush=True)
        up.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
