"""The recovery from a kidnapping (b2_pf_recovery_observe / b2_pf_recovery_inject, PCDSensorUpdaterB200.recovery*) on the device.

  observe : device time of one recoveryObserve without read-back (CUDA events on the updater's stream: the statistics pass and the one-thread
            update), and the whole call with the state read back (host clock around the synchronising call), medians of --reps >= 50;
  inject  : the same for recoveryInject, each rep on a fresh copy of the set with p set exactly beforehand (reset and two observes of one
            particle with rates 0 and 1, outside the timing), for p in {0.01, 0.1, 1}, with the surface (SurfaceConfig.defaults()) and
            without it, max_tries 16, the map's box with roll and pitch 0 and any heading.
Both for 100 000 and 1 000 000 particles spread uniformly over the map (0.2 m over the floor, any heading), on building:1000000 and on a
synth.terrain of about 1M triangles.  The card name and power limit come from the same run.  Writes one JSON line to stdout (a table to
stderr) and nothing into the tree.

    python scripts/bench_pf_recovery.py [--reps 50]
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


def _wall(torch, fn, reps, setup=None):
    """median host time (ms) of fn(), a call that ends in a device synchronise; setup() runs before each, outside the clock"""
    out = []
    for _ in range(reps):
        if setup:
            setup()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
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
    sc = rmcl_b200.SurfaceConfig.defaults()
    rcfg = rmcl_b200.RecoveryConfig.defaults()
    exact = rmcl_b200.RecoveryConfig(0.0, 1.0)
    one = torch.zeros((1, 9), dtype=torch.float32, device="cuda")
    maps = {"building:1000000": synth.building(1_000_000), "terrain:1000000": synth.terrain(1_000_000)}
    res = {"device": info, "observe": {}, "inject": {}}
    for name, (V, F) in maps.items():
        gm = rmcl_b200.Map(V, F, device=0)
        up = rmcl_b200.PCDSensorUpdaterB200(gm)
        up.setStream(stream.cuda_stream)
        lo, hi = V.min(0).astype(np.float64), V.max(0).astype(np.float64)
        box_lo, box_hi = [lo[0], lo[1], 0.0, 0.0, 0.0, -np.pi], [hi[0], hi[1], 0.0, 0.0, 0.0, np.pi]

        def set_p(p):
            up.recoveryReset()
            one[0, 0] = 1.0
            up.recoveryObserve(one, exact)
            one[0, 0] = 1.0 - p
            up.recoveryObserve(one, exact)
        for n in (100_000, 1_000_000):
            P0 = torch.empty((n, 8), dtype=torch.float32, device="cuda")
            A0 = torch.empty((n, 9), dtype=torch.float32, device="cuda")
            up.initSamplesUniform(P0, A0, [lo[0], lo[1], 0.2, 0.0, 0.0, -np.pi], [hi[0], hi[1], 0.2, 0.0, 0.0, np.pi], 1)
            A0[:, 0] = torch.rand(n, device="cuda", generator=torch.Generator(device="cuda").manual_seed(n))
            P, A = P0.clone(), A0.clone()
            up.recoveryObserve(A, rcfg)                                        # warm-up
            key = f"{name} n={n}"
            ms = _events(torch, stream, lambda: up.recoveryObserve(A, rcfg), args.reps)
            wall = _wall(torch, lambda: up.recoveryObserve(A, rcfg, want_state=True), args.reps)
            res["observe"][key] = {"device_ms": ms, "call_ms": wall}
            print(f"observe {key:34s} device {ms * 1e3:8.1f} us   call {wall * 1e3:8.1f} us", file=sys.stderr, flush=True)
            for surface in (False, True):
                for p in (0.01, 0.1, 1.0):
                    kw = dict(surface=sc if surface else None, max_tries=16, seed=5, step=1)

                    def fresh():
                        P.copy_(P0); A.copy_(A0); set_p(p)
                    fresh(); up.recoveryInject(P, A, box_lo, box_hi, **kw)   # warm-up
                    ms = _events(torch, stream, lambda: up.recoveryInject(P, A, box_lo, box_hi, **kw), args.reps, fresh)
                    out = {}

                    def call():
                        out["r"] = up.recoveryInject(P, A, box_lo, box_hi, want_result=True, **kw)
                    wall = _wall(torch, call, args.reps, fresh)
                    r = out["r"]
                    k2 = f"{key} p={p} {'surface' if surface else 'box'}"
                    res["inject"][k2] = {"device_ms": ms, "call_ms": wall, "p": float(r["p_inject"]), "n_replaced": int(r["n_replaced"]),
                                         "n_failed": int(r["n_failed"])}
                    print(f"inject  {k2:48s} device {ms * 1e3:8.1f} us   call {wall * 1e3:8.1f} us   replaced {int(r['n_replaced']):8d}"
                          f"  failed {int(r['n_failed'])}", file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
