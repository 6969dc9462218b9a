"""The surface constraint (b2_pf_project_to_surface, PCDSensorUpdaterB200.projectToSurface) on the device.

  project : device time of one projectToSurface call (CUDA events on the updater's stream, median of --reps >= 50 synchronised calls, each
            on a fresh copy of the set), for 100 000 and 1 000 000 particles, on building:1000000 and on a synth.terrain of about 1M
            triangles, for a converged set (sigma 0.3 m / 5 deg around one pose on the floor) and for a set spread uniformly over the map
            (x, y over its footprint, 0.2 m over the floor, any heading);
  c3      : bench.py's C3 cycle (building:1000000, 100 000 particles: motion, sensor update with 180 beams, likelihoodStats, Gladiator
            resampling), median of --reps cycles, without and with projectToSurface after the motion and after the resampling
            (base_height 0.5 m: the particles stay at the height synth.pf_particles gives them), and the two calls' own device time.

The card name and power limit come from the same run.  Writes one JSON line to stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pf_surface.py [--reps 50]
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


def _events(torch, stream, fn, reps, setup=None):
    """median device time (ms) of fn() over reps synchronised calls; setup() runs before each, outside the events"""
    out = []
    for _ in range(reps):
        if setup:
            setup()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
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
    cfg = rmcl_b200.SurfaceConfig.defaults()
    maps = {"building:1000000": synth.building(1_000_000), "terrain:1000000": synth.terrain(1_000_000)}
    centre = {"building:1000000": (12.5, 7.5), "terrain:1000000": (12.0, 24.0)}        # a floor cell away from walls / features
    res = {"device": info, "project_ms": {}, "c3": {}}
    for name, (V, F) in maps.items():
        gm = rmcl_b200.Map(V, F, device=0)
        up = rmcl_b200.PCDSensorUpdaterB200(gm)
        up.setStream(stream.cuda_stream)
        lo, hi = V.min(0).astype(np.float64), V.max(0).astype(np.float64)
        for n in (100_000, 1_000_000):
            P0 = torch.empty((n, 8), dtype=torch.float32, device="cuda")
            A0 = torch.empty((n, 9), dtype=torch.float32, device="cuda")
            for kind in ("converged", "spread"):
                if kind == "converged":
                    cx, cy = centre[name]
                    up.initSamples(P0, A0, synth.make_transform((cx, cy, 0.2), (0.0, 0.0, 0.5)),
                                   np.diag([0.09, 0.09, 0.0, 0.0, 0.0, np.radians(5.0) ** 2]), 1)
                else:
                    up.initSamplesUniform(P0, A0, [lo[0], lo[1], 0.2, 0.0, 0.0, -np.pi], [hi[0], hi[1], 0.2, 0.0, 0.0, np.pi], 1)
                P, A = P0.clone(), A0.clone()

                def fresh():
                    P.copy_(P0); A.copy_(A0)
                up.projectToSurface(P, A, cfg)                                  # warm-up
                ms = _events(torch, stream, lambda: up.projectToSurface(P, A, cfg), args.reps, fresh)
                fresh(); up.projectToSurface(P, A, cfg); torch.cuda.synchronize()
                lost = float((A[:, 2].view(torch.int32) == 10000).float().mean())
                key = f"{name} n={n} {kind}"
                res["project_ms"][key] = {"ms": ms, "off_surface_share": lost}
                print(f"{key:42s} {ms * 1e3:9.1f} us  ({lost * 100:.2f} % off surface)", file=sys.stderr, flush=True)
        if name != "building:1000000":
            continue
        # ---- bench.py's C3 cycle, without and with the projection ----
        h = rmcl_b200.RCCB200Spherical(gm)
        m = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
        h.setTsb(synth.scenario_tsb()); h.setModel(m); h.find(synth.building_gt_pose())
        beams = synth.pf_beams(h.modelView()["points"], 180)
        Tsb = synth.scenario_tsb()
        Pn_, An_ = synth.pf_particles(100_000)
        Pi = torch.from_numpy(Pn_.view(np.float32).reshape(-1, 8).copy()).cuda()
        Ai = torch.from_numpy(An_.view(np.float32).reshape(-1, 9).copy()).cuda()
        prm, glad = rmcl_b200.PFParams.defaults(), rmcl_b200.GladiatorConfig.defaults()
        Tmo = synth.make_transform((0.02, 0.0, 0.0), (0.0, 0.0, 0.01))
        # synth.pf_particles stand 0.5 m over the floor: base_height 0.5 keeps them there, so the sensor update traces the same rays in both
        # variants.  Each variant gets its own updater (the ray mapping is chosen by timing per updater) and starts from the same set; in the
        # variant with the projection its two calls are also timed on their own.
        c3cfg = rmcl_b200.SurfaceConfig(0.5, 1.0, 0.5, 0.6, 1)
        for project in (False, True):
            uc = rmcl_b200.PCDSensorUpdaterB200(gm)
            uc.setStream(stream.cuda_stream)
            state = {"P": Pi.clone(), "A": Ai.clone(), "i": 0, "proj": []}

            def cycle():
                P, A = state["P"], state["A"]
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                uc.motionUpdate(P, A, Tmo, 0.01)
                if project:
                    ev[0].record(stream); uc.projectToSurface(P, A, c3cfg); ev[1].record(stream)
                uc.update(P, A, Tsb, beams, prm)
                uc.likelihoodStats(A)
                Pn, An = torch.empty_like(P), torch.empty_like(A)
                uc.resample(P, A, Pn, An, glad, seed=1234, step=state["i"])
                if project:
                    ev[2].record(stream); uc.projectToSurface(Pn, An, c3cfg); ev[3].record(stream)
                    state["proj"].append(ev)
                state["P"], state["A"], state["i"] = Pn, An, state["i"] + 1
            for _ in range(3):
                cycle()
            state["proj"].clear()
            ms = _events(torch, stream, cycle, args.reps)
            key = "with_projection" if project else "without_projection"
            res["c3"][key] = ms
            if project:
                proj = float(np.median([e[0].elapsed_time(e[1]) + e[2].elapsed_time(e[3]) for e in state["proj"]]))
                res["c3"]["projection_calls_ms"] = proj
                lost = float((state["A"][:, 2].view(torch.int32) == 10000).float().mean())
                res["c3"]["off_surface_share"] = lost
            print(f"C3 cycle {'with' if project else 'without'} projection: {ms:.3f} ms" +
                  (f" (the two projectToSurface calls: {proj * 1e3:.1f} us)" if project else ""), file=sys.stderr, flush=True)
    c3 = res["c3"]
    c3["projection_share"] = c3["projection_calls_ms"] / c3["with_projection"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
