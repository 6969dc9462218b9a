"""Stein variational steps of the particle set over the distance field (b2_pf_stein_update, PCDSensorUpdaterB200.steinUpdate).

On building:1000000 with its field (h 0.05 m, trunc 1 m) and 180 beams of a C3 scan, for n = 100 000 and 1 000 000 particles, n_ref in
{1024, 4096} (and 0, every particle, at 100 000), on a spread set (uniform over the building) and a converged one (N(true pose, 0.05 m,
0.02 rad)):
  call   : device time (CUDA events) of one steinUpdate of one iteration, poses restored before each call, median of --reps >= 50;
  kernels: per-kernel device time of k_pf_stein_score, k_pf_stein_bandwidth and k_pf_stein_move from torch.profiler (a separate run),
           median over the same calls;
  move   : the pair pass's FP32 instructions per pair (PAIR_INSTR, counted from stein_pair and exp_f: 16 FMAs and 14 other FP32
           operations) times n m pairs over the move's time, against the card's FP32 issue rate (128 lanes per SM per clock at the
           maximum SM clock).
The card name, power limit and maximum SM clock come from the same run.  Writes one JSON line to stdout (a table to stderr) and nothing
into the tree.

    python scripts/bench_pf_stein.py [--reps 50]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_micp_chain import card  # noqa: E402
from bench_pf_surface import _events  # noqa: E402

PAIR_INSTR = 30
KERNELS = ("k_pf_stein_score", "k_pf_stein_bandwidth", "k_pf_stein_move")


def _max_sm_clock_mhz(torch):
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        return float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def _kernel_ms(torch, fn, setup, reps):
    """median per-call device time (ms) of each Stein kernel from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    per = {k: [] for k in KERNELS}
    for _ in range(reps):
        setup()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        tot = {k: 0.0 for k in KERNELS}
        for e in prof.events():
            for k in KERNELS:
                if k in e.name and e.device_type.name == "CUDA":
                    tot[k] += e.device_time / 1e3 if hasattr(e, "device_time") else e.cuda_time / 1e3
        for k in KERNELS:
            per[k].append(tot[k])
    return {k: round(float(np.median(v)), 4) for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
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
    mhz = _max_sm_clock_mhz(torch)
    info["max_sm_clock_mhz"] = mhz if mhz else "not measured"
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    issue = 128 * n_sm * mhz * 1e6 if mhz else None              # FP32 instructions per second
    print(info, file=sys.stderr, flush=True)
    res = {"card": info, "pair_instr": PAIR_INSTR, "runs": []}

    gmap = rmcl_b200.Map(*synth.building(1_000_000))
    f = rmcl_b200.DistanceField(gmap, 0.05, 1.0)
    Tsb, Tgt = synth.scenario_tsb(), synth.building_gt_pose()
    h = rmcl_b200.RCCB200Spherical(gmap)
    sm = synth.SphericalModel(np.radians(-25.0), np.radians(40.0) / 31, 32, -np.pi, 2 * np.pi / 512, 512, 0.5, 120.0)
    h.setTsb(Tsb); h.setModel(sm); h.find(Tgt)
    beams = synth.pf_beams(h.modelView()["points"], 180)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    up.setStream(stream.cuda_stream)
    up.setDistanceField(f)
    prm = rmcl_b200.PFParams.defaults()
    prm.dist_sigma = 0.2
    yaw_gt = 2 * np.arctan2(float(Tgt["R"][2]), float(Tgt["R"][3]))

    def sets(n):
        P, _ = synth.pf_particles(n)
        yield "spread", P
        rng = np.random.default_rng(3)
        Q = synth.transforms(n)
        Q["t"] = np.asarray(Tgt["t"], np.float32)
        Q["t"][:, :2] += rng.normal(0, 0.05, (n, 2)).astype(np.float32)
        yaw = yaw_gt + rng.normal(0, 0.02, n)
        Q["R"][:, 2], Q["R"][:, 3] = np.sin(yaw / 2), np.cos(yaw / 2)
        yield "converged", Q

    for n in (100_000, 1_000_000):
        for label, P in sets(n):
            P0 = torch.from_numpy(P.view(np.float32).reshape(-1, 8).copy()).cuda()
            Pd = P0.clone()
            for n_ref in ((0, 1024, 4096) if n == 100_000 else (1024, 4096)):
                cfg = rmcl_b200.SteinConfig.defaults()
                cfg.iterations, cfg.n_ref = 1, n_ref
                m = n if n_ref == 0 else n_ref

                def call():
                    up.steinUpdate(Pd, Tsb, beams, cfg, prm, seed=1)
                for _ in range(args.warmup):
                    Pd.copy_(P0)
                    call()
                dev = _events(torch, stream, call, args.reps, setup=lambda: Pd.copy_(P0))
                ker = _kernel_ms(torch, call, lambda: Pd.copy_(P0), args.reps)
                pairs = n * m
                row = {"n": n, "set": label, "n_ref": n_ref, "m": m, "call_ms": round(dev, 4), "kernels_ms": ker,
                       "g_pairs_per_s": round(pairs / ker["k_pf_stein_move"] / 1e6, 2) if ker["k_pf_stein_move"] > 0 else None}
                if issue and ker["k_pf_stein_move"] > 0:
                    row["fp32_issue_share"] = round(PAIR_INSTR * pairs / (ker["k_pf_stein_move"] * 1e-3) / issue, 3)
                res["runs"].append(row)
                print(row, file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
