"""The particle filter's beams drawn from a PointCloud2 (b2_pf_sample_cloud) and the sensor update fed from it, against the host sampling it
replaces.  C3 set: 100 000 particles on the 1M-triangle building map, 180 beams; the cloud is a 128 x 1024 spherical scan (C2's model) of
that map, misses as NaN, FLOAT32 x, y, z at point_step 16 and 48, in pageable host, pinned host and device memory.

  sample       : sampleBeams(cloud, 180) -- a device cloud runs k_pf_sample_cloud and brings 68 B per sample back, a host cloud is sampled on
                 the host where the draws land.  Host wall clock around one call, then a device synchronise.
  upload       : a plain copy of the host cloud to the device (what reading a host cloud on the device would add), same clock.
  kernel       : device time of k_pf_sample_cloud (torch.profiler, CUDA activities).
  cloud update : setInput(cloud) + update(poses, attrs) of device-resident particles, same clock.
  host update  : the node-side sampling this replaces -- the cloud's x, y, z on the host (a device cloud downloaded first), synth.pf_beams'
                 seeded choice of 180 finite points -- + update(poses, attrs, beams), same clock.

Every figure is a median over --reps (>= 50) after a warm-up.  The card name and power limit come from the same run.  Writes one JSON line to
stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pf_cloud.py [--reps 50]
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

N_PARTICLES, N_SAMPLES = 100_000, 180


def _median_ms(fn, reps, warmup, sync):
    for _ in range(warmup):
        fn()
    sync()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        sync()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def _kernel_us(prof, name):
    ks = [e for e in prof.events() if e.device_type.name == "CUDA" and name in e.name]
    dur = sorted(e.device_time for e in ks) if ks and hasattr(ks[0], "device_time") else sorted(e.cuda_time for e in ks)
    return float(np.median(dur)) if dur else None


def _host_points(c):
    """x, y, z of a FLOAT32 cloud at offsets 0, 4, 8 as an (n, 3) float32 array (a device cloud is downloaded)"""
    buf = c.data.cpu().numpy() if hasattr(c.data, "cpu") else c.data
    return np.ndarray((c.width * c.height, 3), np.float32, buf, 0, (c.point_step, 4))


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
    sync = torch.cuda.synchronize
    info = card(torch)
    print(info, file=sys.stderr, flush=True)
    gmap = rmcl_b200.Map(*synth.building(1_000_000), device=0)
    m = synth.c2_sensor()
    Tsb = synth.scenario_tsb()
    src = rmcl_b200.RCCB200Spherical(gmap)
    src.setModel(m)
    src.setTsb(Tsb)
    src.find(synth.building_gt_pose())
    scan = src.modelView()["points"]
    W, H = m.theta_size, m.phi_size
    P, A = synth.pf_particles(N_PARTICLES)
    Pd = torch.from_numpy(P.view(np.float32).reshape(-1, 8).copy()).cuda()
    A0 = torch.from_numpy(A.view(np.float32).reshape(-1, 9).copy()).cuda()
    Ad = A0.clone()
    prm = rmcl_b200.PFParams.defaults()
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    up.samples, up.seed = N_SAMPLES, 12345
    res = dict(card=info, width=W, height=H, finite_points=int(np.isfinite(scan).all(1).sum()), particles=N_PARTICLES, samples=N_SAMPLES, reps=args.reps)
    for ps in (16, 48):
        c = synth.pointcloud2(scan, W, H, point_step=ps, offsets=(0, 4, 8))
        srcs = dict(pageable=c.data, pinned=torch.from_numpy(c.data).pin_memory(), device=torch.from_numpy(c.data).cuda())
        row = dict(cloud_bytes=int(c.data.size))
        dev_copy = torch.empty(c.data.size, dtype=torch.uint8, device="cuda")
        for name, buf in srcs.items():
            cc = synth.PointCloud2(c.width, c.height, c.fields, False, c.point_step, c.row_step, buf)
            row[f"sample_{name}_ms"] = _median_ms(lambda: up.sampleBeams(cc, N_SAMPLES, up.seed, 7), args.reps, args.warmup, sync)
            if name != "device":
                t = torch.from_numpy(buf) if isinstance(buf, np.ndarray) else buf
                row[f"upload_{name}_ms"] = _median_ms(lambda: dev_copy.copy_(t, non_blocking=False), args.reps, args.warmup, sync)

            def cloud_update():
                Ad.copy_(A0)
                up.setInput(cc)
                up.update(Pd, Ad, Tsb, params=prm)

            def host_update():
                Ad.copy_(A0)
                beams = synth.pf_beams(_host_points(cc), N_SAMPLES, seed=up.step)
                up.update(Pd, Ad, Tsb, beams, prm)
            row[f"cloud_update_{name}_ms"] = _median_ms(cloud_update, args.reps, args.warmup, sync)
            row[f"host_update_{name}_ms"] = _median_ms(host_update, args.reps, args.warmup, sync)
        cd = synth.PointCloud2(c.width, c.height, c.fields, False, c.point_step, c.row_step, srcs["device"])
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                up.sampleBeams(cd, N_SAMPLES, up.seed, 7)
            sync()
        k = _kernel_us(prof, "k_pf_sample_cloud")
        row["sample_kernel_us"] = k if k is not None else "not measured"
        res[f"point_step_{ps}"] = row
        print(f"point_step {ps}: " + ", ".join(f"{k} {v:.4g}" if isinstance(v, float) else f"{k} {v}" for k, v in row.items()), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
