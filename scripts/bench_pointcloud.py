"""An O1Dn sensor's scan from an organised PointCloud2 (b2_rcc_set_cloud_o1dn) against the host path it replaces, on a 128 x 1024 cloud (a
spherical scan of the 500 000-triangle indoor map, misses as NaN) with point_step 16 and 48 (FLOAT32 x, y, z).

  host   : the conversion on the host (the numpy restatement of tests/pc2_ref, vectorised, so faster than the reference's per-point loop)
           + set_model_o1dn + set_ranges, host wall clock ending in a synchronise.
  call   : setPointCloud with the cloud in pageable host memory, pinned host memory and device memory; host wall clock around one call, then
           a device synchronise.
  kernel : device time of k_o1dn_from_cloud (torch.profiler, CUDA activities, device-memory source, a run of its own), and its rate against
           the bytes it must move: 12 B of coordinates read and 29 B written (direction 12, range 4, point 12, mask 1) per ray.
  find   : find time (CUDA events of correctOnce) of consecutive scans alternating between two poses: a handle fed by setPointCloud keeps its
           tile schedule, one fed by set_model_o1dn + set_ranges starts every scan from the identity order.

Every figure is a median over --reps (>= 50) after a warm-up.  The card name and power limit come from the same run.  Writes one JSON line to
stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pointcloud.py [--reps 50]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import pc2_ref  # noqa: E402  (the host conversion)
from bench_micp_chain import card  # noqa: E402

W, H = 1024, 128
BYTES_PER_RAY = 12 + 29


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if args.reps < 50:
        raise SystemExit("--reps must be at least 50")
    import torch
    import rmcl_b200
    from rmcl_b200 import O1DnCloudFilter, synth
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    sync = torch.cuda.synchronize
    info = card(torch)
    print(info, file=sys.stderr, flush=True)
    gmap = rmcl_b200.Map(*synth.indoor(500_000), device=0)
    m = synth.c2_sensor()
    sph = rmcl_b200.RCCB200Spherical(gmap)
    sph.setModel(m)
    poses = [synth.indoor_gt_pose(), synth.compose(synth.indoor_gt_pose(), synth.make_transform((0.05, 0.02, 0.0), (0.0, 0.0, 0.01)))]
    scans = []
    for T in poses:
        sph.find(T)
        scans.append(sph.modelView()["points"])
    flt = O1DnCloudFilter.defaults(0.3, 50.0)
    Tguess = synth.compose(poses[0], synth.make_transform((0.1, -0.05, 0.0), (0.0, 0.0, 0.02)))
    I = synth.make_transform()
    res = dict(card=info, width=W, height=H, reps=args.reps)
    for ps in (16, 48):
        clouds = [synth.pointcloud2(p, W, H, point_step=ps, offsets=(0, 4, 8)) for p in scans]
        c = clouds[0]
        h = rmcl_b200.RCCB200O1Dn(gmap)

        def host_path():
            r = pc2_ref.convert_np(c, flt)
            h.setModel(synth.O1DnModel(r["width"], r["height"], np.zeros(3, np.float32), r["dirs"], flt.range_min, flt.range_max))
            h.setRanges(r["ranges"])
        row = dict(cloud_bytes=int(c.data.size), host_ms=_median_ms(host_path, args.reps, args.warmup, sync))
        srcs = dict(pageable=c.data, pinned=torch.from_numpy(c.data).pin_memory(), device=torch.from_numpy(c.data).cuda())
        for name, buf in srcs.items():
            cc = synth.PointCloud2(c.width, c.height, c.fields, False, c.point_step, c.row_step, buf)
            row[f"call_{name}_ms"] = _median_ms(lambda: h.setPointCloud(cc, flt), args.reps, args.warmup, sync)
        cd = synth.PointCloud2(c.width, c.height, c.fields, False, c.point_step, c.row_step, srcs["device"])
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                h.setPointCloud(cd, flt)
            sync()
        ks = [e for e in prof.events() if e.device_type.name == "CUDA" and "k_o1dn_from_cloud" in e.name]
        dur = sorted(e.device_time for e in ks) if ks and hasattr(ks[0], "device_time") else sorted(e.cuda_time for e in ks)
        row["kernel_us"] = float(np.median(dur)) if dur else "not measured"
        if dur:
            row["kernel_gbps"] = W * H * BYTES_PER_RAY / (row["kernel_us"] * 1e-6) / 1e9
        # find time over consecutive scans: schedule kept (cloud path) vs reset every scan (table path)
        keep, reset = rmcl_b200.RCCB200O1Dn(gmap), rmcl_b200.RCCB200O1Dn(gmap)
        keep.enableTiming(True)
        reset.enableTiming(True)
        tables = [pc2_ref.convert_np(x, flt) for x in clouds]
        fk, fr = [], []
        for it in range(args.reps + args.warmup):
            k = it % 2
            keep.setPointCloud(clouds[k], flt)
            reset.setModel(synth.O1DnModel(W, H, np.zeros(3, np.float32), tables[k]["dirs"], flt.range_min, flt.range_max))
            reset.setRanges(tables[k]["ranges"])
            keep.correctOnce(Tguess, I, 5, 0.0)
            reset.correctOnce(Tguess, I, 5, 0.0)
            if it >= args.warmup:
                fk.append(keep.lastTiming()[0] * 1e3)
                fr.append(reset.lastTiming()[0] * 1e3)
        row["find_kept_us"], row["find_reset_us"] = float(np.median(fk)), float(np.median(fr))
        res[f"point_step_{ps}"] = row
        print(f"point_step {ps}: " + ", ".join(f"{k} {v:.4g}" if isinstance(v, float) else f"{k} {v}" for k, v in row.items()), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
