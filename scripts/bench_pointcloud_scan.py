"""A spherical sensor's scan from a PointCloud2 (b2_rcc_set_cloud_spherical) against the host path it replaces: a 128 x 2048 cloud (a
spherical scan of the 500 000-triangle indoor map at twice C2's columns, misses as NaN, FLOAT32 x, y, z at point_step 16 and 48) binned
into the C2 model (128 x 1024), two points per cell.

  host   : the C restatement of tests/pc2_scan_ref (Pc2ToScanNode::convert + fillEmpty + unpackMessage, one thread) + set_ranges, host wall
           clock ending in a synchronise.
  call   : setPointCloud with the cloud in pageable host memory, pinned host memory and device memory; host wall clock around one call, then
           a device synchronise.
  kernel : device time of k_scan_bin_cloud and k_scan_cells (torch.profiler, CUDA activities, device-memory source), and their rates against
           the bytes they must move: per point 12 B of coordinates (the cloud's point_step bytes pass through the cache lines either way, also
           reported) and an 8-byte atomic; per cell 8 B key read and reset, 12 B direction read, 4 B range, 12 B point and 1 B mask written.

Every figure is a median over --reps (>= 50) after a warm-up.  The card name and power limit come from the same run.  Writes one JSON line to
stdout (a table to stderr) and nothing into the tree.

    python scripts/bench_pointcloud_scan.py [--reps 50]
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

import pc2_scan_ref  # noqa: E402  (the host conversion)
from bench_micp_chain import card  # noqa: E402

W, H = 2048, 128
CELL_BYTES = 8 + 8 + 12 + 4 + 12 + 1


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
    gmap = rmcl_b200.Map(*synth.indoor(500_000), device=0)
    m = synth.c2_sensor()
    wide = synth.SphericalModel(m.phi_min, m.phi_inc, m.phi_size, m.theta_min, m.theta_inc / 2, 2 * m.theta_size, m.range_min, m.range_max)
    src = rmcl_b200.RCCB200Spherical(gmap)
    src.setModel(wide)
    src.find(synth.indoor_gt_pose())
    scan = src.modelView()["points"]
    n_cells = m.phi_size * m.theta_size
    res = dict(card=info, width=W, height=H, cells=n_cells, reps=args.reps)
    for ps in (16, 48):
        c = synth.pointcloud2(scan, W, H, point_step=ps, offsets=(0, 4, 8))
        h = rmcl_b200.RCCB200Spherical(gmap)
        h.setModel(m)

        def host_path():
            r = pc2_scan_ref.convert(c, m)
            h.setRanges(r["ranges"])
        row = dict(cloud_bytes=int(c.data.size), host_ms=_median_ms(host_path, args.reps, args.warmup, sync))
        srcs = dict(pageable=c.data, pinned=torch.from_numpy(c.data).pin_memory(), device=torch.from_numpy(c.data).cuda())
        for name, buf in srcs.items():
            cc = synth.PointCloud2(c.width, c.height, c.fields, False, c.point_step, c.row_step, buf)
            row[f"call_{name}_ms"] = _median_ms(lambda: h.setPointCloud(cc), args.reps, args.warmup, sync)
        cd = synth.PointCloud2(c.width, c.height, c.fields, False, c.point_step, c.row_step, srcs["device"])
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                h.setPointCloud(cd)
            sync()
        kb, kc = _kernel_us(prof, "k_scan_bin_cloud"), _kernel_us(prof, "k_scan_cells")
        row["bin_kernel_us"] = kb if kb is not None else "not measured"
        row["cells_kernel_us"] = kc if kc is not None else "not measured"
        if kb:
            row["bin_gbps_needed_bytes"] = W * H * (12 + 8) / (kb * 1e-6) / 1e9
            row["bin_gbps_cloud_bytes"] = (c.data.size + W * H * 8) / (kb * 1e-6) / 1e9
        if kc:
            row["cells_gbps"] = n_cells * CELL_BYTES / (kc * 1e-6) / 1e9
        res[f"point_step_{ps}"] = row
        print(f"point_step {ps}: " + ", ".join(f"{k} {v:.4g}" if isinstance(v, float) else f"{k} {v}" for k, v in row.items()), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
