"""Per-phase SM cycles of one k_icp_loop iteration (iteration 1, block 0) for C2 and C4, medians over repeated correctOnce calls.

Needs a library built with `make PROFILE=1` (the tail stamps and the per-block exchange stamps); select it with B2_LIB_PATH.  Phases:
  pass + block reduce      P2L pass over the thread's pairs, warp reduce-scatter, block barrier
  reduce -> publish        fixed-point conversion of the block sums and the `red` of the two limbs (median over blocks)
  publish -> collected     until all blocks' contributions have arrived (median / min / max over blocks)
  statistics               grid sums -> 15 finalised elements -> odom frame, up to the tail
  tail: merge | polar | polish | quat + t | T update | next pre-transforms
Usage: B2_LIB_PATH=... python scripts/exp_loop_phases.py [calls]"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import rmcl_b200
from rmcl_b200 import synth


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:
        return "%s (nvidia-smi: %r)" % (torch.cuda.get_device_name(0), e)


def phases(name, h, Tom, I, calls):
    lib = rmcl_b200.load_library()
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(5):
        h.correctOnce(Tom, I, 5, 0.0)
    rows = []
    out = (C.c_ulonglong * 16)()
    blk = (C.c_ulonglong * 640)()
    for _ in range(calls):
        flush.fill_(1); torch.cuda.synchronize()
        h.correctOnce(Tom, I, 5, 0.0)
        lib.b2_rcc_debug_clocks(h._h, out)
        lib.b2_rcc_debug_blocks(h._h, blk)
        o = np.array(list(out), np.uint64).astype(np.int64)         # stamps before their origin wrap around
        b = np.array(list(blk), np.uint64).astype(np.int64).reshape(160, 4)[:n_sm]
        b = b[b[:, 3] > 0]                                # blocks of this launch (grid = min(SMs, pairs / 512))
        if not o[8:16].any():
            raise SystemExit("no tail stamps: build the library with `make PROFILE=1` and select it with B2_LIB_PATH")
        tail = o[8:16]
        rows.append([o[0], np.median(b[:, 2]), np.median(b[:, 3] - b[:, 2]), (b[:, 3] - b[:, 2]).min(), (b[:, 3] - b[:, 2]).max(),
                     o[1] + o[2] - b[0, 3],              # block 0: collected -> statistics done
                     tail[2], tail[3] - tail[2], tail[4] - tail[3], tail[5] - tail[4], tail[6] - tail[5], tail[7] - tail[6],
                     o[3], o[0] + o[1] + o[2] + o[3], o[5]])
    r = np.median(np.array(rows, np.float64), axis=0)
    print("%s, iteration 1, block 0, median of %d calls (SM cycles):" % (name, calls))
    print("  pass + block reduce %d | reduce -> publish %d | publish -> collected median %d (min %d, max %d) | statistics %d"
          % tuple(r[0:6]))
    print("  tail: merge %d | polar %d | polish %d | quat + t %d | T update %d | next pre-transforms %d | whole tail %d"
          % tuple(r[6:13]))
    print("  iteration total %d | whole kernel (block 0) %d" % (r[13], r[14]))


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 30
    print("card:", card(), "| library:", os.environ.get("B2_LIB_PATH", "shipped"))
    I = synth.make_transform()
    Tsb = synth.scenario_tsb()
    V, F = synth.building(1_000_000)
    gmap = rmcl_b200.Map(V, F)
    m = synth.c2_sensor()
    h = rmcl_b200.RCCB200Spherical(gmap)
    h.setTsb(Tsb); h.setModel(m); h.setParams(1.0, 0.15)
    Tgt = synth.building_gt_pose()
    h.find(Tgt)
    h.setRanges(synth.noisy_ranges(h.modelView()["ranges"], m.range_max))
    phases("C2 (131 072 pairs)", h, synth.compose(Tgt, synth.scenario_pose_offset()), I, calls)
    V4, F4 = synth.indoor(500_000)
    map4 = rmcl_b200.Map(V4, F4)
    m4 = synth.c4_sensor()
    h4 = rmcl_b200.RCCB200Pinhole(map4)
    h4.setTsb(Tsb); h4.setModel(m4); h4.setParams(1.0, 0.15)
    T4 = synth.indoor_gt_pose()
    h4.find(T4)
    h4.setRanges(synth.noisy_ranges(h4.modelView()["ranges"], m4.range_max))
    phases("C4 (307 200 pairs)", h4, synth.compose(T4, synth.scenario_pose_offset()), I, calls)


if __name__ == "__main__":
    main()
