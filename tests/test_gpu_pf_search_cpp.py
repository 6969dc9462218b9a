"""GPU test of the C++ class's globalSearch (include/rmcl_b200/rcc_b200.hpp) through tests/pf_search_cpp/pf_search_cpp.cpp: the result, the
records and the likelihood map equal the Python path's byte for byte, and a refused config throws."""
import math
import subprocess

import numpy as np
import pytest

import native
import test_gpu_pf_search as G

pytestmark = pytest.mark.gpu


def test_cpp_class_matches_the_python_path(tmp_path):
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    exe = native.adapter("pf_search_cpp")
    V, F = synth.indoor(2000)
    V, F = np.ascontiguousarray(V, np.float32), np.ascontiguousarray(F, np.uint32)
    lo, hi = V.min(0), V.max(0)
    cfg = rmcl_b200.SearchConfig(float(lo[0]), float(lo[1]), float(lo[2]) + 0.4, 0.2, int((hi[0] - lo[0]) / 0.2) + 1, int((hi[1] - lo[1]) / 0.2) + 1, 36, 8,
                                 1.0, math.radians(30.0))
    B, Tsb = G._beams(60), synth.scenario_tsb()
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as fh:
        fh.write(np.array([len(V), len(F), len(B)], np.uint32).tobytes())
        fh.write(np.array([0.05, 1.0, 0.2], np.float32).tobytes())
        fh.write(bytes(cfg)); fh.write(V.tobytes()); fh.write(F.tobytes()); fh.write(np.ascontiguousarray(Tsb).tobytes()); fh.write(B.tobytes())
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "REFUSED" in r.stdout and "max_records" in r.stdout
    raw = np.fromfile(out, np.uint8)
    res_cpp = raw[:32].view(np.uint64)
    n_rec = int(res_cpp[3])
    recs_cpp, scores_cpp = raw[32:32 + 48 * n_rec], raw[32 + 48 * n_rec:]
    gmap = rmcl_b200.Map(V, F)
    f = rmcl_b200.DistanceField(gmap, 0.05, 1.0)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    S = torch.empty(cfg.nx * cfg.ny * cfg.n_yaw, dtype=torch.float32, device="cuda")
    res, recs = up.globalSearch(f, Tsb, B, cfg, rmcl_b200.SurfaceConfig.defaults(), G._params(0.2), S)
    assert [int(x) for x in res_cpp] == [res["n_candidates"], res["n_valid"], res["n_peaks"], res["n_records"]]
    assert recs_cpp.tobytes() == recs.tobytes()
    assert scores_cpp.tobytes() == S.cpu().numpy().tobytes()
    assert res["n_valid"] > 0 and n_rec >= 1
