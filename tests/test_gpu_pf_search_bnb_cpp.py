"""GPU test of the C++ class's globalSearchBnB (include/rmcl_b200/rcc_b200.hpp) through tests/pf_search_bnb_cpp/pf_search_bnb_cpp.cpp: the
result and the records equal the Python path's byte for byte, and a refused min_ratio throws."""
import math
import subprocess

import numpy as np
import pytest

import native
from test_gpu_pf_search_bnb import G

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("min_ratio", [0.0, 0.5])
def test_cpp_class_matches_the_python_path(tmp_path, min_ratio):
    import rmcl_b200
    from rmcl_b200 import synth
    exe = native.adapter("pf_search_bnb_cpp")
    V, F = synth.indoor(2000)
    V, F = np.ascontiguousarray(V, np.float32), np.ascontiguousarray(F, np.uint32)
    lo, hi = V.min(0), V.max(0)
    cfg = rmcl_b200.SearchConfig(float(lo[0]), float(lo[1]), float(lo[2]) + 0.4, 0.2, int((hi[0] - lo[0]) / 0.2) + 1, int((hi[1] - lo[1]) / 0.2) + 1, 36, 8,
                                 1.0, math.radians(30.0))
    B, Tsb = G._beams(60), synth.scenario_tsb()
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as fh:
        fh.write(np.array([len(V), len(F), len(B)], np.uint32).tobytes())
        fh.write(np.array([0.05, 1.0, 0.2, min_ratio], np.float32).tobytes())
        fh.write(bytes(cfg)); fh.write(V.tobytes()); fh.write(F.tobytes()); fh.write(np.ascontiguousarray(Tsb).tobytes()); fh.write(B.tobytes())
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "REFUSED" in r.stdout and "min_ratio" in r.stdout
    raw = np.fromfile(out, np.uint8)
    res_cpp = raw[:384].view(synth.SEARCH_BNB_RESULT_DTYPE)[0]
    recs_cpp = raw[384:]
    gmap = rmcl_b200.Map(V, F)
    f = rmcl_b200.DistanceField(gmap, 0.05, 1.0)
    up = rmcl_b200.PCDSensorUpdaterB200(gmap)
    res, recs = up.globalSearchBnB(f, Tsb, B, cfg, rmcl_b200.SurfaceConfig.defaults(), G._params(0.2), min_ratio)
    assert {k: res_cpp[k].tolist() for k in ("n_candidates", "n_leaves", "n_bounded", "n_peaks", "n_records", "best_score", "threshold", "n_passes")} == \
        {k: res[k] for k in ("n_candidates", "n_leaves", "n_bounded", "n_peaks", "n_records", "best_score", "threshold", "n_passes")}
    assert recs_cpp.tobytes() == recs.tobytes() and len(recs) >= 1
