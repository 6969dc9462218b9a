"""GPU tests of the bindings' argument check: the C ABI takes one count for a call's arrays, so both bindings refuse arrays that disagree in
length before anything runs.

* Python (rmcl_b200/api.py): update (map, distance field and host paths), motionUpdate and resample with one real array one record short.
  Each short tensor is a slice of a full one, so a kernel that indexed it with the other arrays' count would change the bytes after it: the
  call raises ValueError, no kernel is launched, every array keeps its bytes and no CUDA error is left behind.  The same calls with arrays
  that agree then run.
* C++ (include/rmcl_b200/rcc_b200.hpp): tests/pf_args_cpp calls every PCDSensorUpdaterB200 entry point that passes one count for poses and
  attributes with mismatched views (std::invalid_argument, no launch) and with matched ones (runs)."""
import subprocess

import numpy as np
import pytest

from conftest import gpu_map
import native

N = 1000


def _case():
    """a cube map, an updater, beams and the full particle tensors: poses and attrs, the resampling's outputs, raw draws and normals"""
    import rmcl_b200
    import torch
    from rmcl_b200 import synth
    up = rmcl_b200.PCDSensorUpdaterB200(gpu_map("cube29"))
    P, A = synth.pf_particles(N, footprint=(16.0, 16.0), z=0.0, margin=0.0)
    P["t"][:, :2] -= 8.0
    beams = np.zeros(8, synth.RANGE_MEAS_DTYPE)
    beams["dir"][:, 0], beams["range"] = 1.0, 5.0
    dev = lambda a, k: torch.from_numpy(a.view(np.float32).reshape(-1, k).copy()).cuda()
    t = {"poses": dev(P, 8), "attrs": dev(A, 9), "poses_new": dev(P, 8), "attrs_new": dev(A, 9),
         "raw": torch.zeros(N, dtype=torch.int32, device="cuda"), "normals": torch.zeros((N, 6), dtype=torch.float32, device="cuda")}
    return up, beams, synth.scenario_tsb(), t, (P, A)


def _short(t, name):
    """the tensors with `name` one record short"""
    return {k: v[:-1] if k == name else v for k, v in t.items()}


CALLS = {
    "update": lambda up, beams, tsb, x: up.update(x["poses"], x["attrs"], tsb, beams),
    "update_field": lambda up, beams, tsb, x: up.update(x["poses"], x["attrs"], tsb, beams),
    "motionUpdate": lambda up, beams, tsb, x: up.motionUpdate(x["poses"], x["attrs"], tsb, 0.01),
    "resample": lambda up, beams, tsb, x: up.resample(x["poses"], x["attrs"], x["poses_new"], x["attrs_new"], raw=x["raw"], normals=x["normals"]),
}
SHORT = {"update": ("poses", "attrs"), "update_field": ("poses", "attrs"), "motionUpdate": ("poses", "attrs"),
         "resample": ("poses", "attrs", "poses_new", "attrs_new", "raw", "normals")}


@pytest.mark.gpu
@pytest.mark.parametrize("call", sorted(CALLS))
def test_python_mismatch_is_refused_before_anything_runs(call):
    import rmcl_b200
    import torch
    up, beams, tsb, t, _ = _case()
    if call == "update_field":
        up.setDistanceField(rmcl_b200.DistanceField(up.map, 0.25, 1.0))
    lib = rmcl_b200.load_library()
    torch.cuda.synchronize()
    before = {k: v.cpu().numpy().tobytes() for k, v in t.items()}
    for name in SHORT[call]:
        k0 = rmcl_b200.kernel_launch_count()
        with pytest.raises(ValueError):
            CALLS[call](up, beams, tsb, _short(t, name))
        torch.cuda.synchronize()
        assert rmcl_b200.kernel_launch_count() == k0, name
        assert {k: v.cpu().numpy().tobytes() for k, v in t.items()} == before, name
        assert lib.b2_peek_cuda_error().decode() == ""
    k0 = rmcl_b200.kernel_launch_count()
    CALLS[call](up, beams, tsb, t)
    torch.cuda.synchronize()
    assert rmcl_b200.kernel_launch_count() > k0
    assert lib.b2_peek_cuda_error().decode() == ""


@pytest.mark.gpu
def test_python_host_update_mismatch_is_refused():
    """update on host arrays: attrs one record short is refused with nothing copied or launched; arrays that agree run"""
    import rmcl_b200
    up, beams, tsb, _, (P, A) = _case()
    A0 = A.tobytes()
    for p, a in ((P, A[:-1]), (P[:-1], A)):
        k0 = rmcl_b200.kernel_launch_count()
        with pytest.raises(ValueError):
            up.update(p, a, tsb, beams, inplace=True)
        assert rmcl_b200.kernel_launch_count() == k0 and A.tobytes() == A0
    assert len(up.update(P, A, tsb, beams)) == N


@pytest.mark.gpu
def test_cpp_updater_refuses_views_of_different_sizes():
    exe = native.adapter("pf_args_cpp")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    methods = {"update RAM": "update", "update VRAM": "update", "update field": "update", "motionUpdate": "motionUpdate",
               "projectToSurface": "projectToSurface", "resample": "resample", "resampleResidual": "resampleResidual", "resampleKLD": "resampleKLD",
               "initSamplesUniform": "initSamplesUniform", "initSamples": "initSamples", "estimateStats": "estimateStats",
               "estimateClusters": "estimateClusters", "recoveryInject": "recoveryInject"}
    lines = r.stdout.splitlines()
    for case, method in methods.items():
        assert f"RAN {case}" in lines, (case, r.stdout)
        for label in ((f"{case} all", f"{case} new") if case.startswith("resample") else (case,)):
            assert f"REFUSED {label}: {method}: poses and attrs differ in size" in lines, (label, r.stdout)
