"""CPU tests of the Python binding's argument check (rmcl_b200/api.py).  The C ABI takes bare pointers and one count per call, so the binding
derives the count from one array and refuses the call when another array the library indexes with it is of a different length.

The library is replaced by a recorder: every b2_* function records its name and arguments and returns 0.  Handles are built with __new__
and CUDA tensors are faked by what the binding reads of them.  For each entry point:
  * arrays that agree: exactly one library call, with the expected count and each array's address;
  * one array one record short: ValueError and no library call;
  * an array whose byte size is not a whole number of records: TypeError and no library call."""
import numpy as np
import pytest

import rmcl_b200
from rmcl_b200 import api, synth

N, N_NEW = 5, 3                     # the count of the particle set and of a resampling's outputs


class _Handle:
    """stands in for a library handle; false, so that close() never hands it to the real library"""

    def __bool__(self):
        return False


class FakeCuda:
    """what the binding reads of a torch CUDA tensor: nbytes bytes of itemsize-byte elements at a made-up device address"""
    _next = 0x7F00_0000_0000

    def __init__(self, nbytes, itemsize=4):
        self._numel, self._itemsize = nbytes // itemsize, itemsize
        self._ptr, FakeCuda._next = FakeCuda._next, FakeCuda._next + (1 << 24)
        self.shape, self.device, self.is_cuda = (self._numel,), "cuda:0", True

    def numel(self):
        return self._numel

    def element_size(self):
        return self._itemsize

    def is_contiguous(self):
        return True

    def data_ptr(self):
        return self._ptr


_NP_RECORDS = {32: synth.TRANSFORM_DTYPE, 36: synth.PARTICLE_ATTR_DTYPE, 64: synth.CROSS_STATS_DTYPE}


def _array(kind, size, count, extra=0):
    """count records of size bytes, plus `extra` bytes that do not make a record: a fake CUDA tensor or a numpy array"""
    if kind == "cuda":
        return FakeCuda(size * count + extra, 1 if size == 1 or extra % 4 else 4)
    if size == 12:
        return np.zeros(3 * count + bool(extra), np.float32)
    if extra or size == 1:
        return np.zeros(size * count + extra, np.uint8)
    return np.zeros(count, _NP_RECORDS[size])


def _address(x):
    return x.data_ptr() if isinstance(x, FakeCuda) else x.ctypes.data


@pytest.fixture
def calls(monkeypatch):
    log = []

    class Recorder:
        def __getattr__(self, name):
            if not name.startswith("b2_"):
                raise AttributeError(name)
            return lambda *args: log.append((name, args)) or 0

    monkeypatch.setattr(api, "load_library", Recorder)
    return log


def _pf(field=False):
    up = rmcl_b200.PCDSensorUpdaterB200.__new__(rmcl_b200.PCDSensorUpdaterB200)
    up._h, up.config, up._input, up._field, up.samples, up.seed, up.step = _Handle(), rmcl_b200.PFParams.defaults(), None, None, 100, 0, 0
    if field:
        up._field = rmcl_b200.DistanceField.__new__(rmcl_b200.DistanceField)
        up._field._h = _Handle()
    return up


def _rcc():
    h = rmcl_b200.RCCB200.__new__(rmcl_b200.RCCB200)
    h._h = _Handle()
    return h


def _map():
    m = rmcl_b200.Map.__new__(rmcl_b200.Map)
    m._h = _Handle()
    return m


TSB, BEAMS = synth.make_transform(), np.zeros(4, synth.RANGE_MEAS_DTYPE)
BOX = [0.0] * 6
COV = np.eye(6).reshape(-1)

# entry point: (library function, array kind, call, {array: (record size, count, argument index)}, {count: argument index}).  An array's
# count is N or N_NEW; the first array of each count gives it.
CASES = {
    "update": ("b2_pf_sensor_update", "cuda", lambda x: _pf().update(x["poses"], x["attrs"], TSB, BEAMS),
               {"poses": (32, N, 1), "attrs": (36, N, 2)}, {N: 3}),
    "update_field": ("b2_pf_sensor_update_field", "cuda", lambda x: _pf(field=True).update(x["poses"], x["attrs"], TSB, BEAMS),
                     {"poses": (32, N, 2), "attrs": (36, N, 3)}, {N: 4}),
    "update_host": ("b2_pf_sensor_update_host", "np", lambda x: _pf().update(x["poses"], x["attrs"], TSB, BEAMS, inplace=True),
                    {"poses": (32, N, 1), "attrs": (36, N, 2)}, {N: 3}),
    "motionUpdate": ("b2_pf_motion_update", "cuda", lambda x: _pf().motionUpdate(x["poses"], x["attrs"], TSB, 0.01),
                     {"poses": (32, N, 1), "attrs": (36, N, 2)}, {N: 3}),
    "resample": ("b2_pf_resample_gladiator", "cuda",
                 lambda x: _pf().resample(x["poses"], x["attrs"], x["poses_new"], x["attrs_new"], raw=x["raw"], normals=x["normals"]),
                 {"poses": (32, N, 1), "attrs": (36, N, 2), "poses_new": (32, N_NEW, 6), "attrs_new": (36, N_NEW, 7), "raw": (4, N_NEW, 11),
                  "normals": (24, N_NEW, 12)}, {N: 3, N_NEW: 5}),
    "projectToSurface": ("b2_pf_project_to_surface", "cuda", lambda x: _pf().projectToSurface(x["poses"], x["attrs"]),
                         {"poses": (32, N, 1), "attrs": (36, N, 2)}, {N: 3}),
    "initSamplesUniform": ("b2_pf_init_uniform", "cuda", lambda x: _pf().initSamplesUniform(x["poses"], x["attrs"], BOX, BOX, 1),
                           {"poses": (32, N, 1), "attrs": (36, N, 2)}, {N: 4}),
    "initSamples": ("b2_pf_init_gaussian", "cuda", lambda x: _pf().initSamples(x["poses"], x["attrs"], TSB, COV, 1),
                    {"poses": (32, N, 1), "attrs": (36, N, 2)}, {N: 4}),
    "estimateStats": ("b2_pf_estimate_stats", "cuda", lambda x: _pf().estimateStats(x["poses"], x["attrs"]),
                      {"poses": (32, N, 1), "attrs": (36, N, 2)}, {N: 3}),
    "recoveryInject": ("b2_pf_recovery_inject", "cuda", lambda x: _pf().recoveryInject(x["poses"], x["attrs"], BOX, BOX),
                       {"poses": (32, N, 1), "attrs": (36, N, 2)}, {N: 4}),
    "estimateClusters": ("b2_pf_cluster_stats", "cuda", lambda x: _pf().estimateClusters(x["poses"], x["attrs"], labels=x["labels"]),
                         {"poses": (32, N, 1), "attrs": (36, N, 2), "labels": (4, N, 6)}, {N: 3}),
    "resampleResidual": ("b2_pf_resample_residual", "cuda", lambda x: _pf().resampleResidual(x["poses"], x["attrs"], x["poses_new"], x["attrs_new"]),
                         {"poses": (32, N, 1), "attrs": (36, N, 2), "poses_new": (32, N_NEW, 7), "attrs_new": (36, N_NEW, 8)}, {N: 3, N_NEW: 6}),
    "resampleKLD": ("b2_pf_resample_kld", "cuda", lambda x: _pf().resampleKLD(x["poses"], x["attrs"], x["poses_new"], x["attrs_new"]),
                    {"poses": (32, N, 1), "attrs": (36, N, 2), "poses_new": (32, N_NEW, 7), "attrs_new": (36, N_NEW, 8)}, {N: 3, N_NEW: 6}),
    "setDataset": ("b2_rcc_set_dataset", "cuda", lambda x: _rcc().setDataset(x["points"], x["mask"]), {"points": (12, N, 1), "mask": (1, N, 2)}, {N: 3}),
    "setDataset_host": ("b2_rcc_set_dataset", "np", lambda x: _rcc().setDataset(x["points"], x["mask"]), {"points": (12, N, 1), "mask": (1, N, 2)},
                        {N: 3}),
    "bindDataset": ("b2_rcc_bind_dataset", "cuda", lambda x: _rcc().bindDataset(x["points"], x["mask"]), {"points": (12, N, 1), "mask": (1, N, 2)},
                    {N: 3}),
    "bindModelBuffers": ("b2_rcc_bind_model_buffers", "cuda", lambda x: _rcc().bindModelBuffers(x["points"], x["normals"], x["hits"]),
                         {"hits": (1, N, 3), "points": (12, N, 1), "normals": (12, N, 2)}, {N: 4}),
    "intersect": ("b2_mesh_intersect", "np", lambda x: _map().intersect(x["origs"], x["dirs"]), {"origs": (12, N, 1), "dirs": (12, N, 2)}, {N: 3}),
    "traversal_stats": ("b2_mesh_intersect_stats", "np", lambda x: _map().traversal_stats(x["origs"], x["dirs"]),
                        {"origs": (12, N, 1), "dirs": (12, N, 2)}, {N: 3}),
    "umeyama_transform": ("b2_umeyama_batch", "np", lambda x: rmcl_b200.umeyama_transform(x["stats"]), {"stats": (64, N, 0)}, {N: 1}),
}


def _arrays(case, short=None, ragged=None):
    """the case's arrays, each of its count; `short` one record short, `ragged` with a partial record after its whole ones"""
    _, kind, _, arrays, _ = CASES[case]
    return {k: _array(kind, size, count - (k == short), 2 if k == ragged else 0) for k, (size, count, _) in arrays.items()}


@pytest.mark.parametrize("case", sorted(CASES))
def test_matched_arrays_reach_the_library_once(calls, case):
    fn, _, call, arrays, counts = CASES[case]
    x = _arrays(case)
    call(x)
    assert [name for name, _ in calls] == [fn]
    args = [getattr(a, "value", a) for a in calls[0][1]]
    for k, (_, _, at) in arrays.items():
        assert args[at] == _address(x[k]), k
    for count, at in counts.items():
        assert args[at] == count


@pytest.mark.parametrize("case, array", [(c, k) for c in sorted(CASES) for k in CASES[c][3] if len(CASES[c][3]) > 1])
def test_an_array_one_record_short_is_refused(calls, case, array):
    with pytest.raises(ValueError):
        CASES[case][2](_arrays(case, short=array))
    assert calls == []


@pytest.mark.parametrize("case, array", [(c, k) for c in sorted(CASES) for k, (size, _, _) in CASES[c][3].items() if size > 1])
def test_a_partial_record_is_refused(calls, case, array):
    with pytest.raises(TypeError):
        CASES[case][2](_arrays(case, ragged=array))
    assert calls == []


def test_host_update_passes_the_copy_it_returns(calls):
    """update on numpy arrays without inplace: the library updates a copy of the attributes, and that copy is returned"""
    x = _arrays("update_host")
    out = _pf().update(x["poses"], x["attrs"], TSB, BEAMS)
    assert out is not x["attrs"] and out.dtype == synth.PARTICLE_ATTR_DTYPE and len(out) == N
    assert [name for name, _ in calls] == ["b2_pf_sensor_update_host"] and calls[0][1][2].value == out.ctypes.data


def test_update_refuses_before_drawing_beams(calls):
    """a refused update draws no beams from the input cloud and leaves the step as it was"""
    up = _pf()
    up._input = synth.pointcloud2(np.ones((4, 3), np.float32), 4, 1)
    x = _arrays("update", short="attrs")
    with pytest.raises(ValueError):
        up.update(x["poses"], x["attrs"], TSB)
    assert calls == [] and up.step == 0


def test_optional_arrays_pass_as_null(calls):
    """resample without raw / normals and estimateClusters without labels: null addresses, the counts from the arrays given"""
    x = _arrays("resample")
    _pf().resample(x["poses"], x["attrs"], x["poses_new"], x["attrs_new"])
    _pf().estimateClusters(x["poses"], x["attrs"])
    (f1, a1), (f2, a2) = calls
    assert (f1, a1[3].value, a1[5].value, a1[11], a1[12]) == ("b2_pf_resample_gladiator", N, N_NEW, None, None)
    assert (f2, a2[3].value, a2[6]) == ("b2_pf_cluster_stats", N, None)
