"""d3b_ingest_sweeps_dev and InferencePipeline.infer_sweeps validate their arguments on the host before any CUDA call
(no GPU needed): status 1 (4 for a short workspace) with a message, and ValueError."""
import numpy as np
import pytest
import torch

from det3d_b200 import _lib

# stand-ins for device pointers: never dereferenced, every call below is rejected first
_P = 0x1000


def _call(raw=_P, capacity=4096, stride=5, n_feat=4, off=_P, samples=_P, tms=_P, lags=_P, flags=_P, table_cap=8,
          batch=2, out=_P, cloud_offsets=_P, ws=_P, ws_bytes=None):
    L = _lib.lib()
    if ws_bytes is None:
        ws_bytes = L.d3b_ingest_dev_workspace_bytes(max(capacity, 0), max(table_cap, 1))
    return L.d3b_ingest_sweeps_dev(raw, capacity, stride, n_feat, off, None, samples, tms, lags, flags, table_cap, batch,
                                   1.0, out, cloud_offsets, None, ws, ws_bytes, None)


def test_null_arguments_are_rejected():
    L = _lib.lib()
    for name in ("off", "samples", "tms", "lags", "flags", "cloud_offsets", "ws"):
        assert _call(**{name: None}) == 1, name
        assert b"null" in L.d3b_last_error(), name
    for name in ("raw", "out"):
        assert _call(**{name: None}) == 1, name
        assert b"null buffer" in L.d3b_last_error(), name


def test_batch_and_table_capacity_bounds():
    L = _lib.lib()
    for batch in (0, -1, 65):
        assert _call(batch=batch, ws_bytes=1 << 30) == 1, batch
        assert b"batch" in L.d3b_last_error()
    for table_cap, batch in ((0, 1), (-3, 2), (17, 1), (33, 2), (1025, 64)):
        assert _call(table_cap=table_cap, batch=batch, ws_bytes=1 << 30) == 1, (table_cap, batch)
        assert b"sweep_capacity" in L.d3b_last_error()


def test_capacity_and_layout_are_checked():
    L = _lib.lib()
    for capacity in (-1, (1 << 30) + 1):
        assert _call(capacity=capacity, ws_bytes=1 << 40) == 1, capacity
        assert b"raw_capacity" in L.d3b_last_error()
    for stride, n_feat in ((3, 4), (5, 2)):
        assert _call(stride=stride, n_feat=n_feat) == 1
        assert b"layout" in L.d3b_last_error()


def test_small_workspace_is_rejected():
    L = _lib.lib()
    need = L.d3b_ingest_dev_workspace_bytes(4096, 8)
    assert need > 0
    assert _call(ws_bytes=need - 1) == 4                              # D3B_ERR_WORKSPACE
    assert b"workspace" in L.d3b_last_error()


def test_workspace_query():
    L = _lib.lib()
    assert L.d3b_ingest_dev_workspace_bytes(-1, 4) == 0 and L.d3b_ingest_dev_workspace_bytes(100, 0) == 0
    # two int arrays of (raw chunks + one partial chunk per sweep), each 256-byte aligned
    assert L.d3b_ingest_dev_workspace_bytes(0, 1) == 512
    assert L.d3b_ingest_dev_workspace_bytes(1 << 20, 64) == 2 * (((1024 + 64) * 4 + 255) // 256 * 256)


def _sample(n_sweeps=3, n=10, stride=5):
    raws = [np.zeros((n, stride), np.float32) for _ in range(n_sweeps)]
    return raws, [None] + [np.eye(4)] * (n_sweeps - 1), [0.05 * s for s in range(n_sweeps)]


def test_check_sweep_samples_accepts_numpy_and_host_tensors():
    from det3d_b200.datasets.pipelines.loading import check_sweep_samples
    raws, tms, lags = _sample()
    raws[1] = torch.from_numpy(raws[1])
    assert check_sweep_samples([(raws, tms, lags), _sample(1, 0)]) == (5, [[10, 10, 10], [0]])


@pytest.mark.parametrize("case", ["no samples", "65 samples", "no sweeps", "17 sweeps", "lags short", "transforms short",
                                  "float64 raw", "1-D raw", "mixed stride", "3x4 transform", "stride < n_feat",
                                  "not a triple"])
def test_infer_sweeps_rejects_malformed_samples(case):
    from det3d_b200.apis import InferencePipeline
    pipe = object.__new__(InferencePipeline)          # the checks run before anything touches the model or the device
    pipe.num_point_features = 5
    raws, tms, lags = _sample()
    bad = {
        "no samples": [],
        "65 samples": [_sample()] * 65,
        "no sweeps": [([], [], [])],
        "17 sweeps": [_sample(17)],
        "lags short": [(raws, tms, lags[:2])],
        "transforms short": [(raws, tms[:2], lags)],
        "float64 raw": [([r.astype(np.float64) for r in raws], tms, lags)],
        "1-D raw": [([r.reshape(-1) for r in raws], tms, lags)],
        "mixed stride": [_sample(), _sample(2, 10, 6)],
        "3x4 transform": [(raws, [None, np.eye(4)[:3], None], lags)],
        "stride < n_feat": [_sample(2, 10, 3)],
        "not a triple": [(raws, tms)],
    }[case]
    with pytest.raises(ValueError):
        pipe.infer_sweeps(bad)


def test_infer_sweeps_rejects_a_feature_count_the_reader_does_not_take():
    from det3d_b200.apis import InferencePipeline
    pipe = object.__new__(InferencePipeline)
    pipe.num_point_features = 5
    with pytest.raises(ValueError, match="reader"):
        pipe.infer_sweeps([_sample()], n_feat=3)
