"""d3b_frustum_crop_dev and InferencePipeline.infer_raw validate their arguments on the host before any CUDA call (no GPU
needed): status 1 (3 for an ndim that is not built, 4 for a short workspace) with a message, and ValueError."""
import numpy as np
import pytest
import torch

from det3d_b200 import _lib

# stand-ins for device pointers: never dereferenced, every call below is rejected first
_P = 0x1000


def _call(points=_P, capacity=4096, ndim=4, off=_P, planes=_P, batch=2, out=_P, cloud_offsets=_P, ws=_P, ws_bytes=None):
    L = _lib.lib()
    if ws_bytes is None:
        ws_bytes = L.d3b_frustum_crop_workspace_bytes(max(capacity, 0), min(max(batch, 1), 64))
    return L.d3b_frustum_crop_dev(points, capacity, ndim, off, planes, batch, out, cloud_offsets, None, ws, ws_bytes,
                                  None)


def test_null_arguments_are_rejected():
    L = _lib.lib()
    for name in ("off", "planes", "cloud_offsets", "ws"):
        assert _call(**{name: None}) == 1, name
        assert b"null argument" in L.d3b_last_error(), name
    for name in ("points", "out"):
        assert _call(**{name: None}) == 1, name
        assert b"null buffer" in L.d3b_last_error(), name
    # an empty capacity needs no point buffers: the call gets as far as the (too small) workspace
    assert _call(points=None, out=None, capacity=0, ws_bytes=0) == 4
    assert b"workspace" in L.d3b_last_error()


def test_batch_bounds():
    L = _lib.lib()
    for batch in (0, -1, 65):
        assert _call(batch=batch, ws_bytes=1 << 30) == 1, batch
        assert b"batch" in L.d3b_last_error()


def test_capacity_bounds():
    L = _lib.lib()
    for capacity in (-1, (1 << 30) + 1):
        assert _call(capacity=capacity, ws_bytes=1 << 40) == 1, capacity
        assert b"point_capacity" in L.d3b_last_error()


def test_ndim_outside_3_to_16_is_not_built():
    L = _lib.lib()
    for ndim in (-1, 0, 2, 17, 64):
        assert _call(ndim=ndim) == 3, ndim                                 # D3B_ERR_UNSUPPORTED
        assert b"ndim" in L.d3b_last_error()
    for ndim in (3, 16):                                                   # accepted, then stopped by the workspace
        assert _call(ndim=ndim, ws_bytes=0) == 4, ndim


def test_small_workspace_is_rejected():
    L = _lib.lib()
    need = L.d3b_frustum_crop_workspace_bytes(4096, 2)
    assert need > 0
    assert _call(ws_bytes=need - 1) == 4                                  # D3B_ERR_WORKSPACE, as the ingest returns
    assert b"workspace" in L.d3b_last_error()


def test_workspace_query():
    L = _lib.lib()
    for cap, batch in ((-1, 1), ((1 << 30) + 1, 1), (100, 0), (100, 65)):
        assert L.d3b_frustum_crop_workspace_bytes(cap, batch) == 0, (cap, batch)
    # two int arrays of (chunks + one partial chunk per cloud), each 256-byte aligned
    assert L.d3b_frustum_crop_workspace_bytes(0, 1) == 512
    assert L.d3b_frustum_crop_workspace_bytes(1 << 20, 64) == 2 * (((1024 + 64) * 4 + 255) // 256 * 256)
    assert L.d3b_frustum_crop_workspace_bytes(1 << 30, 64) == 2 * (((1 << 20) + 64) * 4)


def _calib():
    from det3d_b200.utils.synthetic import kitti_like_calib
    return kitti_like_calib(0)


def _pipe():
    from det3d_b200.apis import InferencePipeline
    return object.__new__(InferencePipeline)          # the checks run before anything touches the model or the device


@pytest.mark.parametrize("case", ["no clouds", "65 clouds", "calibs short", "float64 cloud", "1-D cloud", "mixed ndim",
                                  "ndim 2", "ndim 17", "cuda-less tensor dtype", "missing key", "3x3 rect", "P2 3x3",
                                  "image shape 0", "image shape scalar"])
def test_infer_raw_rejects_malformed_arguments(case):
    c = np.zeros((10, 4), np.float32)
    cal = _calib()
    bad_cal = lambda **kw: dict(cal, **kw)                                # noqa: E731
    clouds, calibs = {
        "no clouds": ([], []),
        "65 clouds": ([c] * 65, [cal] * 65),
        "calibs short": ([c, c], [cal]),
        "float64 cloud": ([c.astype(np.float64)], [cal]),
        "1-D cloud": ([c.reshape(-1)], [cal]),
        "mixed ndim": ([c, np.zeros((3, 5), np.float32)], [cal, cal]),
        "ndim 2": ([np.zeros((3, 2), np.float32)], [cal]),
        "ndim 17": ([np.zeros((3, 17), np.float32)], [cal]),
        "cuda-less tensor dtype": ([torch.zeros((3, 4), dtype=torch.float64)], [cal]),
        "missing key": ([c], [{k: v for k, v in cal.items() if k != "P2"}]),
        "3x3 rect": ([c], [bad_cal(rect=np.eye(3))]),
        "P2 3x3": ([c], [bad_cal(P2=np.eye(3))]),
        "image shape 0": ([c], [bad_cal(image_shape=(0, 1242))]),
        "image shape scalar": ([c], [bad_cal(image_shape=375)]),
    }[case]
    with pytest.raises(ValueError):
        _pipe().infer_raw(clouds, calibs)


def test_frustum_crop_rejects_bad_shapes():
    from det3d_b200.ops.point_cloud.frustum import FrustumCrop
    for kw in (dict(batch=0), dict(batch=65), dict(ndim=2), dict(ndim=17), dict(capacity=-1)):
        args = dict(batch=1, capacity=16, ndim=4, device="cpu")
        args.update(kw)
        with pytest.raises(ValueError):
            FrustumCrop(**args)
