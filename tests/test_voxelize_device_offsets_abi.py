"""d3b_voxelize_dev validates its arguments on the host before any CUDA call (no GPU needed): status 1 (4 for a short
workspace) and a message; the Voxelizer rejects malformed host offsets before anything is allocated or enqueued."""
import ctypes

import pytest
import torch

from det3d_b200 import _lib


def _cfg():
    cfg = _lib.VoxelCfg()
    for j, (vs, lo, g) in enumerate(zip((0.05, 0.05, 0.1), (0.0, -40.0, -3.0), (1408, 1600, 40))):
        cfg.voxel_size[j], cfg.range_min[j], cfg.grid[j] = vs, lo, g
    cfg.ndim, cfg.max_points, cfg.max_voxels = 4, 5, 100
    return cfg


# stand-ins for device pointers: never dereferenced, every call below is rejected first
_P = 0x1000


def _call(cfg, points=_P, capacity=2048, offsets=_P, batch=2, coors=_P, num_points=_P, counts=_P, ws=_P, ws_bytes=None):
    L = _lib.lib()
    if ws_bytes is None:
        ws_bytes = L.d3b_voxelize_workspace_bytes(ctypes.byref(cfg), max(capacity, 0), batch) if cfg is not None else 0
    return L.d3b_voxelize_dev(None if cfg is None else ctypes.byref(cfg), points, capacity, offsets, batch, None, coors,
                              num_points, None, counts, None, ws, ws_bytes, None)


def test_null_arguments_are_rejected():
    L = _lib.lib()
    cfg = _cfg()
    assert _call(None) == 1 and b"null" in L.d3b_last_error()
    for name in ("offsets", "coors", "num_points", "counts", "ws"):
        assert _call(cfg, **{name: None}) == 1, name
        assert b"null" in L.d3b_last_error(), name
    assert _call(cfg, points=None) == 1 and b"points" in L.d3b_last_error()


def test_batch_outside_1_to_64_is_rejected():
    L = _lib.lib()
    for batch in (0, -1, 65):
        assert _call(_cfg(), batch=batch, ws_bytes=1 << 30) == 1, batch
        assert b"batch" in L.d3b_last_error()


def test_negative_capacity_is_rejected():
    L = _lib.lib()
    assert _call(_cfg(), capacity=-1, ws_bytes=1 << 30) == 1
    assert b"capacity" in L.d3b_last_error()


def test_small_workspace_is_rejected():
    L = _lib.lib()
    cfg = _cfg()
    need = L.d3b_voxelize_workspace_bytes(ctypes.byref(cfg), 2048, 2)
    assert need > 0
    assert _call(cfg, ws_bytes=need - 1) == 4                          # D3B_ERR_WORKSPACE
    assert b"workspace" in L.d3b_last_error()


@pytest.mark.parametrize("offsets", [[5, 10], [0, 7, 3, 10], [0, 4, 11], [0, 10, 10, 11], [0], [0] * 66, [-1, 10]])
def test_voxelizer_rejects_malformed_host_offsets(offsets):
    """off[0] != 0, decreasing, past the 10 rows of points (which would read past the buffer), batch 0 or 65."""
    from det3d_b200.ops.point_cloud.voxelize import Voxelizer
    vox = Voxelizer([0.05, 0.05, 0.1], [0, -40.0, -3.0, 70.4, 40.0, 1.0], 5, 100)
    with pytest.raises(_lib.D3BError, match="Voxelizer"):
        vox(torch.zeros((10, 4)), offsets)
    assert vox._bufs == {}                                              # nothing allocated, nothing enqueued
