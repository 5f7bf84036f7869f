"""Device voxelizer: torch wrapper over d3b_voxelize_dev (csrc/voxelize.cu).

Reference semantics: det3d/ops/point_cloud/point_cloud_ops.py:7-55,112-184.
"""
import ctypes as C

import numpy as np
import torch

from ... import _lib
from ..._lib import VoxelCfg
from ...utils.staging import Upload

MAX_BATCH = 64


def grid_size_of(voxel_size, point_cloud_range):
    """round((hi - lo) / vs) in fp32, exactly as voxel_generator.py:7-11 / point_cloud_ops.py:26-29."""
    pcr = np.asarray(point_cloud_range, dtype=np.float32)
    vs = np.asarray(voxel_size, dtype=np.float32)
    return np.round((pcr[3:] - pcr[:3]) / vs).astype(np.int64)


def check_host_offsets(offsets, n_rows):
    """Host cloud offsets [0, n0, n0+n1, ...] as a list of ints; _lib.D3BError unless 1 <= batch <= 64 and
    0 = off[0] <= ... <= off[batch] <= n_rows."""
    offsets = [int(o) for o in offsets]
    batch = len(offsets) - 1
    if not 1 <= batch <= MAX_BATCH:
        raise _lib.D3BError("Voxelizer: batch %d outside [1, %d]" % (batch, MAX_BATCH))
    if offsets[0] != 0 or any(b < a for a, b in zip(offsets[:-1], offsets[1:])):
        raise _lib.D3BError("Voxelizer: cloud offsets not 0 = off[0] <= ... <= off[batch]: %s" % offsets)
    if offsets[-1] > n_rows:
        raise _lib.D3BError("Voxelizer: cloud offsets end at %d, past the %d rows of points" % (offsets[-1], n_rows))
    return offsets


class Voxelizer:
    """Voxelizes a batch of clouds on the GPU in one call; outputs stay on the device.

    out = voxelizer(points, offsets) with points [N_total, ndim] f32 cuda and
    offsets a host list [0, n0, n0+n1, ...] (_lib.D3BError unless 0 = off[0] <= ... <= off[batch] <= N_total with
    1 <= batch <= 64, raised before anything is enqueued).  Returns a dict of device tensors:
      voxels [cap, max_points, ndim] (optional), coors [cap, 4] (b,z,y,x),
      num_points [cap], mean [cap, ndim], counts int32[batch+1] (last = total rows).
    Only the first counts[-1] rows are defined.  A host list is copied to a device int32[batch+1] kept with the call's
    buffers (pinned staging, no host sync, and only when it differs from the previous one).

    `offsets` may instead be an int32 cuda tensor [batch+1]: then points.shape[0] is a capacity, rows at or past
    offsets[-1] are never read, and nothing the host passes depends on the cloud sizes, so the call can be captured in
    a CUDA graph and replayed for clouds of any size.  out["status"] (int32[1]) is then 1 if the offsets were not
    0 = off[0] <= ... <= off[batch] <= capacity (the call ran on them clamped into that shape), else 0.
    Either way d3b_voxelize_dev runs, and its results do not depend on the capacity.
    """

    def __init__(self, voxel_size, point_cloud_range, max_num_points, max_voxels, want_voxels=True,
                 want_mean=True):
        self.voxel_size = np.asarray(voxel_size, dtype=np.float32)
        self.point_cloud_range = np.asarray(point_cloud_range, dtype=np.float32)
        self.grid_size = grid_size_of(self.voxel_size, self.point_cloud_range)
        self.max_num_points = int(max_num_points)
        self.max_voxels = int(max_voxels)
        self.want_voxels = want_voxels
        self.want_mean = want_mean
        self._bufs = {}

    def _cfg(self, ndim):
        cfg = VoxelCfg()
        for j in range(3):
            cfg.voxel_size[j] = float(self.voxel_size[j])
            cfg.range_min[j] = float(self.point_cloud_range[j])
            cfg.grid[j] = int(self.grid_size[j])
        cfg.ndim = ndim
        cfg.max_points = self.max_num_points
        cfg.max_voxels = self.max_voxels
        return cfg

    def _buffers(self, n_total, batch, ndim, device, fixed_capacity=False):
        # With device offsets the buffers of each capacity are kept for good: a captured graph holds their addresses.
        # Host offsets go through the growable buffers' own device copy of them.
        key = (batch, ndim, device, n_total) if fixed_capacity else (batch, ndim, device)
        b = self._bufs.get(key)
        if b is not None and b["n_cap"] >= n_total:
            return b
        n_cap = max(n_total, 1)
        cfg = self._cfg(ndim)
        ws_bytes = _lib.lib().d3b_voxelize_workspace_bytes(C.byref(cfg), n_cap, batch)
        cap = batch * self.max_voxels
        b = {
            "n_cap": n_cap,
            "cfg": cfg,
            "ws": torch.empty(ws_bytes, dtype=torch.uint8, device=device),
            "coors": torch.empty((cap, 4), dtype=torch.int32, device=device),
            "num_points": torch.empty(cap, dtype=torch.int32, device=device),
            "counts": torch.zeros(batch + 1, dtype=torch.int32, device=device),
            "status": torch.zeros(1, dtype=torch.int32, device=device),
            "voxels": torch.empty((cap, self.max_num_points, ndim), dtype=torch.float32, device=device)
            if self.want_voxels else None,
            "mean": torch.empty((cap, ndim), dtype=torch.float32, device=device) if self.want_mean else None,
        }
        if not fixed_capacity:
            b["offsets"] = Upload(torch.zeros(batch + 1, dtype=torch.int32, device=device))
        self._bufs[key] = b
        return b

    def __call__(self, points, offsets=None):
        assert points.dtype == torch.float32 and points.dim() == 2
        n_rows, ndim = points.shape
        if offsets is None:
            offsets = [0, n_rows]
        on_device = torch.is_tensor(offsets) and offsets.is_cuda
        if on_device:
            if offsets.dtype != torch.int32 or offsets.dim() != 1 or offsets.device != points.device:
                raise ValueError("device offsets must be an int32 vector on the points' device")
            offsets = offsets.contiguous()
        else:
            offsets = check_host_offsets(offsets, n_rows)
        assert points.is_cuda
        points = points.contiguous()
        batch = len(offsets) - 1
        b = self._buffers(n_rows, batch, ndim, points.device, fixed_capacity=on_device)
        if not on_device:
            b["offsets"].put(offsets)                # enqueued outside the "voxelize" stage's bracket
            offsets = b["offsets"].dev
        with _lib.on_device_of(points), _lib.timed("voxelize", n_points=n_rows, ndim=ndim, batch=batch):
            st = _lib.lib().d3b_voxelize_dev(
                C.byref(b["cfg"]), points.data_ptr() if n_rows > 0 else None, n_rows, offsets.data_ptr(), batch,
                _lib.ptr(b["voxels"]), b["coors"].data_ptr(), b["num_points"].data_ptr(), _lib.ptr(b["mean"]),
                b["counts"].data_ptr(), b["status"].data_ptr(), b["ws"].data_ptr(), b["ws"].numel(),
                _lib.current_stream(),
            )
        _lib.check(st, "d3b_voxelize_dev")
        out = {k: b[k] for k in ("voxels", "coors", "num_points", "mean", "counts")}
        if on_device:
            out["status"] = b["status"]
        # the per-voxel point-index lists the voxelizer built on the way ([batch][max_voxels][max_points] indices into
        # `points`, valid until the next call): what the fused pillar reader consumes instead of `voxels`
        out["point_lists"] = dict(points=points, lists_ptr=_lib.lib().d3b_voxelize_point_lists(
            C.byref(b["cfg"]), n_rows, batch, b["ws"].data_ptr()), batch=batch, max_voxels=self.max_voxels,
            max_points=self.max_num_points, keepalive=b["ws"])
        return out
