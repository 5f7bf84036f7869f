"""Device camera-frustum crop: torch wrapper over d3b_frustum_crop_dev (csrc/frustum.cu).

Reference semantics: det3d/core/bbox/box_np_ops.py:941-952 (remove_outside_points), for a batch of raw scans with
their own calibrations.  The planes come from det3d_b200.core.bbox.box_np_ops.camera_frustum_planes.
"""
import numpy as np
import torch

from ... import _lib

MAX_BATCH = 64
MIN_NDIM, MAX_NDIM = 3, 16


class FrustumCrop:
    """Static device buffers of one crop shape -- raw points [capacity, ndim], raw cloud offsets [B + 1], planes
    f64 [B, 6, 4], the cropped clouds [capacity, ndim], their cloud offsets [B + 1], status, workspace -- and the
    d3b_frustum_crop_dev call over them.  The addresses never change, so a captured CUDA graph can hold them; the
    cropped clouds and their offsets are in the form the voxelizer's device-offset path takes."""

    def __init__(self, batch, capacity, ndim, device="cuda"):
        if not 1 <= batch <= MAX_BATCH:
            raise ValueError("batch must be in [1, %d], got %d" % (MAX_BATCH, batch))
        if not MIN_NDIM <= ndim <= MAX_NDIM:
            raise ValueError("ndim must be in [%d, %d], got %d" % (MIN_NDIM, MAX_NDIM, ndim))
        if not 0 <= capacity <= 1 << 30:
            raise ValueError("capacity %d outside [0, 2^30]" % capacity)
        dev = torch.device(device)
        self.batch, self.capacity, self.ndim = batch, int(capacity), int(ndim)
        rows = max(self.capacity, 1)
        self.points = torch.empty((rows, ndim), dtype=torch.float32, device=dev)   # rows past offsets[B] are never read
        self.offsets = torch.zeros(batch + 1, dtype=torch.int32, device=dev)
        self.planes = torch.zeros((batch, 6, 4), dtype=torch.float64, device=dev)
        self.out = torch.empty((rows, ndim), dtype=torch.float32, device=dev)
        self.cloud_offsets = torch.zeros(batch + 1, dtype=torch.int32, device=dev)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self.ws = torch.empty(_lib.lib().d3b_frustum_crop_workspace_bytes(self.capacity, batch), dtype=torch.uint8,
                              device=dev)

    def set_table(self, offsets, planes):
        """Synchronous copy of host offsets [B + 1] and planes [B, 6, 4] into the device buffers (graphs stage them
        through pinned memory instead: apis.pipeline)."""
        self.offsets.copy_(torch.as_tensor(np.asarray(offsets, np.int32)))
        self.planes.copy_(torch.as_tensor(np.asarray(planes, np.float64)))

    def launch(self):
        """Crops the raw points under the device offsets and planes into out / cloud_offsets (three kernels, no host
        sync).  Returns (out, cloud_offsets)."""
        L = _lib.lib()
        with _lib.on_device_of(self.points), _lib.timed("frustum_crop", batch=self.batch, capacity=self.capacity):
            st = L.d3b_frustum_crop_dev(
                self.points.data_ptr(), self.capacity, self.ndim, self.offsets.data_ptr(), self.planes.data_ptr(),
                self.batch, self.out.data_ptr(), self.cloud_offsets.data_ptr(), self.status.data_ptr(),
                self.ws.data_ptr(), self.ws.numel(), _lib.current_stream())
        _lib.check(st, "d3b_frustum_crop_dev")
        return self.out, self.cloud_offsets

