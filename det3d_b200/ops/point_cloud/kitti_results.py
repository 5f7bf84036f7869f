"""Device KITTI result rows: torch wrapper over d3b_kitti_results_dev (csrc/kitti_results.cu).

Reference semantics: det3d/datasets/kitti/kitti.py:78-158 (KittiDataset.convert_detection_to_kitti_annos).  The per-box
conversion and the in-image filter run on the device; `calib_table` (numpy, once per calibration) and `to_annos` (the
reference's anno dicts from the kept rows) run on the host.
"""
import numpy as np
import torch

from ... import _lib

MAX_BATCH = 64
CALIB_DOUBLES = 32
COLS = 14                 # bbox 4, alpha, dimensions 3, location 3, rotation_y, score, label
ANNO_KEYS = ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score")


def check_calibs(calibs):
    """Host-side validation of KITTI calibrations dict(rect, Trv2c, P2, image_shape): raises ValueError."""
    for b, cal in enumerate(calibs):
        if not isinstance(cal, dict) or not all(k in cal for k in ("rect", "Trv2c", "P2", "image_shape")):
            raise ValueError("calibration %d: expected dict(rect, Trv2c, P2, image_shape)" % b)
        if np.shape(cal["rect"]) != (4, 4) or np.shape(cal["Trv2c"]) != (4, 4):
            raise ValueError("calibration %d: rect and Trv2c must be 4x4 (the info files' extended form)" % b)
        if np.shape(cal["P2"]) not in ((3, 4), (4, 4)):
            raise ValueError("calibration %d: P2 must be 3x4 or 4x4, got shape %s" % (b, np.shape(cal["P2"])))
        shape = np.asarray(cal["image_shape"]).reshape(-1)
        if shape.shape[0] < 2 or not np.all(shape[:2] > 0):
            raise ValueError("calibration %d: image_shape must be (H, W) > 0, got %r" % (b, cal["image_shape"]))


def calib_table(calib):
    """float64 [32], the kernel's calibration row: M = rect @ Trv2c with numpy's own matmul (the reference's
    lidar_to_camera forms the same product, so these are its bits), P2's rows 0..2, then the image's H and W."""
    t = np.zeros(CALIB_DOUBLES)
    t[:16] = (np.asarray(calib["rect"]) @ np.asarray(calib["Trv2c"])).reshape(-1)
    t[16:28] = np.asarray(calib["P2"], np.float64)[:3].reshape(-1)
    shape = np.asarray(calib["image_shape"]).reshape(-1)
    t[28], t[29] = shape[0], shape[1]
    return t


def empty_result_anno():
    """The reference's anno of a frame with no kept detection (kitti_common.empty_result_anno)."""
    return dict(name=np.array([]), truncated=np.array([]), occluded=np.array([]), alpha=np.array([]),
                bbox=np.zeros([0, 4]), dimensions=np.zeros([0, 3]), location=np.zeros([0, 3]), rotation_y=np.array([]),
                score=np.array([]))


def to_annos(results, counts, class_names):
    """Host results [B, D, 14] f64 and counts [B] -> one anno dict per frame with the reference's keys and dtypes (names
    str, truncated f64, occluded int64, alpha f64, bbox f64 [n, 4], dimensions / location f64 [n, 3], rotation_y f64,
    score f32), or empty_result_anno() for a frame with none.  The arrays are copies."""
    names = np.empty(len(class_names), object)
    names[:] = list(class_names)
    annos = []
    for rows, n in zip(np.asarray(results), np.asarray(counts)):
        n = int(n)
        if n == 0:
            annos.append(empty_result_anno())
            continue
        r = rows[:n]
        # np.array of the names as a list: its dtype is as wide as the longest name kept, not the longest class
        annos.append(dict(name=np.array(names[r[:, 13].astype(np.int64)].tolist()), truncated=np.zeros(n),
                          occluded=np.zeros(n, np.int64), alpha=r[:, 4].copy(), bbox=r[:, 0:4].copy(),
                          dimensions=r[:, 5:8].copy(), location=r[:, 8:11].copy(), rotation_y=r[:, 11].copy(),
                          score=r[:, 12].astype(np.float32)))
    return annos


class KittiResults:
    """Static device buffers of one batch -- the calibration table f64 [B, 32], results f64 [B, D, 14], counts i32 [B]
    -- their pinned host copies, and the d3b_kitti_results_dev call over them.  The results buffers are sized by the
    first detections launched on (D and nd are the model's); the addresses never change after that, so a captured CUDA
    graph can hold them."""

    def __init__(self, batch, device="cuda"):
        if not 1 <= batch <= MAX_BATCH:
            raise ValueError("batch must be in [1, %d], got %d" % (MAX_BATCH, batch))
        self.batch, self.device = batch, torch.device(device)
        self.calib = torch.zeros((batch, CALIB_DOUBLES), dtype=torch.float64, device=self.device)
        self.results = self.counts = None
        self.results_host = self.counts_host = None

    def set_calib(self, table):
        """Synchronous copy of a host table [B, 32] into the device buffer (graphs stage it through pinned memory
        instead: apis.pipeline)."""
        self.calib.copy_(torch.as_tensor(np.asarray(table, np.float64)))

    def launch(self, packed):
        """packed [B, D, nd + 3] f32 device detections (predict's box, score, label, valid) -> (results, counts), one
        kernel, no host sync."""
        B, D, width = packed.shape
        if B != self.batch or packed.dtype != torch.float32 or not packed.is_contiguous():
            raise ValueError("detections must be contiguous f32 [%d, D, nd + 3], got %s %s"
                             % (self.batch, tuple(packed.shape), packed.dtype))
        if self.results is None or self.results.shape[1] != D:
            self.results = torch.zeros((B, D, COLS), dtype=torch.float64, device=self.device)
            self.counts = torch.zeros(B, dtype=torch.int32, device=self.device)
            self.results_host = torch.empty(self.results.shape, dtype=torch.float64, pin_memory=True)
            self.counts_host = torch.empty(B, dtype=torch.int32, pin_memory=True)
        L = _lib.lib()
        with _lib.on_device_of(packed, self.calib), _lib.timed("kitti_results", batch=B, max_det=D):
            st = L.d3b_kitti_results_dev(packed.data_ptr(), self.calib.data_ptr(), B, D, width - 3,
                                         self.results.data_ptr(), self.counts.data_ptr(), _lib.current_stream())
        _lib.check(st, "d3b_kitti_results_dev")
        return self.results, self.counts
