"""On-disk -> device ingest (SURVEY 8f.4): `LoadPointCloudFromFile` with the reference's registry name, constructor
and `__call__(res, info)` contract (det3d/datasets/pipelines/loading.py:67-124), the NuScenes multi-sweep merge done
on the GPU by d3b_ingest_sweeps_dev (csrc/ingest.cu).

File reading stays on the host (it is I/O): KITTI `.bin` = flat float32 [N, num_point_features] (:92-94), nuScenes
and Lyft `.bin` = float32 [N, 5] of which the first 4 columns are kept (`read_file`, :17-31; Lyft reads the
LIDAR_TOP file of `info["ref_info"]`, :128-158, and has no sweeps).  Everything after that --
the 1 m `remove_close` filter of the sweeps (:34-43), the float64 rigid transform (:55-58), the time-lag column and
the concatenation (:115-124) -- is one call over the raw bytes of all sweeps.  `res["lidar"]` receives the same
numpy fields as the reference (`points`, `times`, `combined`) plus `combined_cuda`, the device tensor the
voxelizer consumes directly (no second H2D copy).

`ingest_sweeps_batched` does the same for a batch of samples in one d3b_ingest_sweeps_dev call: the sweep table lives
in device memory and the per-sample cloud offsets stay there, in the form the voxelizer takes, so nothing between the
raw sweeps and the detections waits on the host (InferencePipeline.infer_sweeps).  `ingest_sweeps` is a batch of one.

With `BatchedIngest(gather=True)` the table also says at which raw row each sweep starts (sweep_src), so sweeps are
read where they already lie in device memory (the history slots of apis.SweepStream), and `stream_transforms` gives the
float64 key-frame transforms and lags of such a history.
"""
import collections
import ctypes as C
import numbers
from pathlib import Path

import numpy as np
import torch

from ... import _lib
from ...utils.staging import RowStager
from ..registry import PIPELINES


def read_file(path, tries=2, num_point_feature=4, keep_raw=False):
    """loading.py:17-31: float32 file, truncated to whole 5-float records; [n, num_point_feature] (or the raw
    [n, 5] records with keep_raw, which is what the device ingest uploads)."""
    points = None
    try_cnt = 0
    while points is None and try_cnt < tries:
        try_cnt += 1
        try:
            points = np.fromfile(path, dtype=np.float32)
            s = points.shape[0]
            if s % 5 != 0:
                points = points[: s - (s % 5)]
            points = points.reshape(-1, 5)
            if not keep_raw:
                points = points[:, :num_point_feature]
        except Exception:
            points = None
    return points


def ingest_sweeps(raw_sweeps, transforms, time_lags, radius=1.0, n_feat=4, device="cuda"):
    """raw_sweeps: list of float32 [n_s, 5] arrays, key frame first.  transforms[s]: 4x4 array or None;
    time_lags[s]: float.  The key frame (s = 0) is neither filtered nor transformed, as in the reference.
    Returns the device tensor [N, n_feat + 1] (x, y, z, .., time lag), input order preserved: ingest_sweeps_batched on
    a batch of one, cut to its exact length (one sync)."""
    points, offsets = ingest_sweeps_batched([(raw_sweeps, transforms, time_lags)], radius, n_feat, device)
    return points[:int(offsets[1])]              # API boundary: the reference returns exactly-sized arrays


MAX_SWEEPS = 16          # D3B_INGEST_MAX_SWEEPS: sweeps per sample, key frame included
MAX_BATCH = 64           # samples per batched ingest, as the voxelizer's batch


def check_sweep_samples(samples, n_feat=4):
    """Host-side validation of a batch of multi-sweep samples [(raw_sweeps, transforms, time_lags), ...] with
    ingest_sweeps' per-sample contract: raises ValueError, before anything is enqueued.  Raw sweeps are float32
    [n, raw_stride] numpy arrays or CPU tensors (pinned ones are copied to the device directly), one raw_stride for the
    whole batch.  Returns (raw_stride, per-sample lists of sweep sizes)."""
    samples = list(samples)
    if not 1 <= len(samples) <= MAX_BATCH:
        raise ValueError("a batch holds 1 to %d samples, got %d" % (MAX_BATCH, len(samples)))
    if n_feat < 3:
        raise ValueError("n_feat must be >= 3, got %d" % n_feat)
    stride, sizes = None, []
    for b, sample in enumerate(samples):
        if len(sample) != 3:
            raise ValueError("sample %d: expected (raw_sweeps, transforms, time_lags)" % b)
        raws, tms, lags = sample
        if not 1 <= len(raws) <= MAX_SWEEPS:
            raise ValueError("sample %d: %d sweeps, expected 1 to %d (key frame included)" % (b, len(raws), MAX_SWEEPS))
        if len(tms) != len(raws) or len(lags) != len(raws):
            raise ValueError("sample %d: %d sweeps but %d transforms and %d time lags" % (b, len(raws), len(tms), len(lags)))
        for s, r in enumerate(raws):
            if torch.is_tensor(r):
                ok = r.dtype == torch.float32 and r.device.type == "cpu"
            else:
                ok = isinstance(r, np.ndarray) and r.dtype == np.float32
            if not ok or r.ndim != 2:
                raise ValueError("sample %d sweep %d: raw points must be a 2-D float32 host array" % (b, s))
            stride = int(r.shape[1]) if stride is None else stride
            if int(r.shape[1]) != stride:
                raise ValueError("sample %d sweep %d: raw stride %d, the batch has %d" % (b, s, r.shape[1], stride))
        for s, t in enumerate(tms):
            if t is not None and np.shape(t) != (4, 4):
                raise ValueError("sample %d sweep %d: transform must be 4x4 or None, got shape %s" % (b, s, np.shape(t)))
        if np.asarray(lags, dtype=np.float64).shape != (len(raws),):
            raise ValueError("sample %d: time lags must be %d numbers" % (b, len(raws)))
        sizes.append([int(r.shape[0]) for r in raws])
    if stride < n_feat:
        raise ValueError("raw_stride %d < n_feat %d" % (stride, n_feat))
    if sum(map(sum, sizes)) > 1 << 30:
        raise ValueError("more than 2^30 raw points in one batch")
    return stride, sizes


def sweep_table_capacity(n_sweeps, batch):
    """Sweep capacity of a batched ingest's device table: the smallest power of two >= n_sweeps, at most 16 * batch."""
    return min(1 << (max(int(n_sweeps), 1) - 1).bit_length(), MAX_SWEEPS * batch)


def sweep_table_views(buf, sweep_capacity, batch, gather=False):
    """Typed views over one byte buffer (numpy or torch) holding a device sweep table, laid out as
    transforms f64 [S, 16] | sweep_offsets i32 [S + 1] | sample_sweeps i32 [B + 1] | time_lag f32 [S] | flags u8 [S],
    with sweep_src i32 [S] after sample_sweeps when `gather`."""
    S, B = sweep_capacity, batch
    parts = (("transforms", 8, S * 16), ("sweep_offsets", 4, S + 1), ("sample_sweeps", 4, B + 1)) \
        + ((("sweep_src", 4, S),) if gather else ()) + (("time_lag", 4, S), ("flags", 1, S))
    views, at = {}, 0
    is_np = isinstance(buf, np.ndarray)
    for name, size, count in parts:
        raw = buf[at:at + size * count]
        dt = {8: np.float64, 4: np.float32 if name == "time_lag" else np.int32, 1: np.uint8}[size]
        views[name] = raw.view(dt) if is_np else raw.view(_TORCH_DTYPE[dt])
        at += size * count
    return views


_TORCH_DTYPE = {np.float64: torch.float64, np.float32: torch.float32, np.int32: torch.int32, np.uint8: torch.uint8}


def sweep_table_bytes(sweep_capacity, batch, gather=False):
    return sweep_capacity * (16 * 8 + 4 + 4 + 1 + (4 if gather else 0)) + 4 * (batch + 2)


def fill_sweep_table(views, samples, sizes):
    """Writes the table of `samples` (validated by check_sweep_samples) into host views (sweep_table_views).  As
    ingest_sweeps: the key frame (sweep 0 of each sample) is never filtered, its transform and lag are used as given."""
    for v in views.values():
        v[:] = 0
    s = 0
    rows = 0
    views["sweep_offsets"][0] = 0
    views["sample_sweeps"][0] = 0
    for b, ((_raws, tms, lags), n) in enumerate(zip(samples, sizes)):
        lags = np.asarray(lags, np.float64).astype(np.float32)         # times.astype(points.dtype), loading.py:119
        for j, t in enumerate(tms):
            if t is not None:
                views["transforms"][s * 16:(s + 1) * 16] = np.asarray(t, np.float64).reshape(16)
            views["flags"][s] = (1 if t is not None else 0) | (2 if j > 0 else 0)
            views["time_lag"][s] = lags[j]
            rows += n[j]
            views["sweep_offsets"][s + 1] = rows
            s += 1
        views["sample_sweeps"][b + 1] = s
    views["sweep_offsets"][s + 1:] = rows         # unused table rows: empty sweeps past the last sample


def stream_transforms(poses, timestamps):
    """Key-frame transforms and time lags of one sweep history, newest (the key frame) first: poses are sensor-to-world
    4x4 float64 matrices, timestamps in seconds.  Sweep s > 0 gets inv(P_key) @ P_s in float64 (its points to the key
    frame's sensor frame), the key frame None; lags are t_key - t_s (the table rounds them to float32 once).  Returns
    (transforms, time_lags) in ingest_sweeps' form."""
    key_inv = np.linalg.inv(np.asarray(poses[0], np.float64))
    tms = [None] + [key_inv @ np.asarray(p, np.float64) for p in poses[1:]]
    t_key = float(timestamps[0])
    return tms, [t_key - float(t) for t in timestamps]


class SweepHistory:
    """Host bookkeeping of B sweep histories of K sweeps each, kept in S >= K slots per stream (apis.SweepStream keeps
    the sweeps themselves on the device).  A push goes to slot (pushes since the last reset) mod S of its stream, so
    the slot it overwrites held the stream's (S - K + 1)-th oldest sweep once S sweeps were pushed; reset(b) forgets
    stream b's sweeps.

    Frames that have not finished -- they may still have to be re-run from their slots -- hold their slots (acquire /
    release); check_free refuses a push into a held slot.  With S = K + k - 1 a push finds its slot free while at most
    k - 1 frames are unfinished, so with one more frame submitted after the push, k frames can be in flight."""

    def __init__(self, batch, history, slots=None):
        self.batch, self.history = batch, history
        self.slots = history if slots is None else int(slots)
        if self.slots < history:
            raise ValueError("%d slots cannot hold a history of %d sweeps" % (self.slots, history))
        self.count = [0] * batch                  # pushes since the last reset
        # per stream, oldest first: (slot, rows, pose f64 [4, 4], timestamp) of the sweeps still held
        self.held = [collections.deque(maxlen=history) for _ in range(batch)]
        self.readers = [[0] * self.slots for _ in range(batch)]      # unfinished frames reading each slot

    def check_stream(self, b):
        if not isinstance(b, numbers.Integral) or not 0 <= b < self.batch:
            raise ValueError("stream index %r outside [0, %d)" % (b, self.batch))

    def next_slot(self, b):
        return self.count[b] % self.slots

    def check_free(self, b):
        """ValueError when stream b's next push would overwrite a slot an unfinished frame reads."""
        slot = self.next_slot(b)
        if self.readers[b][slot]:
            raise ValueError("stream %d: the next push would overwrite slot %d, which %d unfinished frame(s) read; "
                             "collect the oldest frame's result first (or give the stream more in_flight)"
                             % (b, slot, self.readers[b][slot]))

    def acquire(self, frame):
        """Marks the slots of `frame` (frame()'s value) as read by one more unfinished frame.  Returns the
        (stream, slot) pairs to pass to release once that frame has finished."""
        held = [(b, k) for b, (ks, _ns, _tms, _lags) in enumerate(frame) for k in ks]
        for b, k in held:
            self.readers[b][k] += 1
        return held

    def release(self, held):
        for b, k in held:
            self.readers[b][k] -= 1

    def record(self, b, rows, pose, timestamp):
        """Books stream b's new sweep into next_slot(b), which it returns."""
        slot = self.next_slot(b)
        self.held[b].append((slot, int(rows), np.array(pose, dtype=np.float64), float(timestamp)))
        self.count[b] += 1
        return slot

    def reset(self, b):
        self.check_stream(b)
        self.count[b] = 0
        self.held[b].clear()

    def frame(self):
        """The current frame: per stream (slots, rows, transforms, time_lags), newest sweep (the key frame) first, with
        stream_transforms' transforms and lags.  ValueError when a stream holds no sweep."""
        out = []
        for b, held in enumerate(self.held):
            if not held:
                raise ValueError("stream %d has no sweep: push one before inferring" % b)
            newest = list(reversed(held))
            tms, lags = stream_transforms([h[2] for h in newest], [h[3] for h in newest])
            out.append(([h[0] for h in newest], [h[1] for h in newest], tms, lags))
        return out


def stage_raw_sweeps(samples, sizes, raw_dev):
    """Enqueues the H2D copies of every raw sweep into raw_dev, back to back in sample order, through a RowStager of
    its own.  `sizes` (check_sweep_samples') is not read: each array's shape gives its rows.  Returns the number of
    rows."""
    return RowStager().put([r for raws, _tms, _lags in samples for r in raws], raw_dev)


class BatchedIngest:
    """Device buffers of one batched-ingest shape -- raw [raw_capacity, raw_stride], the sweep table, the ingested
    clouds [raw_capacity, n_feat + 1], cloud_offsets [B + 1], status, workspace -- and the d3b_ingest_sweeps_dev call
    over them.  The addresses never change, so a captured CUDA graph can hold them.  With `gather` the table also holds
    sweep_src (the raw row where each sweep starts), which launch() passes; without it each sweep starts at its offset."""

    def __init__(self, batch, raw_capacity, sweep_capacity, raw_stride, n_feat=4, radius=1.0, device="cuda",
                 gather=False):
        dev = torch.device(device)
        self.batch, self.raw_capacity, self.sweep_capacity = batch, raw_capacity, sweep_capacity
        self.raw_stride, self.n_feat, self.radius, self.gather = raw_stride, n_feat, radius, gather
        self.raw = torch.empty((raw_capacity, raw_stride), dtype=torch.float32, device=dev)   # rows no sweep covers are never read
        self.table = torch.zeros(sweep_table_bytes(sweep_capacity, batch, gather), dtype=torch.uint8, device=dev)
        self.tables = sweep_table_views(self.table, sweep_capacity, batch, gather)
        self.out = torch.empty((raw_capacity, n_feat + 1), dtype=torch.float32, device=dev)
        self.cloud_offsets = torch.zeros(batch + 1, dtype=torch.int32, device=dev)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self.ws = torch.empty(_lib.lib().d3b_ingest_dev_workspace_bytes(raw_capacity, sweep_capacity), dtype=torch.uint8,
                              device=dev)

    def host_table(self, samples, sizes, out=None, sweep_src=None):
        """The table image of `samples` as uint8 host bytes (into `out`, e.g. a pinned buffer, when given).  A gather
        table takes sweep_src, the raw start row of every sweep in sample order (unused rows stay 0)."""
        buf = np.zeros(self.table.numel(), np.uint8) if out is None else out
        views = sweep_table_views(buf, self.sweep_capacity, self.batch, self.gather)
        fill_sweep_table(views, samples, sizes)
        if self.gather:
            src = np.asarray([] if sweep_src is None else sweep_src, np.int64)
            if src.shape != (sum(map(len, sizes)),):
                raise ValueError("a gather table needs one sweep_src per sweep (%d), got %s"
                                 % (sum(map(len, sizes)), src.shape))
            views["sweep_src"][:src.shape[0]] = src
        return buf

    def launch(self):
        """Ingests the raw sweeps under the device table into out / cloud_offsets (three kernels, no host sync)."""
        t = self.tables
        with _lib.on_device_of(self.raw), _lib.timed("ingest_sweeps", batch=self.batch, capacity=self.raw_capacity):
            st = _lib.lib().d3b_ingest_sweeps_dev(
                self.raw.data_ptr(), self.raw_capacity, self.raw_stride, self.n_feat, t["sweep_offsets"].data_ptr(),
                _lib.ptr(t.get("sweep_src")), t["sample_sweeps"].data_ptr(), t["transforms"].data_ptr(),
                t["time_lag"].data_ptr(), t["flags"].data_ptr(), self.sweep_capacity, self.batch, C.c_float(self.radius),
                self.out.data_ptr(), self.cloud_offsets.data_ptr(), self.status.data_ptr(), self.ws.data_ptr(),
                self.ws.numel(), _lib.current_stream())
        _lib.check(st, "d3b_ingest_sweeps_dev")
        return self.out, self.cloud_offsets


def ingest_sweeps_batched(samples, radius=1.0, n_feat=4, device="cuda", capacity=None, return_ingest=False):
    """Batched ingest_sweeps: samples = [(raw_sweeps, transforms, time_lags), ...], each with ingest_sweeps' contract
    (key frame first; it is neither filtered nor transformed unless a transform is given).  One d3b_ingest_sweeps_dev
    call, no host sync.  Returns (points [capacity, n_feat + 1], cloud_offsets int32 [B + 1]), both on the device:
    sample b's cloud is points[cloud_offsets[b]:cloud_offsets[b + 1]], the bits that sample gives alone (ingest_sweeps);
    rows past cloud_offsets[B] are undefined.  capacity (default: the raw total) must be >= the raw total."""
    if not torch.cuda.is_available():
        raise RuntimeError("det3d_b200: the multi-sweep ingest needs a CUDA device (there is no CPU fallback)")
    samples = list(samples)
    stride, sizes = check_sweep_samples(samples, n_feat)
    total = sum(map(sum, sizes))
    capacity = max(total, 1) if capacity is None else int(capacity)
    if capacity < total:
        raise ValueError("capacity %d < %d raw points" % (capacity, total))
    ing = BatchedIngest(len(samples), capacity, sweep_table_capacity(sum(map(len, sizes)), len(samples)), stride,
                        n_feat, radius, device)
    table = torch.empty(ing.table.numel(), dtype=torch.uint8, pin_memory=True)
    ing.host_table(samples, sizes, out=table.numpy())
    with torch.cuda.device(ing.raw.device):
        ing.table.copy_(table, non_blocking=True)
        stage_raw_sweeps(samples, sizes, ing.raw)
        points, offsets = ing.launch()
    return (points, offsets, ing) if return_ingest else (points, offsets)


@PIPELINES.register_module
class LoadPointCloudFromFile(object):
    def __init__(self, dataset="KittiDataset", **kwargs):
        self.type = dataset
        self.random_select = kwargs.get("random_select", False)
        self.npoints = kwargs.get("npoints", 16834)
        self.device = kwargs.get("device", "cuda")

    def __call__(self, res, info):
        res["type"] = self.type
        if self.type == "KittiDataset":
            pc_info = info["point_cloud"]
            velo_path = Path(pc_info["velodyne_path"])
            if not velo_path.is_absolute():
                velo_path = Path(res["metadata"]["image_prefix"]) / pc_info["velodyne_path"]
            reduced = velo_path.parent.parent / (velo_path.parent.stem + "_reduced") / velo_path.name
            if reduced.exists():
                velo_path = reduced
            points = np.fromfile(str(velo_path), dtype=np.float32, count=-1).reshape(
                [-1, res["metadata"]["num_point_features"]])
            res["lidar"]["points"] = points
        elif self.type == "NuScenesDataset":
            nsweeps = res["lidar"]["nsweeps"]
            raws = [read_file(str(Path(info["lidar_path"])), keep_raw=True)]
            transforms, lags = [None], [0.0]
            assert (nsweeps - 1) <= len(info["sweeps"]), "nsweeps {} should not greater than list length {}.".format(
                nsweeps, len(info["sweeps"]))
            for i in np.random.choice(len(info["sweeps"]), nsweeps - 1, replace=False):      # same RNG call as :110
                sweep = info["sweeps"][i]
                raws.append(read_file(str(sweep["lidar_path"]), keep_raw=True))
                transforms.append(sweep["transform_matrix"])
                lags.append(sweep["time_lag"])
            combined = ingest_sweeps(raws, transforms, lags, radius=1.0, n_feat=4, device=self.device)
            host = combined.cpu().numpy()
            res["lidar"]["points"] = host[:, :4]
            res["lidar"]["times"] = host[:, 4:5]
            res["lidar"]["combined"] = host
            res["lidar"]["combined_cuda"] = combined
        elif self.type == "LyftDataset":
            # loading.py:128-158: the top lidar only (the side-lidar merge there is commented out); read_file keeps
            # x, y, z, intensity of each 5-float record and drops a trailing partial record
            res["lidar"]["points"] = read_file(info["ref_info"]["LIDAR_TOP"]["lidar_path"])
        else:
            raise NotImplementedError("LoadPointCloudFromFile: dataset type %s" % self.type)
        return res, info


def _kitti_boxes_camera_to_lidar(annos, r_rect, velo2cam):
    """location/dimensions/rotation_y (camera frame, bottom-centre) -> lidar boxes [n,7] x,y,z,w,l,h,r with the
    gravity centre: box_np_ops.box_camera_to_lidar + change_box3d_center_ (box_np_ops.py:909-930,1346-1349)."""
    gt = np.concatenate([annos["location"], annos["dimensions"], annos["rotation_y"][..., np.newaxis]], axis=1).astype(np.float32)
    xyz = np.concatenate([gt[:, 0:3], np.ones((gt.shape[0], 1))], axis=-1)
    xyz_lidar = (xyz @ np.linalg.inv((r_rect @ velo2cam).T))[..., :3]
    l, h, w, r = gt[:, 3:4], gt[:, 4:5], gt[:, 5:6], gt[:, 6:7]
    boxes = np.concatenate([xyz_lidar, w, l, h, r], axis=1)
    boxes[..., :3] += boxes[..., 3:6] * (np.array([0.5, 0.5, 0.5], boxes.dtype) - np.array([0.5, 0.5, 0], boxes.dtype))
    return boxes


@PIPELINES.register_module
class LoadPointCloudAnnotations(object):
    """det3d/datasets/pipelines/loading.py:165-224: calibration + (when the info record has them) ground-truth boxes
    for evaluation.  Host metadata only -- nothing here is on the compute path."""

    def __init__(self, with_bbox=True, **kwargs):
        pass

    def __call__(self, res, info):
        if res["type"] in ["NuScenesDataset", "LyftDataset"] and "gt_boxes" in info:
            res["lidar"]["annotations"] = {
                "boxes": info["gt_boxes"].astype(np.float32),
                "names": info["gt_names"],
                "tokens": info["gt_boxes_token"],
                "velocities": info["gt_boxes_velocity"].astype(np.float32),
            }
        elif res["type"] == "KittiDataset":
            calib = info["calib"]
            res["calib"] = {"rect": calib["R0_rect"], "Trv2c": calib["Tr_velo_to_cam"], "P2": calib["P2"]}
            if "annos" in info:
                annos = info["annos"]
                keep = [i for i, x in enumerate(annos["name"]) if x != "DontCare"]       # kitti_common.remove_dontcare
                annos = {k: v[keep] for k, v in annos.items()}
                res["lidar"]["annotations"] = {
                    "boxes": _kitti_boxes_camera_to_lidar(annos, calib["R0_rect"], calib["Tr_velo_to_cam"]),
                    "names": annos["name"],
                }
                res.setdefault("cam", {})["annotations"] = {"boxes": annos["bbox"], "names": annos["name"]}
        elif res["type"] in ["NuScenesDataset", "LyftDataset"]:
            pass
        else:
            raise NotImplementedError("LoadPointCloudAnnotations: dataset type %r" % (res["type"],))
        return res, info
