"""End-to-end, device-resident inference: raw points -> detections.

The reference splits this path between DataLoader worker processes (numba voxelizer,
per-sample CPU anchor generation, numpy collate; det3d/datasets/pipelines/preprocess.py:
259-304,346-378, det3d/torchie/parallel/collate.py:90-150), the GPU model
(det3d/models/detectors/voxelnet.py:30-52) and a CPU NMS (core/bbox/box_torch_ops.py:
528-549).  `InferencePipeline` keeps the same stages and the same model objects (built
from an unmodified Det3D config through the registries) but runs every stage on the GPU
with fixed-shape buffers: points are voxelized for the whole batch in one call with the
batch index and the VoxelFeatureExtractorV3 mean fused in, anchors are generated once
and cached on the device, and detections come back as fixed-shape tensors.
"""
import collections
import numbers
import warnings

import numpy as np
import torch

from det3d_b200 import _lib
from det3d_b200.core.anchor.anchor_generator import anchors_for_tasks
from det3d_b200.datasets.pipelines.loading import (MAX_BATCH, MAX_SWEEPS, BatchedIngest, SweepHistory,
                                                    check_sweep_samples, ingest_sweeps_batched, stage_raw_sweeps,
                                                    sweep_table_capacity)
from det3d_b200.models import build_detector
from det3d_b200.ops.point_cloud.voxelize import Voxelizer


class InferencePipeline:
    def __init__(self, cfg, model=None, device="cuda", strict_fp32=True):
        self.cfg = cfg
        self.device = torch.device(device)
        if model is None:
            model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
        self.model = model.to(self.device).eval()
        vg = cfg.voxel_generator
        # VoxelFeatureExtractorV3 only needs the per-voxel mean (fused into the voxelizer); the pillar reader
        # consumes the point slots themselves
        self._reader_takes_points = cfg.model["reader"]["type"] != "VoxelFeatureExtractorV3"
        # a pillar reader that can walk the voxelizer's point-index lists does not need the [M, P, ndim] tensor either
        self._reader_takes_lists = (self._reader_takes_points and hasattr(self.model.reader, "forward_lists")
                                    and len(getattr(self.model.reader, "pfn_layers", [])) == 1)
        self.voxelizer = Voxelizer(vg["voxel_size"], vg["range"], vg["max_points_in_voxel"], vg["max_voxel_num"],
                                   want_voxels=self._reader_takes_points and not self._reader_takes_lists,
                                   want_mean=not self._reader_takes_points)
        self.grid_size = self.voxelizer.grid_size
        self.num_point_features = int(cfg.model["reader"].get("num_input_features", 4))
        out_size_factor = cfg.assigner["out_size_factor"] if "assigner" in cfg else 8
        anchors = anchors_for_tasks(cfg.target_assigner, self.grid_size, out_size_factor)
        self._anchors = [torch.from_numpy(a).to(self.device) for a in anchors]
        self._anchor_cache = {}
        self.strict_fp32 = strict_fp32
        # (batch, bucket, ndim) -> _GraphEntry, (batch, raw bucket, table capacity, raw_stride, n_feat) ->
        # _SweepGraphEntry (infer_sweeps) and ("stream", B, K, slot_capacity, raw_stride, n_feat) -> _StreamGraphEntry
        # (SweepStream.infer), least recently used first
        self._graphs = collections.OrderedDict()
        self.max_graphs = 8
        self._ovf_host = None

    def anchors(self, batch):
        a = self._anchor_cache.get(batch)
        if a is None:
            a = self._anchor_cache[batch] = [t.unsqueeze(0).expand(batch, -1, -1).contiguous() for t in self._anchors]
        return a

    @torch.no_grad()
    def forward_device(self, points, offsets):
        """points [N_total, ndim] f32 on the device, offsets host list -> fixed-shape detections.

        `offsets` may also be an int32 device tensor [B+1]; points.shape[0] is then a capacity (Voxelizer)."""
        batch = len(offsets) - 1
        vox = self.voxelizer(points, offsets)
        example = dict(
            voxels=vox["voxels"] if self._reader_takes_points else vox["mean"], coordinates=vox["coors"], num_points=vox["num_points"],
            num_voxels=[None] * batch, shape=[self.grid_size], anchors=self.anchors(batch),
            n_voxels_dev=vox["counts"][batch:batch + 1],
        )
        if self._reader_takes_lists:
            example["point_lists"] = dict(vox["point_lists"], counts=vox["counts"])
        prev, prev_bench = torch.backends.cudnn.allow_tf32, torch.backends.cudnn.benchmark
        if self.strict_fp32:
            torch.backends.cudnn.allow_tf32 = False
        # shapes are static per pipeline: let cuDNN pick its fastest fp32 algorithm for the dense layers that stay on it
        # (strided / multi-stage RPNs: PointPillars, CBGS)
        torch.backends.cudnn.benchmark = True
        try:
            det = self.model(example, return_loss=False, device_output=True)
        finally:
            torch.backends.cudnn.allow_tf32 = prev
            torch.backends.cudnn.benchmark = prev_bench
        det["voxel_counts"] = vox["counts"]
        return det

    # ---- f16-range guard of the FP16x3 kernels -------------------------------------------------------------------
    def overflow_flag(self):
        """Device int32[1]: nonzero once a feature left the f16 range (the FP16x3 kernels never saturate silently)."""
        flag = getattr(self.model, "overflow_flag", None)
        return None if flag is None else flag(self.device)

    def set_math(self, math):
        """Switch the model's convolutions to `math` ("fp16x3", the default; "fp16", single-pass FP16; or "tf32x3") and
        drop the captured graphs: a graph replays the kernels it was captured with, so one captured under another math
        would keep running that math."""
        self.model.set_math(math)
        self._graphs.clear()

    def check_overflow(self, flag_value):
        """Host side of the guard: on a raised flag switch the model to the tf32x3 kernels (permanently: the weights /
        inputs that overflowed once will again) and tell the caller to re-run.  Returns True if a re-run is needed.
        The tf32x3 kernels are output-stationary like the FP16x3 ones, so re-run results are reproducible bit for bit."""
        if not flag_value:
            return False
        warnings.warn("det3d_b200: a feature left the f16 range (|x| >= 65504); re-running on the tf32x3 kernels")
        self.model.set_math("tf32x3")
        self.overflow_flag().zero_()
        self._graphs.clear()
        return True

    @staticmethod
    def bucket_of(n_points):
        """Point capacity of the graph that serves a batch of n_points: the smallest power of two >= max(n, 1024)."""
        return 1 << (max(int(n_points), 1024) - 1).bit_length()

    @staticmethod
    def check_offsets(offsets, n_points=None):
        """Host-side validation of cloud offsets [0, n0, n0+n1, ...]: raises ValueError, before anything is enqueued."""
        offsets = [int(o) for o in offsets]
        if not 2 <= len(offsets) <= 65:
            raise ValueError("offsets must hold batch + 1 entries with 1 <= batch <= 64, got %d" % len(offsets))
        if offsets[0] != 0:
            raise ValueError("offsets[0] must be 0, got %d" % offsets[0])
        if any(b < a for a, b in zip(offsets[:-1], offsets[1:])):
            raise ValueError("offsets must be non-decreasing: %s" % offsets)
        if n_points is not None and offsets[-1] != n_points:
            raise ValueError("offsets[-1] = %d but points has %d rows" % (offsets[-1], n_points))
        return offsets

    def _graph_entry(self, batch, n_points, ndim):
        """The graph of (batch, bucket, ndim), least recently used last; a new entry has buffers but no graph yet."""
        key = (batch, self.bucket_of(n_points), ndim)
        entry = self._graphs.get(key)
        if entry is not None:
            self._graphs.move_to_end(key)
            return entry
        while len(self._graphs) >= self.max_graphs:
            self._graphs.popitem(last=False)
        entry = self._graphs[key] = _GraphEntry(key[1], batch, ndim, self.device)
        return entry

    def _replay(self, entry, offsets):
        """Make the graph's device offsets `offsets`, capture the graph on first use, replay.  The clouds must already
        be in entry.points[:offsets[-1]]."""
        key = tuple(offsets)
        if entry.last_offsets != key:
            # the pinned staging buffer may still feed the previous copy: wait for that one before rewriting it
            entry.copied.synchronize()
            entry.staging.numpy()[:] = key
            entry.offsets.copy_(entry.staging, non_blocking=True)
            entry.copied.record()
            entry.last_offsets = key
        return self._run_graph(entry, lambda: self.pack(self.forward_device(entry.points, entry.offsets)))

    def _run_graph(self, entry, step):
        """Capture `step` (which returns the packed detections) into entry.graph on first use, then replay it."""
        if entry.graph is None:
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(3):                      # warm-up: lazy buffers, weight packing, cuDNN plans
                    step()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                entry.out = step()
                _lib.graph_mark("end")          # (bench.py's in-graph stage timing; nothing unless _lib.GRAPH_MARKS is set)
            entry.graph = graph
        entry.graph.replay()
        return entry.out

    @torch.no_grad()
    def forward_graphed(self, points, offsets):
        """forward_device + pack replayed from a CUDA graph.

        Every stage has static shapes and device-resident counts, and the voxelizer reads the cloud offsets from a
        device tensor, so the whole forward -- ~50 det3d_b200 launches plus the torch glue -- is one graph launch, and
        one graph per (batch, bucket, ndim) serves clouds of any size: `bucket` (bucket_of) is the point capacity of the
        graph's static input buffer.  `offsets` is a host list [0, n0, n0+n1, ...] (ValueError if malformed); it is
        copied to the device only when it differs from the graph's previous replay.  `points` [offsets[-1], ndim] may
        live on the host (pinned) or the device; it is copied into the graph's static input buffer.
        Returns the packed detections [B, D, nd+3] (a static buffer: consume before the next call)."""
        offsets = self.check_offsets(offsets, points.shape[0])
        entry = self._graph_entry(len(offsets) - 1, offsets[-1], points.shape[1])
        entry.points[:offsets[-1]].copy_(points, non_blocking=True)
        return self._replay(entry, offsets)

    @staticmethod
    def pack(det):
        """-> one [B, D, nd+3] f32 tensor: box, score, label, valid (the D2H / all-gather payload)."""
        if "packed" in det:
            return det["packed"]
        return torch.cat([det["boxes"], det["scores"].unsqueeze(-1), det["labels"].float().unsqueeze(-1),
                          det["valid"].float().unsqueeze(-1)], dim=-1).contiguous()

    @torch.no_grad()
    def infer_host(self, clouds, pinned_out=None, graphed=False):
        """clouds: list of pinned (or plain) host float32 tensors [N_i, ndim].
        H2D copy, forward, D2H of the packed detections.  Returns a host tensor [B, D, nd+3].
        graphed=True copies the clouds into the static input of the (batch, bucket) graph and replays it
        (forward_graphed); the detections are the same bits."""
        offsets = [0]
        for c in clouds:
            offsets.append(offsets[-1] + c.shape[0])
        ndim = clouds[0].shape[1]
        if graphed:
            self.check_offsets(offsets)
        else:
            pts = torch.empty((offsets[-1], ndim), dtype=torch.float32, device=self.device)
            for c, a, b in zip(clouds, offsets[:-1], offsets[1:]):
                pts[a:b].copy_(c, non_blocking=True)
        for _attempt in range(2):
            if graphed:         # (a re-run after an overflow captures a new graph: check_overflow dropped them all)
                entry = self._graph_entry(len(clouds), offsets[-1], ndim)
                for c, a, b in zip(clouds, offsets[:-1], offsets[1:]):
                    entry.points[a:b].copy_(c, non_blocking=True)
                packed = self._replay(entry, offsets)
            else:
                packed = self.pack(self.forward_device(pts, offsets))
            pinned_out, rerun = self._fetch(packed, pinned_out)
            if not rerun:
                break
        return pinned_out

    def _fetch(self, packed, pinned_out):
        """D2H of the packed detections and of the f16-range flag, then one sync.  Returns (pinned_out, rerun): rerun is
        True when the flag was raised and the model has switched to tf32x3 (check_overflow)."""
        if pinned_out is None:
            pinned_out = torch.empty(packed.shape, dtype=torch.float32, pin_memory=True)
        pinned_out.copy_(packed, non_blocking=True)
        flag = self.overflow_flag()
        if flag is not None:
            if self._ovf_host is None:
                self._ovf_host = torch.zeros(1, dtype=torch.int32, pin_memory=True)
            self._ovf_host.copy_(flag, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return pinned_out, flag is not None and self.check_overflow(int(self._ovf_host[0]))

    @torch.no_grad()
    def infer_sweeps(self, samples, pinned_out=None, graphed=False, n_feat=4, radius=1.0):
        """Multi-sweep samples -> host detections [B, D, nd+3], as infer_host.

        samples: [(raw_sweeps, transforms, time_lags), ...], one per cloud, each with ingest_sweeps' contract (raw
        float32 [n, raw_stride] host arrays or pinned tensors, key frame first and neither filtered nor transformed
        unless given a transform; 4x4 or None transforms; one time lag per sweep).  One batched ingest
        (d3b_ingest_sweeps_dev) writes the clouds and their device offsets, which the voxelizer reads directly: no host
        sync before the D2H of the detections.  graphed=True replays one CUDA graph covering ingest, voxelize and
        forward per (B, raw bucket, sweep-table capacity, raw_stride, n_feat) (bucket_of of the raw total); the raw
        sweeps are copied into its static raw buffer and the sweep table is copied H2D only when it changed.  Raises
        ValueError before anything is enqueued when the samples are malformed or n_feat + 1 is not the reader's
        feature count.  The overflow fallback is infer_host's."""
        if n_feat + 1 != self.num_point_features:
            raise ValueError("ingested clouds have n_feat + 1 = %d features, the reader takes %d"
                             % (n_feat + 1, self.num_point_features))
        samples = list(samples)
        stride, sizes = check_sweep_samples(samples, n_feat)
        batch, total = len(samples), sum(map(sum, sizes))
        bucket = self.bucket_of(total)
        table_cap = sweep_table_capacity(sum(map(len, sizes)), batch)
        if not graphed:
            # the voxelizer keeps its device-offset buffers per capacity: the bucket bounds how many it keeps
            points, cloud_offsets = ingest_sweeps_batched(samples, radius, n_feat, self.device, capacity=bucket)
        for _attempt in range(2):
            if graphed:         # (a re-run after an overflow captures a new graph: check_overflow dropped them all)
                entry = self._sweep_graph_entry(batch, bucket, table_cap, stride, n_feat, radius)
                entry.stage(samples, sizes)
                ing = entry.ingest
                packed = self._run_graph(entry, lambda: self.pack(self.forward_device(*ing.launch())))
            else:
                packed = self.pack(self.forward_device(points, cloud_offsets))
            pinned_out, rerun = self._fetch(packed, pinned_out)
            if not rerun:
                break
        return pinned_out

    def _sweep_graph_entry(self, batch, bucket, table_cap, raw_stride, n_feat, radius):
        """The infer_sweeps graph of (batch, bucket, table_cap, raw_stride, n_feat), in the LRU of forward_graphed."""
        key = (batch, bucket, table_cap, raw_stride, n_feat)
        entry = self._graphs.get(key)
        if entry is not None and entry.ingest.radius == radius:
            self._graphs.move_to_end(key)
            return entry
        self._graphs.pop(key, None)
        while len(self._graphs) >= self.max_graphs:
            self._graphs.popitem(last=False)
        entry = self._graphs[key] = _SweepGraphEntry(BatchedIngest(batch, bucket, table_cap, raw_stride, n_feat, radius,
                                                                   self.device))
        return entry

    @staticmethod
    def unpack(packed_host):
        """host [B, D, nd+3] -> list of dict(box3d_lidar, scores, label_preds) per sample."""
        out = []
        for row in packed_host:
            m = row[:, -1] > 0.5
            out.append(dict(box3d_lidar=row[m, :-3], scores=row[m, -3], label_preds=row[m, -2].long()))
        return out


class _GraphEntry:
    """Static buffers of one captured forward: points [bucket, ndim], device offsets [batch + 1] and their pinned
    staging copy, the graph and its packed output."""

    def __init__(self, bucket, batch, ndim, device):
        self.points = torch.zeros((bucket, ndim), dtype=torch.float32, device=device)
        self.offsets = torch.zeros(batch + 1, dtype=torch.int32, device=device)
        self.staging = torch.zeros(batch + 1, dtype=torch.int32, pin_memory=True)
        self.copied = torch.cuda.Event()
        self.last_offsets = None
        self.graph = None
        self.out = None


class _SweepGraphEntry:
    """Static buffers of one captured infer_sweeps forward: the BatchedIngest (raw sweeps, sweep table, clouds, cloud
    offsets), the pinned staging of the table and of raw sweeps that are not pinned already, the graph and its output."""

    def __init__(self, ingest):
        self.ingest = ingest
        self.table_staging = torch.zeros(ingest.table.numel(), dtype=torch.uint8, pin_memory=True)
        self.raw_staging = None
        self.copied = torch.cuda.Event()
        self.last_table = None
        self.graph = None
        self.out = None

    def stage(self, samples, sizes):
        """Enqueue the H2D copies of the raw sweeps and, when it differs from the previous replay's, of the table."""
        # the pinned staging buffers may still feed the previous copies: wait for those before rewriting them
        self.copied.synchronize()
        table = self.ingest.host_table(samples, sizes)
        if self.last_table is None or not np.array_equal(table, self.last_table):
            self.table_staging.numpy()[:] = table
            self.ingest.table.copy_(self.table_staging, non_blocking=True)
            self.last_table = table
        if self.raw_staging is None and not all(torch.is_tensor(r) and r.is_pinned() for s in samples for r in s[0]):
            self.raw_staging = torch.empty(self.ingest.raw.shape, dtype=torch.float32, pin_memory=True)
        stage_raw_sweeps(samples, sizes, self.ingest.raw, self.raw_staging)
        self.copied.record()


class _StreamGraphEntry:
    """One captured SweepStream forward: the stream whose buffers the graph holds, the graph and its packed output."""

    def __init__(self, stream):
        self.stream = stream
        self.graph = None
        self.out = None


class SweepStream:
    """B independent LiDAR streams whose sweep histories stay in device memory, feeding infer_sweeps' model.

    Each stream keeps its last K (<= 16) sweeps in slots of one device buffer [B, K, slot_capacity, raw_stride]: push()
    writes a new sweep into slot (pushes since reset) mod K of its stream with one H2D copy (pinned tensors directly,
    anything else through a pinned staging buffer), so a sweep is uploaded once however many frames it takes part in.
    In a frame the newest push of each stream is its key frame (neither filtered nor transformed) and its earlier sweeps
    follow newest first, each under inv(P_key) @ P_s (float64, on the host) with lag t_key - t_s rounded to float32 and
    the `radius` remove_close filter, exactly as infer_sweeps treats a sample.  infer() sends only the sweep table (a few
    KB: offsets, slot starts, transforms, lags, flags) and runs d3b_ingest_sweeps_gather over the slots; the detections
    are bit-identical to infer_sweeps(samples()).  A stream with fewer than K pushes uses the sweeps it has; reset(b)
    empties a stream (e.g. at a scene change).

    Not reproduced: the reference draws a sample's sweeps with np.random.choice (a random order, and the voxelizer's
    output depends on input order); here they are always newest first.  Nor is the reference's nuScenes pose chain: its
    info files carry a transform_matrix built from ego and calibration poses, which can differ from inv(P_key) @ P_s in
    the last bits.

    With graphed=True one CUDA graph keyed ("stream", B, K, slot_capacity, raw_stride, n_feat) in the pipeline's LRU
    covers ingest, voxelize and forward.  Its raw capacity is B * K * slot_capacity, so frames of any size replay it;
    the slot copies happen outside it.  A graph holds one stream's buffers: a second stream of the same shape on the same
    pipeline replaces the entry (and recaptures) when it infers."""

    def __init__(self, pipe, batch, history=10, slot_capacity=40000, raw_stride=5, n_feat=4, radius=1.0):
        if not 1 <= batch <= MAX_BATCH:
            raise ValueError("batch must be in [1, %d], got %d" % (MAX_BATCH, batch))
        if not 1 <= history <= MAX_SWEEPS:
            raise ValueError("history must be in [1, %d] sweeps (key frame included), got %d" % (MAX_SWEEPS, history))
        if slot_capacity < 1 or batch * history * slot_capacity > 1 << 30:
            raise ValueError("slot_capacity %d outside [1, 2^30 / (batch * history)]" % slot_capacity)
        if n_feat < 3 or raw_stride < n_feat:
            raise ValueError("bad layout: n_feat %d, raw_stride %d" % (n_feat, raw_stride))
        if n_feat + 1 != pipe.num_point_features:
            raise ValueError("ingested clouds have n_feat + 1 = %d features, the reader takes %d"
                             % (n_feat + 1, pipe.num_point_features))
        self.pipe, self.batch, self.history, self.slot_capacity = pipe, batch, history, slot_capacity
        self.raw_stride, self.n_feat, self.radius = raw_stride, n_feat, radius
        self.key = ("stream", batch, history, slot_capacity, raw_stride, n_feat)
        self.sweeps = SweepHistory(batch, history)
        self.pending_h2d_bytes = 0                # pushed since the last infer()
        self.last_h2d_bytes = 0                   # of the last infer(): the pushes before it + its table
        self._ingest = None                       # device buffers, allocated on the first push
        self._push_staging = None                 # pinned [B, slot_capacity, raw_stride], allocated on first need
        self._push_copied = None

    def _buffers(self):
        """The gather BatchedIngest whose raw buffer holds the slots, and the slots' [B, K, slot_capacity, raw_stride]
        view of it (allocated on first use)."""
        if self._ingest is None:
            B, K = self.batch, self.history
            self._ingest = BatchedIngest(B, B * K * self.slot_capacity, B * K, self.raw_stride, self.n_feat, self.radius,
                                         self.pipe.device, gather=True)
            self._slots = self._ingest.raw.view(B, K, self.slot_capacity, self.raw_stride)
            self._table_staging = torch.zeros(self._ingest.table.numel(), dtype=torch.uint8, pin_memory=True)
            self._table_copied = torch.cuda.Event()
        return self._ingest, self._slots

    def check_push(self, b, raw, pose, timestamp):
        """Host-side validation of push()'s arguments: raises ValueError.  Returns the number of raw points."""
        self.sweeps.check_stream(b)
        if torch.is_tensor(raw):
            ok = raw.dtype == torch.float32 and raw.device.type == "cpu"
        else:
            ok = isinstance(raw, np.ndarray) and raw.dtype == np.float32
        if not ok or raw.ndim != 2:
            raise ValueError("stream %d: raw points must be a 2-D float32 host array" % b)
        if int(raw.shape[1]) != self.raw_stride:
            raise ValueError("stream %d: raw stride %d, the stream has %d" % (b, raw.shape[1], self.raw_stride))
        if int(raw.shape[0]) > self.slot_capacity:
            raise ValueError("stream %d: %d raw points exceed the slot capacity %d" % (b, raw.shape[0], self.slot_capacity))
        if np.shape(pose) != (4, 4):
            raise ValueError("stream %d: pose must be a 4x4 matrix, got shape %s" % (b, np.shape(pose)))
        if not isinstance(timestamp, numbers.Real):
            raise ValueError("stream %d: timestamp must be a number, got %r" % (b, timestamp))
        return int(raw.shape[0])

    def push(self, b, raw, pose, timestamp):
        """Stream b's new sweep, which becomes its key frame: raw float32 [n, raw_stride] host array or tensor (pinned
        tensors are copied directly and must stay unchanged until the copy has run), pose the sensor-to-world 4x4
        matrix, timestamp in seconds.  Enqueues one H2D copy into the stream's oldest slot; ValueError before anything
        is enqueued when an argument is malformed."""
        rows = self.check_push(b, raw, pose, timestamp)
        _ing, slots = self._buffers()
        slot = self.sweeps.next_slot(b)
        if rows:
            with torch.cuda.device(slots.device):
                src = raw if torch.is_tensor(raw) and raw.is_pinned() else None
                if src is None:
                    if self._push_staging is None:
                        self._push_staging = torch.empty((self.batch, self.slot_capacity, self.raw_stride),
                                                         dtype=torch.float32, pin_memory=True)
                        self._push_copied = [torch.cuda.Event() for _ in range(self.batch)]
                    self._push_copied[b].synchronize()          # stream b's staging may still feed its previous copy
                    src = self._push_staging[b, :rows]
                    src.copy_(torch.as_tensor(raw))
                    slots[b, slot, :rows].copy_(src, non_blocking=True)
                    self._push_copied[b].record()
                else:
                    slots[b, slot, :rows].copy_(src, non_blocking=True)
        self.sweeps.record(b, rows, pose, timestamp)
        self.pending_h2d_bytes += rows * self.raw_stride * 4

    def reset(self, b):
        """Forget stream b's history: its next push is a key frame with no earlier sweeps."""
        self.sweeps.reset(b)

    def samples(self):
        """The current frame as infer_sweeps' samples [(raw_sweeps, transforms, time_lags), ...], the raw sweeps read
        back from the device slots: a test oracle and debugging aid (it synchronizes)."""
        frame = self.sweeps.frame()
        _ing, slots = self._buffers()
        return [([slots[b, k, :n].cpu().numpy() for k, n in zip(ks, ns)], tms, lags)
                for b, (ks, ns, tms, lags) in enumerate(frame)]

    def _stage_table(self):
        """Writes the current frame's sweep table into the pinned staging buffer and enqueues its H2D copy."""
        frame = self.sweeps.frame()
        ing, _slots = self._buffers()
        K, cap = self.history, self.slot_capacity
        src = [(b * K + k) * cap for b, (ks, _ns, _tms, _lags) in enumerate(frame) for k in ks]
        self._table_copied.synchronize()          # the staging buffer may still feed the previous frame's copy
        ing.host_table([(None, tms, lags) for _ks, _ns, tms, lags in frame], [ns for _ks, ns, _tms, _lags in frame],
                       out=self._table_staging.numpy(), sweep_src=src)
        with torch.cuda.device(ing.table.device):
            ing.table.copy_(self._table_staging, non_blocking=True)
            self._table_copied.record()
        self.last_h2d_bytes = self.pending_h2d_bytes + ing.table.numel()
        self.pending_h2d_bytes = 0

    def _graph_entry(self):
        graphs = self.pipe._graphs
        entry = graphs.get(self.key)
        if entry is not None and entry.stream is self:
            graphs.move_to_end(self.key)
            return entry
        graphs.pop(self.key, None)
        while len(graphs) >= self.pipe.max_graphs:
            graphs.popitem(last=False)
        entry = graphs[self.key] = _StreamGraphEntry(self)
        return entry

    @torch.no_grad()
    def infer(self, pinned_out=None, graphed=False):
        """Detections of the current frame, host [B, D, nd+3] as infer_sweeps returns them, and bit-identical to
        infer_sweeps(samples()).  The only H2D is the sweep table (the sweeps went with push).  graphed=True replays the
        stream's CUDA graph.  On an f16-range overflow the model switches to tf32x3 and the same frame is re-run, as in
        infer_sweeps; the history is not touched.  ValueError when a stream holds no sweep."""
        self._stage_table()
        pipe, ing = self.pipe, self._ingest
        step = lambda: pipe.pack(pipe.forward_device(*ing.launch()))      # noqa: E731
        for _attempt in range(2):
            if graphed:         # (a re-run after an overflow captures a new graph: check_overflow dropped them all)
                packed = pipe._run_graph(self._graph_entry(), step)
            else:
                packed = step()
            pinned_out, rerun = pipe._fetch(packed, pinned_out)
            if not rerun:
                break
        return pinned_out
