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
from det3d_b200.core.bbox.box_np_ops import camera_frustum_planes
from det3d_b200.datasets.pipelines.loading import (MAX_BATCH, MAX_SWEEPS, BatchedIngest, RowStager, SweepHistory,
                                                    check_sweep_samples, sweep_table_capacity)
from det3d_b200.models import build_detector
from det3d_b200.ops.point_cloud.frustum import MAX_NDIM, MIN_NDIM, FrustumCrop
from det3d_b200.ops.point_cloud.kitti_results import KittiResults, calib_table, check_calibs, to_annos
from det3d_b200.ops.point_cloud.nusc_results import (ND as NUSC_ND, NuscResults, attribute_table, check_tokens,
                                                     pose_table, to_nusc_annos)
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
        # _GraphEntry by key, least recently used first: (batch, bucket, ndim) (forward_graphed, infer_host), (batch,
        # raw bucket, table capacity, raw_stride, n_feat) (infer_sweeps), ("stream", B, K, slot_capacity, raw_stride,
        # n_feat) (SweepStream.infer), ("frustum", B, raw bucket, ndim) / ("frustum_kitti", B, raw bucket, ndim)
        # (infer_raw without / with kitti_results); ("sweeps_nusc",) + infer_sweeps' key and the stream's key + ("nusc",)
        # (nusc_results=True)
        self._graphs = collections.OrderedDict()
        self.max_graphs = 8
        self._ovf_host = None
        self._planes = collections.OrderedDict()      # calibration bytes -> frustum planes f64 [6, 4] (infer_raw)
        self._kitti_tables = collections.OrderedDict()   # calibration bytes -> KITTI results table f64 [32]
        self._nusc_tables = collections.OrderedDict()    # pose record bytes -> nuScenes pose table f64 [32]

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

    # ---- the graph cache and the run-and-fetch loop every entry point goes through -----------------------------------
    def _cached(self, key, make, fits=None):
        """The graph-cache entry at `key`, marked most recently used.  A missing entry, or one `fits` rejects, is
        replaced by make(), after evicting least recently used entries until there is room under max_graphs."""
        entry = self._graphs.get(key)
        if entry is not None and (fits is None or fits(entry)):
            self._graphs.move_to_end(key)
            return entry
        self._graphs.pop(key, None)
        while len(self._graphs) >= self.max_graphs:
            self._graphs.popitem(last=False)
        entry = self._graphs[key] = make()
        return entry

    def _serve(self, graphed, key, make, step, fetch, stage=None, fits=None):
        """Runs one entry point: takes its entry (graphed: _cached(key, make, fits); eager: a transient make()), stages
        the inputs into it (stage(entry)), runs step(entry) -- eagerly, or captured into and replayed from entry.graph
        -- enqueues the D2H copies of fetch(entry, step's outputs), and syncs once.  When the f16-range flag was raised,
        the model has switched to tf32x3 and check_overflow has dropped the graphs, so everything runs once more from
        a fresh lookup.  Returns fetch's host result."""
        for _attempt in range(2):
            entry = self._cached(key, make, fits) if graphed else make()
            if stage is not None:
                stage(entry)
            out = self._run_graph(entry, lambda: step(entry)) if graphed else step(entry)
            host = fetch(entry, out)
            if not self._sync_overflow():
                break
        return host

    @staticmethod
    def _packed_into(pinned_out):
        """_serve's fetch of the packed detections: their D2H copy into pinned_out (allocated pinned when None)."""
        def fetch(_entry, packed):
            nonlocal pinned_out
            if pinned_out is None:
                pinned_out = torch.empty(packed.shape, dtype=torch.float32, pin_memory=True)
            return pinned_out.copy_(packed, non_blocking=True)
        return fetch

    def _sync_overflow(self):
        """D2H of the f16-range flag behind the copies already enqueued, then one sync.  Returns True when the flag was
        raised and the model has switched to tf32x3 (check_overflow)."""
        flag = self.overflow_flag()
        if flag is not None:
            if self._ovf_host is None:
                self._ovf_host = torch.zeros(1, dtype=torch.int32, pin_memory=True)
            self._ovf_host.copy_(flag, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return flag is not None and self.check_overflow(int(self._ovf_host[0]))

    def _points_entry(self, batch, bucket, ndim):
        """forward_graphed's entry (batch, bucket, ndim): static points [bucket, ndim] and device offsets [batch + 1]."""
        return _GraphEntry(points=torch.zeros((bucket, ndim), dtype=torch.float32, device=self.device), rows=RowStager(),
                           offsets=_Upload(torch.zeros(batch + 1, dtype=torch.int32, device=self.device)))

    def _graph_entry(self, batch, n_points, ndim):
        """The graph-cache entry of (batch, bucket_of(n_points), ndim); a new entry has buffers but no graph yet."""
        key = (batch, self.bucket_of(n_points), ndim)
        return self._cached(key, lambda: self._points_entry(*key))

    def _replay(self, entry, offsets):
        """Make the graph's device offsets `offsets`, capture the graph on first use, replay.  The clouds must already
        be in entry.points[:offsets[-1]]."""
        entry.offsets.put(offsets)
        return self._run_graph(entry, lambda: self.pack(self.forward_device(entry.points, entry.offsets.dev)))

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
        batch, ndim = len(clouds), clouds[0].shape[1]
        if graphed:
            self.check_offsets(offsets)
            key = (batch, self.bucket_of(offsets[-1]), ndim)
            make = lambda: self._points_entry(*key)                                                       # noqa: E731
            step = lambda e: self.pack(self.forward_device(e.points, e.offsets.dev))                      # noqa: E731
        else:           # an exactly sized buffer and host offsets
            key = None
            make = lambda: _GraphEntry(points=torch.empty((offsets[-1], ndim), dtype=torch.float32,      # noqa: E731
                                                          device=self.device), rows=RowStager())
            step = lambda e: self.pack(self.forward_device(e.points, offsets))                            # noqa: E731

        def stage(e):
            e.rows.put(clouds, e.points)
            if graphed:
                e.offsets.put(offsets)
        return self._serve(graphed, key, make, step, self._packed_into(pinned_out), stage)

    @torch.no_grad()
    def infer_sweeps(self, samples, pinned_out=None, graphed=False, n_feat=4, radius=1.0, nusc_results=False, poses=None,
                     tokens=None):
        """Multi-sweep samples -> host detections [B, D, nd+3], as infer_host.

        samples: [(raw_sweeps, transforms, time_lags), ...], one per cloud, each with ingest_sweeps' contract (raw
        float32 [n, raw_stride] host arrays or pinned tensors, key frame first and neither filtered nor transformed
        unless given a transform; 4x4 or None transforms; one time lag per sweep).  One batched ingest
        (d3b_ingest_sweeps_dev) writes the clouds and their device offsets, which the voxelizer reads directly: no host
        sync before the D2H of the detections.  graphed=True replays one CUDA graph covering ingest, voxelize and
        forward per (B, raw bucket, sweep-table capacity, raw_stride, n_feat) (bucket_of of the raw total); the raw
        sweeps are copied into its static raw buffer and the sweep table is copied H2D only when it changed.  Raises
        ValueError before anything is enqueued when the samples are malformed or n_feat + 1 is not the reader's
        feature count.  The overflow fallback is infer_host's.

        nusc_results=True returns instead what the reference reports for nuScenes (NuScenesDataset.evaluation,
        det3d/datasets/nuscenes/nuscenes.py:180-274): the nusc_annos dict, results keyed by tokens[b] in sample order,
        each detection in predict's order as a submission box in the global frame -- translation, size, orientation
        quaternion, velocity, class name (self.class_names()), score and attribute -- and the reference's meta.
        poses[b] holds sample b's key-frame records dict(calibrated_sensor=dict(translation, rotation),
        ego_pose=dict(translation, rotation)) and tokens[b] its sample token.  d3b_nusc_results_dev runs right after
        predict, inside the same graph when graphed (keyed ("sweeps_nusc",) + the plain key); the pose table
        (nusc_pose_table, cached per record) goes H2D only when it differs from that graph's last replay, and the rows,
        their counts and the f16-range flag come back before one sync.  ValueError before anything is enqueued when
        poses or tokens are missing or not one per sample, a token is not a str or repeats, a record is malformed, a
        class has no nuScenes attribute, or the model's boxes have no velocity (nd != 9)."""
        if n_feat + 1 != self.num_point_features:
            raise ValueError("ingested clouds have n_feat + 1 = %d features, the reader takes %d"
                             % (n_feat + 1, self.num_point_features))
        samples = list(samples)
        stride, sizes = check_sweep_samples(samples, n_feat)
        batch, total = len(samples), sum(map(sum, sizes))
        key = (batch, self.bucket_of(total), sweep_table_capacity(sum(map(len, sizes)), batch), stride, n_feat)
        nusc = _NuscStep(self, batch, poses, tokens) if nusc_results else None

        def make():
            # eager too, the voxelizer's capacity is the bucket: it keeps its device-offset buffers per capacity
            ingest = BatchedIngest(*key, radius, self.device)
            entry = _GraphEntry(ingest=ingest, table=_Upload(ingest.table), rows=RowStager())
            return entry if nusc is None else nusc.attach(entry)

        def stage(e):
            e.table.put(e.ingest.host_table(samples, sizes))
            e.rows.put([r for raws, _tms, _lags in samples for r in raws], e.ingest.raw)
            if nusc is not None:
                nusc.stage(e)

        def step(e):
            packed = self.pack(self.forward_device(*e.ingest.launch()))
            return packed if nusc is None else e.nusc.launch(packed)
        if nusc is None:
            return self._serve(graphed, key, make, step, self._packed_into(pinned_out), stage,
                               fits=lambda e: e.ingest.radius == radius)
        return nusc.annos(self._serve(graphed, ("sweeps_nusc",) + key, make, step, _NuscStep.fetch, stage,
                                      fits=lambda e: e.ingest.radius == radius))

    # ---- raw KITTI scans: camera-frustum crop on the device ----------------------------------------------------------
    @staticmethod
    def check_raw_clouds(clouds, calibs):
        """Host-side validation of infer_raw's arguments: raises ValueError, before anything is enqueued.  Returns
        (ndim, cloud sizes)."""
        clouds, calibs = list(clouds), list(calibs)
        if not 1 <= len(clouds) <= MAX_BATCH:
            raise ValueError("a batch holds 1 to %d clouds, got %d" % (MAX_BATCH, len(clouds)))
        if len(calibs) != len(clouds):
            raise ValueError("%d clouds but %d calibrations" % (len(clouds), len(calibs)))
        ndim, sizes = None, []
        for b, c in enumerate(clouds):
            if torch.is_tensor(c):
                ok = c.dtype == torch.float32 and c.device.type == "cpu"
            else:
                ok = isinstance(c, np.ndarray) and c.dtype == np.float32
            if not ok or c.ndim != 2:
                raise ValueError("cloud %d: raw points must be a 2-D float32 host array" % b)
            ndim = int(c.shape[1]) if ndim is None else ndim
            if int(c.shape[1]) != ndim:
                raise ValueError("cloud %d: %d columns, the batch has %d" % (b, c.shape[1], ndim))
            sizes.append(int(c.shape[0]))
        if not MIN_NDIM <= ndim <= MAX_NDIM:
            raise ValueError("raw clouds must have %d to %d columns, got %d" % (MIN_NDIM, MAX_NDIM, ndim))
        if sum(sizes) > 1 << 30:
            raise ValueError("more than 2^30 raw points in one batch")
        check_calibs(calibs)
        return ndim, sizes

    @staticmethod
    def _cached_per_calib(cache, calib, compute):
        """compute(calib, (H, W)) cached by the calibration's bytes (KITTI calibrations change per drive, not per
        frame), the 256 most recently used kept."""
        # keyed on each matrix's dtype, shape and bytes: the tables are computed from the arrays as given, and numpy's
        # inv / qr give a float32 calibration other planes than the same values in float64
        parts = [np.ascontiguousarray(calib[k]) for k in ("rect", "Trv2c", "P2")]
        shape = tuple(int(v) for v in np.asarray(calib["image_shape"]).reshape(-1)[:2])
        key = b"".join(p.tobytes() for p in parts) + repr((shape, [(p.dtype.str, p.shape) for p in parts])).encode()
        value = cache.get(key)
        if value is None:
            value = cache[key] = compute(calib, shape)
            while len(cache) > 256:
                cache.popitem(last=False)
        else:
            cache.move_to_end(key)
        return value

    def frustum_planes(self, calib):
        """camera_frustum_planes of one calibration, cached by the calibration's bytes."""
        return self._cached_per_calib(self._planes, calib, lambda c, shape: camera_frustum_planes(
            c["rect"], c["Trv2c"], c["P2"], shape))

    def kitti_calib_table(self, calib):
        """The KITTI results kernel's calibration row f64 [32] (ops.point_cloud.kitti_results.calib_table: rect @ Trv2c
        by numpy's matmul, P2, the image shape), cached by the calibration's bytes."""
        return self._cached_per_calib(self._kitti_tables, calib,
                                      lambda c, shape: calib_table(dict(c, image_shape=shape)))

    def nusc_pose_table(self, record):
        """The nuScenes results kernel's pose row f64 [32] of one sample's records (ops.point_cloud.nusc_results.
        pose_table), cached by the records' bytes (the sensor calibration is fixed per scene and the ego pose changes per
        sample), the 256 most recently used kept.  ValueError for a malformed record."""
        try:
            parts = [np.ascontiguousarray(record[k][f], np.float64) for k in ("calibrated_sensor", "ego_pose")
                     for f in ("translation", "rotation")]
        except (KeyError, TypeError, ValueError):
            return pose_table(record)                   # raises the record's ValueError
        key = b"".join(p.tobytes() for p in parts) + repr([p.shape for p in parts]).encode()
        value = self._nusc_tables.get(key)
        if value is None:
            value = self._nusc_tables[key] = pose_table(record)
            while len(self._nusc_tables) > 256:
                self._nusc_tables.popitem(last=False)
        else:
            self._nusc_tables.move_to_end(key)
        return value

    def class_names(self):
        """The config's class names flattened over its tasks, the order predict's labels index."""
        return [n for t in self.cfg.tasks for n in t["class_names"]]

    @torch.no_grad()
    def infer_raw(self, clouds, calibs, pinned_out=None, graphed=False, kitti_results=False):
        """Raw KITTI scans -> host detections [B, D, nd+3], as infer_host: each scan is first cropped to its camera's
        view frustum (box_np_ops.remove_outside_points, bit-exact), on the device.

        clouds: float32 [N_i, ndim] host arrays or tensors (pinned tensors are copied to the device directly), the full
        360° scans; calibs[i]: dict(rect, Trv2c, P2, image_shape) -- res["calib"] plus the image shape (H, W).  One
        d3b_frustum_crop_dev call crops the batch and writes the cropped clouds' device offsets, which the voxelizer
        reads directly: no host sync before the D2H of the detections, which are the bits infer_host gives on the
        cropped clouds.  graphed=True replays one CUDA graph covering crop, voxelize and forward per ("frustum", B,
        raw bucket, ndim) (bucket_of of the raw total), in the LRU of forward_graphed; the scans are copied into its
        static raw buffer, and the offsets and the plane table H2D only when they differ from that graph's last
        replay.  The voxelizer's capacity is the raw bucket (the crop only removes points).  Raises ValueError before
        anything is enqueued when the arguments are malformed.  The overflow fallback is infer_host's.

        kitti_results=True returns instead what the reference reports for KITTI
        (KittiDataset.convert_detection_to_kitti_annos, det3d/datasets/kitti/kitti.py:78-158): one anno dict per scan
        with the reference's keys and dtypes, holding the detections whose image box meets the image, in predict's
        order -- their clipped image box, alpha, camera-frame dimensions, location and rotation_y, score and class
        name (self.class_names()).  d3b_kitti_results_dev runs right after predict, inside the same graph when
        graphed (keyed ("frustum_kitti", B, raw bucket, ndim), apart from the plain one); each scan's calibration table
        (kitti_calib_table, cached per calibration) goes H2D only when it differs from that graph's last replay, and
        the kept rows, their counts and the f16-range flag come back in one D2H before one sync."""
        clouds, calibs = list(clouds), list(calibs)
        ndim, sizes = self.check_raw_clouds(clouds, calibs)
        planes = np.stack([self.frustum_planes(c) for c in calibs])
        tables = np.stack([self.kitti_calib_table(c) for c in calibs]) if kitti_results else None
        offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
        batch, bucket = len(clouds), self.bucket_of(int(offsets[-1]))

        def make():
            crop = FrustumCrop(batch, bucket, ndim, self.device)
            kitti = KittiResults(batch, self.device) if kitti_results else None
            return _GraphEntry(crop=crop, offsets=_Upload(crop.offsets), planes=_Upload(crop.planes), rows=RowStager(),
                               kitti=kitti, calib=None if kitti is None else _Upload(kitti.calib),
                               planes_uploads=0, calib_uploads=0)          # H2D copies of each table so far

        def stage(e):
            e.rows.put(clouds, e.crop.points)
            e.offsets.put(offsets)
            e.planes_uploads += e.planes.put(planes)
            if e.kitti is not None:
                e.calib_uploads += e.calib.put(tables)

        def step(e):
            packed = self.pack(self.forward_device(*e.crop.launch()))
            return packed if e.kitti is None else e.kitti.launch(packed)

        def fetch(e, out):
            if e.kitti is None:
                return packed_into(e, out)
            e.kitti.results_host.copy_(out[0], non_blocking=True)
            e.kitti.counts_host.copy_(out[1], non_blocking=True)
            return e.kitti
        packed_into = self._packed_into(pinned_out)
        key = ("frustum_kitti" if kitti_results else "frustum", batch, bucket, ndim)
        got = self._serve(graphed, key, make, step, fetch, stage)
        if kitti_results:
            return to_annos(got.results_host.numpy(), got.counts_host.numpy(), self.class_names())
        return got

    @staticmethod
    def unpack(packed_host):
        """host [B, D, nd+3] -> list of dict(box3d_lidar, scores, label_preds) per sample."""
        out = []
        for row in packed_host:
            m = row[:, -1] > 0.5
            out.append(dict(box3d_lidar=row[m, :-3], scores=row[m, -3], label_preds=row[m, -2].long()))
        return out


class _NuscStep:
    """infer_sweeps' and SweepStream.infer's nuScenes results post-step.  The constructor checks the arguments and
    builds the pose tables (ValueError before anything is enqueued); attach adds a NuscResults and its pose _Upload to a
    new entry, stage uploads the poses when they changed, fetch enqueues the D2H of the rows, annos formats them."""

    def __init__(self, pipe, batch, poses, tokens):
        if poses is None or tokens is None:
            raise ValueError("nusc_results needs poses and tokens, one per sample")
        poses = list(poses)
        if len(poses) != batch:
            raise ValueError("%d samples but %d pose records" % (batch, len(poses)))
        self.tokens = check_tokens(tokens, batch)
        nd = pipe.model.bbox_head.box_coder.n_dim            # the decoded box (code_size adds the sin / cos pair)
        if nd != NUSC_ND:
            raise ValueError("nuScenes results need boxes with velocity (nd = %d), the model's have nd = %d"
                             % (NUSC_ND, nd))
        self.class_names = pipe.class_names()
        self.table = attribute_table(self.class_names)
        self.poses = np.stack([pipe.nusc_pose_table(p) for p in poses])
        self.batch, self.device = batch, pipe.device

    def attach(self, entry):
        entry.nusc = NuscResults(self.batch, self.device)
        entry.poses = _Upload(entry.nusc.poses)
        entry.pose_uploads = 0                        # H2D copies of the pose table so far
        return entry

    def stage(self, entry):
        entry.pose_uploads += entry.poses.put(self.poses)

    @staticmethod
    def fetch(entry, _out):
        return entry.nusc.fetch()

    def annos(self, nusc):
        return to_nusc_annos(nusc.results_host.numpy(), nusc.counts_host.numpy(), self.class_names, self.tokens,
                             self.table)


class _GraphEntry:
    """One entry point's state: the static buffers it attaches (points, a BatchedIngest, a FrustumCrop, a KittiResults,
    their _Uploads and RowStager) and, once captured, the graph and its output.  A graphed entry lives in the graph
    cache; an eager one serves one call."""

    def __init__(self, **buffers):
        self.graph = self.out = None
        self.__dict__.update(buffers)


class _Upload:
    """A small device table `dev` that goes H2D only when its bytes change, through a pinned staging copy."""

    def __init__(self, dev):
        self.dev = dev
        self.staging = torch.empty(dev.shape, dtype=dev.dtype, pin_memory=True)
        self.copied = torch.cuda.Event()
        self.last = None

    def put(self, value, always=False):
        """Enqueues the H2D copy of the host `value` (dev's shape, converted to its dtype) unless its bytes equal the
        last put's; always=True copies in any case.  Returns whether it copied."""
        host = self.staging.numpy()
        value = np.asarray(value, host.dtype)
        raw = value.tobytes()
        if raw == self.last and not always:
            return False
        self.copied.synchronize()                 # the staging buffer may still feed the previous copy
        host[...] = value
        with torch.cuda.device(self.dev.device):
            self.dev.copy_(self.staging, non_blocking=True)
            self.copied.record()
        self.last = raw
        return True


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

    def _buffers(self):
        """The gather BatchedIngest whose raw buffer holds the slots, and the slots' [B, K, slot_capacity, raw_stride]
        view of it (allocated on first use)."""
        if self._ingest is None:
            B, K = self.batch, self.history
            self._ingest = BatchedIngest(B, B * K * self.slot_capacity, B * K, self.raw_stride, self.n_feat, self.radius,
                                         self.pipe.device, gather=True)
            self._slots = self._ingest.raw.view(B, K, self.slot_capacity, self.raw_stride)
            self._table = _Upload(self._ingest.table)
            self._rows = [RowStager() for _ in range(B)]            # one staging buffer [slot_capacity] per stream
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
        self._rows[b].put([raw], slots[b, self.sweeps.next_slot(b)])
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
        """Enqueues the H2D copy of the current frame's sweep table (every frame: it changes with each push)."""
        frame = self.sweeps.frame()
        ing, _slots = self._buffers()
        K, cap = self.history, self.slot_capacity
        src = [(b * K + k) * cap for b, (ks, _ns, _tms, _lags) in enumerate(frame) for k in ks]
        self._table.put(ing.host_table([(None, tms, lags) for _ks, _ns, tms, lags in frame],
                                       [ns for _ks, ns, _tms, _lags in frame], sweep_src=src), always=True)
        self.last_h2d_bytes = self.pending_h2d_bytes + ing.table.numel()
        self.pending_h2d_bytes = 0

    @torch.no_grad()
    def infer(self, pinned_out=None, graphed=False, nusc_results=False, poses=None, tokens=None):
        """Detections of the current frame, host [B, D, nd+3] as infer_sweeps returns them, and bit-identical to
        infer_sweeps(samples()).  The only H2D is the sweep table (the sweeps went with push).  graphed=True replays the
        stream's CUDA graph.  On an f16-range overflow the model switches to tf32x3 and the same frame is re-run, as in
        infer_sweeps; the history is not touched.  ValueError when a stream holds no sweep.

        nusc_results=True (with poses and tokens, one per stream) returns the frame's nusc_annos as
        infer_sweeps(samples(), nusc_results=True) does, from the stream's graph keyed key + ("nusc",); the pose table
        goes H2D only when it changed."""
        pipe = self.pipe
        nusc = _NuscStep(pipe, self.batch, poses, tokens) if nusc_results else None
        self._stage_table()

        def step(e):
            packed = pipe.pack(pipe.forward_device(*self._ingest.launch()))
            return packed if nusc is None else e.nusc.launch(packed)
        if nusc is None:
            return pipe._serve(graphed, self.key, lambda: _GraphEntry(stream=self), step, pipe._packed_into(pinned_out),
                               fits=lambda e: e.stream is self)
        return nusc.annos(pipe._serve(graphed, self.key + ("nusc",), lambda: nusc.attach(_GraphEntry(stream=self)),
                                      step, _NuscStep.fetch, nusc.stage, fits=lambda e: e.stream is self))
