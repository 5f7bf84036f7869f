"""KITTI camera-frustum crop on the device (d3b_frustum_crop_dev, csrc/frustum.cu) and raw scans -> detections
(InferencePipeline.infer_raw, Preprocess(remove_outside_points=True)).

The rows the device keeps are compared bit for bit with points[mask], the mask being the reference's own
(tests/golden/frustum_kitti_*.npz) or, for inputs the goldens do not hold, oracle/frustum.keep_mask, which is pinned to
the goldens on the CPU (tests/test_frustum.py).  End to end, infer_raw must give the packed detections infer_host gives
on the cropped clouds, bit for bit."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

pytestmark = pytest.mark.gpu

CASES = ("scans", "adversarial")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _calib(g, b):
    return dict(rect=g["rect"][b], Trv2c=g["Trv2c"][b], P2=g["P2"][b], image_shape=g["image_shape"][b])


def _crop(clouds, planes, capacity=None, poison=np.nan, offsets=None):
    """One d3b_frustum_crop_dev call over host clouds; rows past the live total are filled with `poison`.  Returns
    (host rows per cloud, device cloud_offsets, status, FrustumCrop)."""
    from det3d_b200.ops.point_cloud.frustum import FrustumCrop
    ndim = clouds[0].shape[1]
    live = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
    capacity = int(live[-1]) if capacity is None else capacity
    crop = FrustumCrop(len(clouds), capacity, ndim)
    crop.points.fill_(poison)
    crop.out.fill_(np.nan)
    if live[-1]:
        crop.points[:live[-1]].copy_(torch.from_numpy(np.concatenate(clouds)))
    crop.set_table(live if offsets is None else offsets, planes)
    out, cloud_offsets = crop.launch()
    off = cloud_offsets.cpu().numpy()
    host = out.cpu().numpy()
    rows = [host[off[b]:off[b + 1]] for b in range(len(clouds))]
    return rows, off, int(crop.status.item()), crop


def _golden_clouds(g):
    off = g["offsets"]
    return ([g["points"][off[b]:off[b + 1]] for b in range(off.shape[0] - 1)],
            [g["mask"][off[b]:off[b + 1]] for b in range(off.shape[0] - 1)])


# ---- the kernel ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES + ("rounding",))
def test_rows_equal_the_reference_rows_bit_for_bit(case):
    """Scans, adversarial points and the rounding golden, whose points an FMA-contracted or reordered plane test decides
    differently from the reference (tests/test_frustum.py)."""
    g = load_golden("frustum_kitti_" + case)
    clouds, masks = _golden_clouds(g)
    rows, off, status, _ = _crop(clouds, g["planes"])                  # the whole golden as one batch
    assert status == 0
    for b, (c, m) in enumerate(zip(clouds, masks)):
        assert np.array_equal(_bits(rows[b]), _bits(c[m])), b
        alone, _, _, _ = _crop([c], g["planes"][b:b + 1])
        assert np.array_equal(_bits(alone[0]), _bits(c[m])), b
    assert np.array_equal(off, np.concatenate([[0], np.cumsum([m.sum() for m in masks])]))


@pytest.mark.parametrize("case", CASES)
def test_remove_outside_points_equals_the_reference(case):
    from det3d_b200.core.bbox.box_np_ops import remove_outside_points
    g = load_golden("frustum_kitti_" + case)
    clouds, masks = _golden_clouds(g)
    for b, (c, m) in enumerate(zip(clouds, masks)):
        cal = _calib(g, b)
        got = remove_outside_points(c, cal["rect"], cal["Trv2c"], cal["P2"], cal["image_shape"])
        assert got.dtype == np.float32 and got.shape == (int(m.sum()), c.shape[1])
        assert np.array_equal(_bits(got), _bits(c[m])), b


def _mixed(batch, seed, ndim=4):
    """batch clouds: golden scans and adversarial points (possibly with extra columns), an empty cloud, one entirely
    behind the camera and one entirely inside; their planes [B, 6, 4]."""
    from oracle.frustum import keep_mask
    rng = np.random.default_rng(seed)
    gs = [load_golden("frustum_kitti_" + c) for c in CASES]
    pools = [(_golden_clouds(g)[0], g["planes"]) for g in gs]
    clouds, planes = [], []
    for b in range(batch):
        src, pl = pools[b % 2]
        k = int(rng.integers(len(src)))
        c = src[k]
        kind = b % 7
        if kind == 2:
            c = c[:0]
        elif kind == 3:
            c = c[keep_mask(c, pl[k]) == 0]
            c = c[np.isfinite(c[:, :3]).all(1) & (c[:, 0] < -1)]          # behind the camera
        elif kind == 4:
            c = c[keep_mask(c, pl[k])]
        else:
            c = c[rng.permutation(c.shape[0])[:int(rng.integers(1, c.shape[0] + 1))]]
        if ndim != 4:
            wide = rng.standard_normal((c.shape[0], ndim)).astype(np.float32)
            wide[:, :min(4, ndim)] = c[:, :min(4, ndim)]
            c = wide
        clouds.append(np.ascontiguousarray(c))
        planes.append(pl[k])
    return clouds, np.stack(planes)


@pytest.mark.parametrize("batch,ndim", [(1, 4), (2, 3), (5, 4), (8, 5), (16, 16), (64, 4)])
def test_batches_with_empty_all_outside_and_all_inside_clouds(batch, ndim):
    """Every cloud's rows == its oracle rows in input order; cloud_offsets == the prefix of the kept counts; a
    capacity above the live total whose NaN-poisoned rows must never be read; two runs bit-identical."""
    from oracle.frustum import keep_mask
    clouds, planes = _mixed(batch, 100 + batch, ndim)
    total = sum(c.shape[0] for c in clouds)
    rows, off, status, _ = _crop(clouds, planes, capacity=total + 3000)
    again, off2, _, _ = _crop(clouds, planes, capacity=total + 3000)
    assert status == 0 and np.array_equal(off, off2)
    kept = [int(keep_mask(c, p).sum()) for c, p in zip(clouds, planes)]
    assert np.array_equal(off, np.concatenate([[0], np.cumsum(kept)]))
    for b, (c, p) in enumerate(zip(clouds, planes)):
        want = c[keep_mask(c, p)]
        assert rows[b].shape == want.shape and np.array_equal(_bits(rows[b]), _bits(want)), b
        assert np.array_equal(_bits(again[b]), _bits(rows[b])), b
    if batch >= 5:
        assert kept[2] == 0 and kept[3] == 0 and kept[4] == clouds[4].shape[0] > 0


def _clamped(raw, cap):
    """The kernel's clamp: off[0] = 0, off[i] = min(max(0, raw[1..i]), cap)."""
    out = np.zeros_like(raw)
    run = 0
    for i in range(1, raw.shape[0]):
        run = max(run, int(raw[i]))
        out[i] = min(run, cap)
    return out


@pytest.mark.parametrize("case", ["decreasing", "past capacity", "negative", "nonzero first"])
def test_malformed_device_offsets_are_clamped_and_reported(case):
    from oracle.frustum import keep_mask
    clouds, planes = _mixed(4, 7)
    cap = sum(c.shape[0] for c in clouds)
    pts = np.concatenate(clouds)
    live = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
    raw = live.copy()
    if case == "decreasing":
        raw[2] = raw[1] - 5
    elif case == "past capacity":
        raw[3:] = cap + 1000
    elif case == "negative":
        raw[1] = -7
    else:
        raw[0] = 5
    rows, off, status, _ = _crop(clouds, planes, capacity=cap, offsets=raw)
    assert status == 1
    good = _clamped(raw, cap)
    for b in range(4):
        seg = pts[good[b]:good[b + 1]]
        want = seg[keep_mask(seg, planes[b])]
        assert np.array_equal(_bits(rows[b]), _bits(want)), (case, b)


# ---- end to end ---------------------------------------------------------------------------------------------------
E2E = {"second_kitti_car": ("second_kitti_car.py", 1, 120000, 0.03),
       "second_kitti_all": ("second_kitti_all.py", 2, 120000, 0.03),
       "pointpillars_kitti_car": ("pointpillars_kitti_car.py", 8, 60000, 0.02)}
_PIPES = {}


def _pipeline(name):
    if name not in _PIPES:
        from det3d.models import build_detector
        from det3d.torchie import Config
        from det3d_b200.apis import InferencePipeline
        from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud
        cfg_file, _b, _n, pass_fraction = E2E[name]
        cfg = Config.fromfile(os.path.join(ROOT, "configs", cfg_file))
        torch.manual_seed(0)
        model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 0)
        calibrate_demo_weights_(model, cfg, [lidar_like_cloud(15000, cfg.voxel_generator.range, 4, 700 + i)
                                             for i in range(2)], 0, pass_fraction=pass_fraction)
        _PIPES[name] = InferencePipeline(cfg, model=model, device="cuda")
    return _PIPES[name]


def _raw_frames(batch, n, seed, pinned):
    from det3d_b200.utils.synthetic import KITTI_IMAGE_SHAPES, kitti_like_calib, raw_velodyne_scan
    scans = [raw_velodyne_scan(n - 997 * b, 4, seed=seed + b) for b in range(batch)]
    calibs = [kitti_like_calib(seed % 3 + b, KITTI_IMAGE_SHAPES[b % 4]) for b in range(batch)]
    if pinned:
        scans = [torch.from_numpy(s).pin_memory() for s in scans]
    return scans, calibs


def _cropped_on_host(scans, calibs):
    from det3d_b200.core.bbox.box_np_ops import camera_frustum_planes
    from oracle.frustum import keep_mask
    out = []
    for s, c in zip(scans, calibs):
        s = np.asarray(s)
        out.append(torch.from_numpy(s[keep_mask(s, camera_frustum_planes(c["rect"], c["Trv2c"], c["P2"],
                                                                         c["image_shape"]))]).pin_memory())
    return out


@pytest.mark.parametrize("name", sorted(E2E))
def test_infer_raw_equals_infer_host_on_the_cropped_clouds(name):
    pipe = _pipeline(name)
    _cfg, batch, n, _p = E2E[name]
    detections = 0
    for k in range(2):
        scans, calibs = _raw_frames(batch, n, 40 + k, pinned=k == 0)
        want = pipe.infer_host(_cropped_on_host(scans, calibs)).clone()
        eager = pipe.infer_raw(scans, calibs).clone()
        graphed = pipe.infer_raw(scans, calibs, graphed=True).clone()
        assert torch.equal(eager, want), k
        assert torch.equal(graphed, want), k
        detections += int((want[..., -1] > 0.5).sum())
    assert detections > 0
    assert int(pipe.overflow_flag().item()) == 0


def test_one_graph_serves_scans_of_distinct_sizes_and_calibrations():
    from det3d_b200.utils.synthetic import kitti_like_calib, raw_velodyne_scan
    pipe = _pipeline("second_kitti_car")
    pipe._graphs.clear()
    calibs = [kitti_like_calib(1), kitti_like_calib(2)]
    graph, entry, sizes = None, None, set()
    for k in range(6):
        scan = raw_velodyne_scan(100000 + 3000 * k, 4, seed=300 + k)
        sizes.add(scan.shape[0])
        cal = calibs[k // 2 % 2]                                       # calibration changes every other frame
        got = pipe.infer_raw([scan], [cal], graphed=True).clone()
        want = pipe.infer_host(_cropped_on_host([scan], [cal])).clone()
        assert torch.equal(got, want), k
        keys = [key for key in pipe._graphs if key[0] == "frustum"]
        assert len(keys) == 1 and keys[0] == ("frustum", 1, pipe.bucket_of(scan.shape[0]), 4)
        e = pipe._graphs[keys[0]]
        if graph is None:
            graph, entry = e.graph, e
        assert e is entry and e.graph is graph, "a graph was captured while the frames ran"
    assert len(sizes) == 6
    assert entry.planes_uploads == 3                                   # cal 1, cal 2, cal 1: only on change
    # forward_graphed's keys (batch, bucket, ndim) never collide with the crop's
    pipe.forward_graphed(torch.from_numpy(scan[:5000]), [0, 5000])
    assert ("frustum", 1, pipe.bucket_of(scan.shape[0]), 4) in pipe._graphs and (1, 8192, 4) in pipe._graphs


def test_graphed_forward_runs_no_vendor_kernel():
    import re

    from torch.profiler import ProfilerActivity, profile
    vendor_re = re.compile(r"cudnn|cublas|xmma|cutlass|gemm|winograd|convolve|fprop|dgrad|wgrad|fft[12]d|conv2d",
                           re.IGNORECASE)
    pipe = _pipeline("pointpillars_kitti_car")
    scans, calibs = _raw_frames(8, 60000, 90, pinned=True)
    pipe.infer_raw(scans, calibs, graphed=True)
    torch.cuda.synchronize()
    # the eager step is what the graph captures; then the replay itself.  Two frames per trace: after a few minutes of
    # GPU work in the same process, a trace can lack the device records of its first operations (a lone frame's H2D
    # copies and crop kernels were missing although their launches were recorded on the host), so the second frame is
    # the one the trace holds whole.
    for graphed in (False, True):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(2):
                pipe.infer_raw(scans, calibs, graphed=graphed)
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        if not graphed:
            assert any("crop_emit" in n for n in names) and any("bev_conv16" in n for n in names), sorted(names)
        vendor = sorted(n for n in names if vendor_re.search(n))
        assert not vendor, "vendor kernels on the %s forward: %s" % ("graphed" if graphed else "eager", vendor)


@pytest.mark.parametrize("image_in", ["metadata", "image"])
def test_test_pipeline_with_remove_outside_points_from_disk(tmp_path, image_in):
    """.bin files + info dicts -> LoadPointCloudFromFile, LoadPointCloudAnnotations, Preprocess(remove_outside_points)
    -> res["lidar"]["points"] == the reference's reduced array, bit for bit."""
    from det3d.datasets.pipelines import Compose
    g = load_golden("frustum_kitti_scans")
    clouds, masks = _golden_clouds(g)
    pre = dict(mode="val", shuffle_points=False, remove_environment=False, remove_unknown_examples=False,
               remove_outside_points=True)
    pipe = Compose([dict(type="LoadPointCloudFromFile"), dict(type="LoadPointCloudAnnotations", with_bbox=True),
                    dict(type="Preprocess", cfg=pre)])
    for b, (c, m) in enumerate(zip(clouds, masks)):
        path = tmp_path / ("%06d.bin" % b)
        c.tofile(str(path))
        info = dict(point_cloud=dict(velodyne_path=str(path), num_features=4),
                    calib=dict(R0_rect=g["rect"][b], Tr_velo_to_cam=g["Trv2c"][b], P2=g["P2"][b]))
        shape = g["image_shape"][b]
        meta = dict(image_prefix=str(tmp_path), num_point_features=4, token=b)
        res = dict(lidar=dict(type="lidar", points=None), metadata=meta, calib=None, cam={}, mode="val")
        if image_in == "image":
            res["image"] = dict(image_shape=shape)
            meta["image_shape"] = np.array([1, 1])                     # res["image"] wins, as in the reference
        else:
            meta["image_shape"] = shape
        out, _ = pipe(res, info)
        assert np.array_equal(_bits(out["lidar"]["points"]), _bits(c[m])), b
