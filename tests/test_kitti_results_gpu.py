"""KITTI result rows on the device (d3b_kitti_results_dev, csrc/kitti_results.cu) and raw scans -> KITTI annos
(InferencePipeline.infer_raw(kitti_results=True), datasets.kitti.convert_detection_to_kitti_annos).

The kernel's rows are compared with the reference's (tests/golden/kitti_results_*.npz) within oracle/kitti_results'
error bound, and bit for bit with the oracle's fixed-order restatement wherever no sin / cos / atan2 enters (location,
dimensions, rotation_y, score, label); on the exact golden the image boxes are compared bit for bit too.  End to end, the
annos must be the reference's conversion (oracle.kitti_results.reference_annos, pinned to the reference's own functions
by the golden generator) of infer_raw's own detections."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import kitti_results as okr

pytestmark = pytest.mark.gpu

CASES = ("cases", "nd9", "exact")
ORACLE_EXACT = [5, 6, 7, 8, 9, 10, 11, 12, 13]       # no transcendental on their path: the oracle's bits
REF_EXACT = [5, 6, 7, 11, 12, 13]                    # copies of float32 values: the reference's bits


def _u64(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _same_bits(a, b):
    """Bit for bit, except that any NaN equals any NaN (CUDA's canonical NaN is not x86's)."""
    return a.shape == b.shape and bool(np.all((_u64(a) == _u64(b)) | (np.isnan(a) & np.isnan(b))))


def _same_anno(a, b):
    """Two anno dicts: the same keys, dtypes and values (a NaN equals a NaN)."""
    return list(a) == list(b) and all(
        a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f") for k in a)


def _within(got, want, bound):
    with np.errstate(invalid="ignore"):
        return bool(np.all((got == want) | (np.isnan(got) & np.isnan(want)) | (np.abs(got - want) <= bound)))


def _run(packed, tables, poison=True):
    """One d3b_kitti_results_dev call; the result buffer holds NaN before it.  -> (results, counts) on the host."""
    from det3d_b200.ops.point_cloud.kitti_results import KittiResults
    kr = KittiResults(packed.shape[0])
    kr.set_calib(tables)
    det = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
    kr.launch(det)
    if poison:
        kr.results.fill_(float("nan"))
        kr.counts.fill_(-1)
        kr.launch(det)
    return kr.results.cpu().numpy(), kr.counts.cpu().numpy()


def _check_frame(got_rows, count, packed, nd, table, want_rows=None, exact=False):
    """The kernel's rows of one frame against the oracle (bits / bound) and the reference's kept rows."""
    rows, keep, _a = okr.kernel_order(packed, nd, table)
    bound, margin = okr.error_bound(packed, nd, table)
    assert count == int(keep.sum())
    got = got_rows[:count]
    assert _same_bits(got[:, ORACLE_EXACT], rows[keep][:, ORACLE_EXACT])
    assert _within(got[:, :5], rows[keep][:, :5], bound[keep][:, :5])
    assert np.all(got_rows[count:] == 0) and not np.signbit(got_rows[count:]).any()
    if want_rows is not None:
        assert got.shape == want_rows.shape
        assert _same_bits(got[:, REF_EXACT], want_rows[:, REF_EXACT])
        assert _within(got[:, :5], want_rows[:, :5], bound[keep][:, :5])
        assert _within(got[:, 8:11], want_rows[:, 8:11], bound[keep][:, 8:11])
        if exact:
            assert np.array_equal(got[:, :4], want_rows[:, :4])
    return margin


@pytest.mark.parametrize("case", CASES)
def test_kernel_equals_the_reference(case):
    g = load_golden("kitti_results_" + case)
    nd = int(g["nd"])
    results, counts = _run(g["packed"], g["tables"])
    assert np.array_equal(counts, g["counts"])
    off = np.concatenate([[0], np.cumsum(g["counts"])])
    for b in range(g["packed"].shape[0]):
        _check_frame(results[b], counts[b], g["packed"][b], nd, g["tables"][b], g["rows"][off[b]:off[b + 1]],
                     exact=case == "exact")


@pytest.mark.parametrize("batch", [1, 7, 64])
def test_batches_with_empty_samples_equal_each_sample_alone(batch):
    g = load_golden("kitti_results_cases")
    rng = np.random.default_rng(batch)
    pick = rng.integers(0, g["packed"].shape[0], batch)
    pick[rng.integers(0, batch)] = 5                                    # the frame with no valid detection
    packed, tables = g["packed"][pick], g["tables"][pick]
    results, counts = _run(packed, tables)
    for b in range(batch):
        alone, n = _run(packed[b:b + 1], tables[b:b + 1], poison=False)
        assert counts[b] == n[0] and np.array_equal(_u64(results[b]), _u64(alone[0])), b
        _check_frame(results[b], counts[b], packed[b], 7, tables[b])
    assert 0 in counts


def test_runs_and_graph_replays_are_bit_identical():
    from det3d_b200.ops.point_cloud.kitti_results import KittiResults
    g = load_golden("kitti_results_cases")
    kr = KittiResults(g["packed"].shape[0])
    kr.set_calib(g["tables"])
    det = torch.from_numpy(g["packed"]).cuda()
    first = [t.clone() for t in kr.launch(det)]
    second = [t.clone() for t in kr.launch(det)]
    assert all(torch.equal(a.view(torch.int64) if a.dtype == torch.float64 else a,
                           b.view(torch.int64) if b.dtype == torch.float64 else b) for a, b in zip(first, second))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        kr.launch(det)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        kr.launch(det)
    for _ in range(2):
        kr.results.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(kr.results.view(torch.int64), first[0].view(torch.int64))
        assert torch.equal(kr.counts, first[1])


# ---- end to end ---------------------------------------------------------------------------------------------------
E2E = {"second_kitti_car": ("second_kitti_car.py", 1, 120000, 0.03),
       "second_kitti_all": ("second_kitti_all.py", 2, 120000, 0.03),
       "pointpillars_kitti_car": ("pointpillars_kitti_car.py", 8, 60000, 0.02)}
_PIPES = {}


def _pipeline(name):
    if name not in _PIPES:
        import os

        from conftest import ROOT
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


def _assert_annos_are_the_reference(annos, packed, calibs, class_names):
    """annos (the device path's) against the reference's conversion of the same packed detections: keys, dtypes,
    names, the kept set and order, exact fields bit for bit, the rest within the bound.  Returns the kept count."""
    from det3d_b200.ops.point_cloud.kitti_results import calib_table
    nd = packed.shape[-1] - 3
    kept = 0
    for b, (a, cal) in enumerate(zip(annos, calibs)):
        ref = okr.reference_annos(packed[b], nd, cal, class_names)
        assert list(a) == list(ref)
        for k in ref:
            assert a[k].dtype == ref[k].dtype and a[k].shape == ref[k].shape, (b, k)
        _rows, keep, _aux = okr.kernel_order(packed[b], nd, calib_table(cal))
        bound, margin = okr.error_bound(packed[b], nd, calib_table(cal))
        assert np.all(margin[packed[b][:, nd + 2] > 0.5] > 1), "a decision inside the error bound"
        bd = bound[keep]
        assert list(a["name"]) == list(ref["name"])
        for k in ("rotation_y", "score", "dimensions"):
            assert np.array_equal(a[k], ref[k]), (b, k)
        assert _within(a["bbox"], ref["bbox"], bd[:, :4])
        assert _within(a["alpha"], ref["alpha"], bd[:, 4])
        assert _within(a["location"], ref["location"], bd[:, 8:11])
        kept += a["name"].shape[0]
    return kept


@pytest.mark.parametrize("name", sorted(E2E))
def test_infer_raw_kitti_results_equal_the_reference_conversion(name):
    from det3d_b200.datasets.kitti import convert_detection_to_kitti_annos
    pipe = _pipeline(name)
    _cfg, batch, n, _p = E2E[name]
    kept = 0
    for k in range(2):
        scans, calibs = _raw_frames(batch, n, 40 + k, pinned=k == 0)
        packed = pipe.infer_raw(scans, calibs).clone().numpy()
        graphed_packed = pipe.infer_raw(scans, calibs, graphed=True).clone().numpy()
        assert np.array_equal(packed.view(np.uint32), graphed_packed.view(np.uint32))
        eager = pipe.infer_raw(scans, calibs, kitti_results=True)
        graphed = pipe.infer_raw(scans, calibs, graphed=True, kitti_results=True)
        again = pipe.infer_raw(scans, calibs, graphed=True, kitti_results=True)
        for x, y in ((eager, graphed), (graphed, again)):
            assert all(_same_anno(a, b) for a, b in zip(x, y))
        kept += _assert_annos_are_the_reference(graphed, packed, calibs, pipe.class_names())
        # the plain infer_raw still returns the same detections after the KITTI graph ran
        assert np.array_equal(pipe.infer_raw(scans, calibs, graphed=True).numpy().view(np.uint32),
                              packed.view(np.uint32))
        free = convert_detection_to_kitti_annos(torch.from_numpy(packed).cuda(), calibs, pipe.class_names())
        assert all(_same_anno(a, b) for a, b in zip(free, graphed))
    assert kept > 0
    assert int(pipe.overflow_flag().item()) == 0


def test_a_scan_gives_the_same_annos_alone_and_in_a_batch():
    pipe = _pipeline("pointpillars_kitti_car")
    scans, calibs = _raw_frames(8, 60000, 70, pinned=True)
    batch = pipe.infer_raw(scans, calibs, graphed=True, kitti_results=True)
    for b in (0, 5):
        alone = pipe.infer_raw(scans[b:b + 1], calibs[b:b + 1], graphed=True, kitti_results=True)[0]
        assert _same_anno(alone, batch[b]), b


def test_calibration_table_goes_up_only_when_it_changes():
    from det3d_b200.utils.synthetic import kitti_like_calib, raw_velodyne_scan
    pipe = _pipeline("second_kitti_car")
    pipe._graphs.clear()
    calibs = [kitti_like_calib(1), kitti_like_calib(2)]
    entry = graph = None
    for k in range(6):
        scan = raw_velodyne_scan(100000 + 3000 * k, 4, seed=500 + k)
        cal = calibs[k // 2 % 2]                                       # calibration changes every other frame
        got = pipe.infer_raw([scan], [dict(cal)], graphed=True, kitti_results=True)
        packed = pipe.infer_raw([scan], [cal]).numpy()
        _assert_annos_are_the_reference(got, packed, [cal], pipe.class_names())
        key = ("frustum_kitti", 1, pipe.bucket_of(scan.shape[0]), 4)
        e = pipe._graphs[key]
        if entry is None:
            entry, graph = e, e.graph
        assert e is entry and e.graph is graph, "a graph was captured while the frames ran"
    assert entry.calib_uploads == 3 and entry.planes_uploads == 3       # cal 1, cal 2, cal 1: only on change
    assert len(pipe._kitti_tables) == 2
