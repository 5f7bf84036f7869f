"""nuScenes result rows on the device (d3b_nusc_results_dev, csrc/nusc_results.cu) and multi-sweep samples -> nusc_annos
(InferencePipeline.infer_sweeps(nusc_results=True), SweepStream.infer(nusc_results=True),
datasets.nuscenes.convert_detection_to_nusc_annos).

The kernel's rows are compared with the reference's (tests/golden/nusc_results_*.npz) within oracle/nusc_results'
error bound, and bit for bit on the exact golden.  End to end, the annos must be the reference's conversion
(oracle.nusc_results.reference_annos) of infer_sweeps' own detections."""
import warnings

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import nusc_results as onr
from test_ingest_batched_gpu import _cbgs_pipeline, _nusc_samples, _pillars_nusc_pipeline, _raise_deblock_overflow

pytestmark = pytest.mark.gpu

U = 2.0 ** -53


def _u64(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def _records(g):
    return [{"calibrated_sensor": {"translation": list(g["cs_translation"][b]), "rotation": list(g["cs_rotation"][b])},
             "ego_pose": {"translation": list(g["ego_translation"][b]), "rotation": list(g["ego_rotation"][b])}}
            for b in range(g["packed"].shape[0])]


def _run(packed, tables, poison=True):
    """One d3b_nusc_results_dev call; the result buffer holds NaN before it.  -> (results, counts) on the host."""
    from det3d_b200.ops.point_cloud.nusc_results import NuscResults
    nr = NuscResults(packed.shape[0])
    nr.set_poses(tables)
    det = torch.from_numpy(np.ascontiguousarray(packed)).cuda()
    nr.launch(det)
    if poison:
        nr.results.fill_(float("nan"))
        nr.counts.fill_(-1)
        nr.launch(det)
    return nr.results.cpu().numpy(), nr.counts.cpu().numpy()


def _within(got, want, bound):
    return bool(np.all((got == want) | (np.abs(got - want) <= bound)))


def _check_sample(got_rows, count, packed, table, record=None):
    """The kernel's rows of one sample against the oracle: copies and flags equal, the rest within the bound."""
    rows, valid, _a = onr.kernel_order(packed, table)
    bound, margin = onr.error_bound(packed, table, record)
    assert count == int(valid.sum())
    assert np.all(margin[valid] > 1)
    got, want = got_rows[:count], rows[valid]
    assert np.array_equal(_u64(got[:, 3:6]), _u64(want[:, 3:6]))
    assert np.array_equal(got[:, 12:15], want[:, 12:15])
    assert _within(got[:, :12], want[:, :12], bound[valid][:, :12])
    assert np.all(got_rows[count:] == 0) and not np.signbit(got_rows[count:]).any()
    return got


@pytest.mark.parametrize("case", ["cases", "exact"])
def test_kernel_equals_the_reference(case):
    from det3d_b200.ops.point_cloud.nusc_results import to_nusc_annos
    g = load_golden("nusc_results_" + case)
    results, counts = _run(g["packed"], g["tables"])
    assert np.array_equal(counts, g["counts"])
    off = np.concatenate([[0], np.cumsum(g["counts"])])
    recs = _records(g)
    for b in range(g["packed"].shape[0]):
        got = _check_sample(results[b], counts[b], g["packed"][b], g["tables"][b], recs[b])
        s = slice(off[b], off[b + 1])
        want = np.concatenate([g["translation"][s], g["size"][s], g["rotation"][s], g["velocity"][s]], 1)
        bound, _m = onr.error_bound(g["packed"][b], g["tables"][b], recs[b])
        assert np.array_equal(got[:, 3:6], want[:, 3:6])
        assert np.array_equal(got[:, 12], g["score"][s]) and np.array_equal(got[:, 13], g["label"][s])
        assert _within(got[:, :12], want, bound[g["packed"][b][:, 11] > 0.5][:, :12])
        if case == "exact":
            assert np.array_equal(got[:, :12], want), b
    names, tokens = [str(n) for n in g["class_names"]], [str(t) for t in g["tokens"]]
    annos = to_nusc_annos(results, counts, names, tokens)
    assert list(annos["results"]) == tokens
    flat = [a for t in tokens for a in annos["results"][t]]
    assert [a["detection_name"] for a in flat] == list(g["names"])
    assert [a["attribute_name"] for a in flat] == list(g["attributes"])


@pytest.mark.parametrize("batch", [1, 4, 64])
def test_batches_with_empty_samples_equal_each_sample_alone(batch):
    g = load_golden("nusc_results_cases")
    rng = np.random.default_rng(batch)
    pick = rng.integers(0, g["packed"].shape[0], batch)
    pick[rng.integers(0, batch)] = 3                                    # the sample with no valid detection
    packed, tables = g["packed"][pick], g["tables"][pick]
    results, counts = _run(packed, tables)
    for b in range(batch):
        alone, n = _run(packed[b:b + 1], tables[b:b + 1], poison=False)
        assert counts[b] == n[0] and np.array_equal(_u64(results[b]), _u64(alone[0])), b
        _check_sample(results[b], counts[b], packed[b], tables[b])
    assert 0 in counts


def test_runs_and_graph_replays_are_bit_identical():
    from det3d_b200.ops.point_cloud.nusc_results import NuscResults
    g = load_golden("nusc_results_cases")
    nr = NuscResults(g["packed"].shape[0])
    nr.set_poses(g["tables"])
    det = torch.from_numpy(g["packed"]).cuda()
    first = [t.clone() for t in nr.launch(det)]
    second = [t.clone() for t in nr.launch(det)]
    assert torch.equal(first[0].view(torch.int64), second[0].view(torch.int64)) and torch.equal(first[1], second[1])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        nr.launch(det)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        nr.launch(det)
    for _ in range(2):
        nr.results.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(nr.results.view(torch.int64), first[0].view(torch.int64))
        assert torch.equal(nr.counts, first[1])


# ---- end to end ---------------------------------------------------------------------------------------------------
def _quat(axis, angle):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return np.concatenate([[np.cos(angle / 2)], axis * np.sin(angle / 2)])


def _record(seed):
    """A nuScenes-like key-frame record: LIDAR_TOP about -90 deg about z, the ego 300-2500 m out at any yaw."""
    rng = np.random.default_rng(seed)
    cs_q = onr._q_matrix(_quat([0, 0, 1], -np.pi / 2 + rng.uniform(-0.02, 0.02))) @ _quat([1, 0, 0],
                                                                                           rng.uniform(-0.005, 0.005))
    ego_q = onr._q_matrix(_quat([0, 0, 1], rng.uniform(-np.pi, np.pi))) @ _quat([0, 1, 0], rng.uniform(-0.03, 0.03))
    r, a = rng.uniform(300, 2500), rng.uniform(-np.pi, np.pi)
    return {"calibrated_sensor": {"translation": [0.94, 0.0, 1.84], "rotation": [float(v) for v in cs_q]},
            "ego_pose": {"translation": [r * np.cos(a), r * np.sin(a), 0.1], "rotation": [float(v) for v in ego_q]}}


def _same_annos(a, b):
    """Two nusc_annos dicts: equal keys, order, types and values, floats bit for bit."""
    return (list(a) == list(b) and a["meta"] == b["meta"] and list(a["results"]) == list(b["results"])
            and all(len(a["results"][t]) == len(b["results"][t]) and
                    all(list(x) == list(y) and repr(x) == repr(y) for x, y in zip(a["results"][t], b["results"][t]))
                    for t in a["results"]))


def _assert_annos_are_the_reference(annos, packed, records, tokens, pipe):
    """annos (the device path's) against the reference's conversion of the same packed detections: keys, types, order,
    names, attributes, sizes and scores equal, the rest within the bound.  Returns the box count."""
    from det3d_b200.ops.point_cloud.nusc_results import pose_table
    ref = onr.reference_annos(packed, records, tokens, pipe.class_names())
    assert list(annos) == list(ref) and annos["meta"] == ref["meta"] and list(annos["results"]) == tokens
    n = 0
    for b, t in enumerate(tokens):
        got, want = annos["results"][t], ref["results"][t]
        assert len(got) == len(want)
        bound, margin = onr.error_bound(packed[b], pose_table(records[b]), records[b])
        valid = packed[b][:, 11] > 0.5
        assert np.all(margin[valid] > 1), "a speed decision inside the error bound"
        bound = bound[valid]
        for i, (x, y) in enumerate(zip(got, want)):
            assert list(x) == list(y) and all(type(x[k]) is type(y[k]) for k in y)
            for k in ("sample_token", "size", "detection_name", "detection_score", "attribute_name"):
                assert x[k] == y[k], (t, i, k)
            for k, cols in (("translation", slice(0, 3)), ("rotation", slice(6, 10)), ("velocity", slice(10, 12))):
                assert _within(np.array(x[k]), np.array(y[k]), bound[i, cols]), (t, i, k)
        n += len(got)
    return n


_PIPES = {}


def _pipe(name):
    if name not in _PIPES:
        _PIPES[name] = _cbgs_pipeline() if name == "cbgs" else _pillars_nusc_pipeline()
    return _PIPES[name]


@pytest.mark.parametrize("name", ["cbgs", "pillars_nusc"])
def test_infer_sweeps_nusc_results_equal_the_reference_conversion(name):
    from det3d_b200.datasets.nuscenes import convert_detection_to_nusc_annos
    pipe = _pipe(name)
    boxes = 0
    for k in range(2):
        samples = _nusc_samples(pipe, 4, 500 + k, pinned=k == 0)
        records = [_record(10 * k + b) for b in range(4)]
        tokens = ["tok%d_%d" % (k, b) for b in range(4)]
        packed = pipe.infer_sweeps(samples).clone().numpy()
        eager = pipe.infer_sweeps(samples, nusc_results=True, poses=records, tokens=tokens)
        graphed = pipe.infer_sweeps(samples, graphed=True, nusc_results=True, poses=records, tokens=tokens)
        again = pipe.infer_sweeps(samples, graphed=True, nusc_results=True, poses=records, tokens=tokens)
        assert _same_annos(eager, graphed) and _same_annos(graphed, again)
        boxes += _assert_annos_are_the_reference(graphed, packed, records, tokens, pipe)
        # the plain infer_sweeps still returns the same detections after the nuScenes graph ran
        assert np.array_equal(pipe.infer_sweeps(samples, graphed=True).numpy().view(np.uint32), packed.view(np.uint32))
        free = convert_detection_to_nusc_annos(torch.from_numpy(packed).cuda(), records, tokens, pipe.class_names())
        assert _same_annos(free, graphed)
    assert boxes > 0
    assert int(pipe.overflow_flag().item()) == 0


def _motion(rng, yaw=0.05, shift=1.5):
    a = rng.uniform(-yaw, yaw)
    m = np.eye(4)
    m[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    m[:3, 3] = rng.uniform(-shift, shift, 3) * [1, 1, 0.05]
    return m


@pytest.mark.parametrize("name", ["cbgs", "pillars_nusc"])
def test_stream_nusc_results_equal_infer_sweeps_and_upload_poses_on_change(name):
    from det3d_b200.apis import SweepStream
    from det3d_b200.utils.synthetic import lidar_like_cloud
    pipe = _pipe(name)
    rng = np.random.default_rng(9)
    st = SweepStream(pipe, 4, 10, 5000)
    key = st.key + ("nusc",)
    pipe._graphs.pop(key, None)
    poses, t = [np.eye(4) for _ in range(4)], 0.0
    entry = graph = None
    boxes = 0
    for f in range(6):
        t += 0.05
        for b in range(4):
            poses[b] = poses[b] @ _motion(rng)
            st.push(b, lidar_like_cloud(int(rng.integers(3000, 5000)), pipe.cfg.voxel_generator.range, 5, 90 * f + b),
                    poses[b], t)
        records = [_record(1000 + b + 10 * (f // 2)) for b in range(4)]           # records change every other frame
        tokens = ["f%d_%d" % (f, b) for b in range(4)]
        got = st.infer(graphed=True, nusc_results=True, poses=records, tokens=tokens)
        samples = st.samples()
        want = pipe.infer_sweeps(samples, nusc_results=True, poses=records, tokens=tokens)
        assert _same_annos(got, want), f
        boxes += _assert_annos_are_the_reference(got, pipe.infer_sweeps(samples).clone().numpy(), records, tokens, pipe)
        e = pipe._graphs[key]
        if entry is None:
            entry, graph = e, e.graph
        assert e is entry and e.graph is graph, "a graph was captured while the frames ran"
    assert entry.pose_uploads == 3
    assert boxes > 0


@pytest.mark.parametrize("graphed", [False, True])
def test_overflow_reruns_on_tf32x3_and_converts_its_detections(graphed):
    pipe = _pillars_nusc_pipeline(_raise_deblock_overflow)
    samples = _nusc_samples(pipe, 1, 301)
    records, tokens = [_record(77)], ["overflow"]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        got = pipe.infer_sweeps(samples, graphed=graphed, nusc_results=True, poses=records, tokens=tokens)
    assert any("f16 range" in str(w.message) for w in caught), [str(w.message) for w in caught]
    assert pipe.model.math == "tf32x3" and int(pipe.overflow_flag().item()) == 0
    packed = pipe.infer_sweeps(samples, graphed=graphed).clone().numpy()         # the tf32x3 detections
    assert _assert_annos_are_the_reference(got, packed, records, tokens, pipe) > 0
    assert _same_annos(got, pipe.infer_sweeps(samples, graphed=graphed, nusc_results=True, poses=records,
                                              tokens=tokens))
