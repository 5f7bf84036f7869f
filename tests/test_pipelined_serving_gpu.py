"""Frames in flight through every InferencePipeline entry point (block=False, PendingResult, max_in_flight): each
frame's output is bit-identical to what the same sequence of blocking calls gives -- across point-capacity buckets that
capture new graphs mid-sequence, in any collection order, with two entry points interleaved, and across an f16-range
overflow that re-runs the frames still in flight on tf32x3 -- and the blocking defaults keep their graph keys, captures
and table uploads."""
import warnings

import numpy as np
import pytest
import torch

from test_ingest_batched_gpu import _cbgs_pipeline, _nusc_samples
from test_kitti_results_gpu import E2E, _pipeline, _raw_frames
from test_nusc_results_gpu import _motion, _record
from test_pipelined_serving import assert_same

pytestmark = pytest.mark.gpu

SIZES = [15000, 40000, 9000, 70000, 20000, 33000, 16000]         # buckets 16k, 64k, 16k, 128k, 32k, 64k, 16k
_CBGS = []


def _cbgs():
    if not _CBGS:
        _CBGS.append(_cbgs_pipeline())
    return _CBGS[0]


def _same(a, b, where="frame"):
    """Packed tensors bit for bit (NaN included), anno lists / dicts by assert_same."""
    if torch.is_tensor(a):
        assert torch.is_tensor(b) and a.shape == b.shape and a.dtype == b.dtype, where
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), where
    else:
        assert_same(a, b, where)


def _clouds(ndim, seed, sizes=SIZES):
    from det3d_b200.utils.synthetic import lidar_like_cloud
    pcr = _pipeline("second_kitti_car").cfg.voxel_generator.range
    out = []
    for i, n in enumerate(sizes):
        c = lidar_like_cloud(n, pcr, ndim, seed + i)
        out.append(torch.from_numpy(c).pin_memory() if i % 2 == 0 else torch.from_numpy(c))   # pinned and pageable
    return out


def _run_modes(pipe, calls, depths=(2, 3), order=None):
    """Runs calls[i](block) -- one frame each -- blocking, then with block=False at each max_in_flight in `depths`,
    every mode from an empty graph cache.  Results are collected in `order` (default: submission order).  Asserts
    every frame equal to the blocking one and returns (blocking results, graph keys and capture count per mode)."""
    pipe.drain()
    modes = []
    pipe._graphs.clear()
    pipe.max_in_flight = 1
    want = [c(True) for c in calls]
    modes.append((list(pipe._graphs), len(pipe._graphs)))
    for depth in depths:
        pipe._graphs.clear()
        pipe.max_in_flight = depth
        handles = [c(False) for c in calls]
        assert len(pipe._pending) <= depth
        got = [None] * len(calls)
        for i in (range(len(calls)) if order is None else order):
            got[i] = handles[i].result()
        for i, (w, g) in enumerate(zip(want, got)):
            _same(g, w, "depth %d frame %d" % (depth, i))
            _same(handles[i].result(), w, "collected again: frame %d" % i)
            assert handles[i].done() and not handles[i].rerun
        modes.append((list(pipe._graphs), len(pipe._graphs)))
    pipe.max_in_flight = 2
    return want, modes


# ---- infer_host --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graphed", [True, False])
def test_infer_host_second(graphed):
    pipe = _pipeline("second_kitti_car")
    clouds = _clouds(4, 100)
    calls = [lambda block, c=c: pipe.infer_host([c], graphed=graphed, block=block) for c in clouds]
    want, modes = _run_modes(pipe, calls)
    assert sum(int((w[..., -1] > 0.5).sum()) for w in want) > 0
    if graphed:
        assert all(m == modes[0] for m in modes) and modes[0][1] == 4       # same keys and captures in every mode


@pytest.mark.parametrize("order", ["reverse", "shuffled"])
def test_collection_order_does_not_matter(order):
    pipe = _pipeline("second_kitti_car")
    clouds = _clouds(4, 200)
    idx = list(range(len(clouds)))[::-1] if order == "reverse" else [3, 0, 6, 2, 5, 1, 4]
    calls = [lambda block, c=c: pipe.infer_host([c], graphed=True, block=block) for c in clouds]
    _run_modes(pipe, calls, order=idx)


def test_pinned_out_is_the_callers_buffer():
    pipe = _pipeline("second_kitti_car")
    clouds = _clouds(4, 300, SIZES[:3])
    want = [pipe.infer_host([c], graphed=True).clone() for c in clouds]
    outs = [torch.empty_like(w).pin_memory() for w in want]
    pipe.max_in_flight = 3
    handles = [pipe.infer_host([c], pinned_out=o, graphed=True, block=False) for c, o in zip(clouds, outs)]
    for h, o, w in zip(handles, outs, want):
        assert h.result() is o
        _same(o, w)
    pipe.max_in_flight = 2


# ---- infer_raw ---------------------------------------------------------------------------------------------------
def _raw_calls(pipe, name, kitti_results, graphed=True):
    _cfg, batch, n, _pf = E2E[name]
    calls = []
    for f, scale in enumerate([1.0, 0.3, 1.0, 0.55, 0.3, 1.0]):             # raw buckets cross twice
        scans, calibs = _raw_frames(batch, int(n * scale), 40 + 7 * f, pinned=f % 2 == 0)
        calls.append(lambda block, s=scans, c=calibs: pipe.infer_raw(s, c, graphed=graphed, kitti_results=kitti_results,
                                                                      block=block))
    return calls


@pytest.mark.parametrize("kitti_results", [False, True])
@pytest.mark.parametrize("name", ["second_kitti_car", "pointpillars_kitti_car"])
def test_infer_raw(name, kitti_results):
    pipe = _pipeline(name)
    want, modes = _run_modes(pipe, _raw_calls(pipe, name, kitti_results))
    assert all(m == modes[0] for m in modes)
    if kitti_results:
        assert sum(len(a["name"]) for w in want for a in w) > 0


# ---- infer_sweeps ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nusc_results", [False, True])
def test_infer_sweeps_cbgs(nusc_results):
    pipe = _cbgs()
    calls = []
    for f, per_sweep in enumerate([3500, 1200, 3500, 2500, 1200, 3500]):     # raw buckets cross
        samples = _nusc_samples(pipe, 2, 60 + f, per_sweep=per_sweep, pinned=f % 2 == 0)
        kw = dict(nusc_results=True, poses=[_record(5 * f + b) for b in range(2)],
                  tokens=["f%d_%d" % (f, b) for b in range(2)]) if nusc_results else {}
        calls.append(lambda block, s=samples, kw=kw: pipe.infer_sweeps(s, graphed=True, block=block, **kw))
    want, modes = _run_modes(pipe, calls)
    assert all(m == modes[0] for m in modes)
    if nusc_results:
        assert sum(len(v) for w in want for v in w["results"].values()) > 0


# ---- interleaved entry points --------------------------------------------------------------------------------------
def test_two_entry_points_interleaved():
    pipe = _pipeline("second_kitti_car")
    clouds = _clouds(4, 400, SIZES[:4])
    raw = _raw_calls(pipe, "second_kitti_car", True)[:4]
    calls = []
    for c, r in zip(clouds, raw):
        calls += [lambda block, c=c: pipe.infer_host([c], graphed=True, block=block), r]
    _run_modes(pipe, calls)


# ---- SweepStream ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nusc_results", [False, True])
def test_sweep_stream_frames_in_flight(nusc_results):
    from det3d_b200.apis import SweepStream
    from det3d_b200.utils.synthetic import lidar_like_cloud
    pipe = _cbgs()
    pipe.drain()
    B, K, k, frames = 2, 4, 3, 9
    rng = np.random.default_rng(3)
    pcr = pipe.cfg.voxel_generator.range
    pushes = []
    poses, t = [np.eye(4) for _ in range(B)], 0.0
    for f in range(frames):
        t += 0.05
        frame = []
        for b in range(B):
            poses[b] = poses[b] @ _motion(rng)
            c = lidar_like_cloud(int(rng.integers(1500, 5000)), pcr, 5, 77 * f + b)
            frame.append((torch.from_numpy(c).pin_memory() if b == 0 else c, poses[b].copy(), t))
        pushes.append(frame)

    def kw(f):
        return dict(nusc_results=True, poses=[_record(3 * f + b) for b in range(B)],
                    tokens=["s%d_%d" % (f, b) for b in range(B)]) if nusc_results else {}

    blocking = SweepStream(pipe, B, K, 5000)
    want = []
    for f in range(frames):
        for b, (c, p, ts) in enumerate(pushes[f]):
            blocking.push(b, c, p, ts)
        want.append(blocking.infer(graphed=True, **kw(f)))
    stream = SweepStream(pipe, B, K, 5000, in_flight=k)
    assert stream.key == blocking.key + (("in_flight", k),) and stream.sweeps.slots == K + k - 1
    pipe.max_in_flight = k
    handles, samples, refused = [], [], 0
    for f in range(frames):
        while len(pipe._pending) > k - 1:
            if f >= K + k - 1:                                  # every slot is held: the push is refused
                with pytest.raises(ValueError, match="unfinished"):
                    stream.push(0, *pushes[f][0])
                refused += 1
            pipe._pending[0].result()
        for b, (c, p, ts) in enumerate(pushes[f]):
            stream.push(b, c, p, ts)
        handles.append(stream.infer(graphed=True, block=False, **kw(f)))
        samples.append(stream.samples())
    assert refused > 0
    for f in reversed(range(frames)):
        _same(handles[f].result(), want[f], "frame %d" % f)
    pipe.max_in_flight = 2
    assert all(c == 0 for r in stream.sweeps.readers for c in r)
    for f in range(frames):                                     # the frames are still infer_sweeps(samples())'
        _same(pipe.infer_sweeps(samples[f], **kw(f)), want[f], "infer_sweeps frame %d" % f)


# ---- overflow ------------------------------------------------------------------------------------------------------
def _fresh_second(math=None):
    from det3d.models import build_detector
    from det3d_b200.apis import InferencePipeline
    src = _pipeline("second_kitti_car")
    model = build_detector(src.cfg.model, train_cfg=None, test_cfg=src.cfg.test_cfg)
    model.load_state_dict({k: v.detach().cpu() for k, v in src.model.state_dict().items()})
    pipe = InferencePipeline(src.cfg, model=model.eval(), device="cuda")
    if math is not None:
        pipe.set_math(math)
    return pipe


def _overflow_clouds():
    """Six frames of SECOND; frame 3 carries points whose intensity (1e7) drives the first sparse layer past the f16
    range."""
    clouds = _clouds(4, 500, [15000, 40000, 9000, 20000, 33000, 16000])
    hot = clouds[3].clone()
    hot[::50, 3] = 1e7
    clouds[3] = hot.pin_memory()
    return clouds


def _serve_all(pipe, clouds, graphed, block):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        out = [pipe.infer_host([c], graphed=graphed, block=block) for c in clouds]
        if not block:
            out = [h.result() for h in out], out
    return out, sum("f16 range" in str(w.message) for w in caught)


@pytest.mark.parametrize("graphed", [True, False])
def test_overflow_in_frame_3_of_6(graphed):
    clouds = _overflow_clouds()
    blocking = _fresh_second()
    want, warned = _serve_all(blocking, clouds, graphed, True)
    assert warned == 1 and blocking.model.math == "tf32x3"
    # frames 0-2 ran on FP16x3, frames 3-5 on tf32x3
    fp16 = _fresh_second()
    for f in range(3):
        _same(want[f], fp16.infer_host([clouds[f]], graphed=graphed), "fp16x3 frame %d" % f)
    tf32 = _fresh_second("tf32x3")
    for f in range(3, 6):
        _same(want[f], tf32.infer_host([clouds[f]], graphed=graphed), "tf32x3 frame %d" % f)
    for depth in (2, 3):
        pipe = _fresh_second()
        pipe.max_in_flight = depth
        (got, handles), warned = _serve_all(pipe, clouds, graphed, False)
        assert warned == 1 and pipe.model.math == "tf32x3"
        for f in range(6):
            _same(got[f], want[f], "depth %d frame %d" % (depth, f))
        # no frame before the one that overflowed was blamed for it
        assert [h.rerun for h in handles[:4]] == [False, False, False, True], depth
        assert int(pipe.overflow_flag().item()) == 0


def test_a_raised_flag_names_its_frame():
    """Frame 3 overflows and has finished on the device before frames 0-2 are collected: their results are still the
    FP16x3 ones, and only frame 3 is re-run."""
    clouds = _overflow_clouds()[:4]
    fp16 = _fresh_second()
    want = [fp16.infer_host([c], graphed=True) for c in clouds[:3]]
    pipe = _fresh_second()
    pipe.max_in_flight = 4
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        handles = [pipe.infer_host([c], graphed=True, block=False) for c in clouds]
        torch.cuda.synchronize()
        for f in range(3):
            _same(handles[f].result(), want[f], "frame %d" % f)
        assert pipe.model.math == "fp16x3"
        handles[3].result()
    assert [h.rerun for h in handles] == [False, False, False, True] and pipe.model.math == "tf32x3"


# ---- defaults ------------------------------------------------------------------------------------------------------
def test_blocking_defaults_keep_keys_captures_and_uploads():
    pipe = _pipeline("second_kitti_car")
    pipe.drain()
    assert pipe.max_in_flight == 2
    pipe._graphs.clear()
    pipe.max_in_flight = 1
    scans, calibs = _raw_frames(1, 120000, 11, pinned=True)
    _s2, calibs2 = _raw_frames(1, 120000, 13, pinned=True)
    for c in (calibs, calibs, calibs2, calibs2, calibs):
        annos = pipe.infer_raw(scans, c, graphed=True, kitti_results=True)
        assert isinstance(annos, list)
    packed = pipe.infer_host([scans[0][:20000]], graphed=True)
    assert torch.is_tensor(packed) and packed.is_pinned()
    bucket = pipe.bucket_of(scans[0].shape[0])
    assert list(pipe._graphs) == [("frustum_kitti", 1, bucket, 4), (1, 32768, 4)]
    e = pipe._graphs[("frustum_kitti", 1, bucket, 4)]
    assert e.calib_uploads == 3 and e.planes_uploads == 3
    pipe.max_in_flight = 2


def test_stream_default_key_and_pose_uploads():
    from det3d_b200.apis import SweepStream
    from det3d_b200.utils.synthetic import lidar_like_cloud
    pipe = _cbgs()
    pipe.drain()
    st = SweepStream(pipe, 2, 4, 5000)
    assert st.key == ("stream", 2, 4, 5000, 5, 4) and st.sweeps.slots == 4
    pipe._graphs.pop(st.key + ("nusc",), None)
    for f in range(4):
        for b in range(2):
            st.push(b, lidar_like_cloud(3000, pipe.cfg.voxel_generator.range, 5, 10 * f + b), np.eye(4), 0.05 * f)
        st.infer(graphed=True, nusc_results=True, poses=[_record(100 + b + 10 * (f // 2)) for b in range(2)],
                 tokens=["d%d_%d" % (f, b) for b in range(2)])
    assert pipe._graphs[st.key + ("nusc",)].pose_uploads == 2


def test_validation_errors_come_before_anything_is_enqueued():
    pipe = _pipeline("second_kitti_car")
    pipe.drain()
    scans, calibs = _raw_frames(1, 20000, 1, pinned=False)
    with pytest.raises(ValueError):
        pipe.infer_raw(scans, calibs + calibs, graphed=True, block=False)
    assert len(pipe._pending) == 0
