"""Batched multi-sweep ingest with a device sweep table (d3b_ingest_sweeps_dev, ingest_sweeps_batched,
InferencePipeline.infer_sweeps): every sample's rows are the bits that sample gives as a batch of one (ingest_sweeps;
its values are pinned by the reference golden in test_ingest.py), one captured graph serves tables of any size,
malformed device tables are clamped and reported, and detections from raw sweeps equal the per-sample ingest followed
by infer_host, for the CBGS and nuScenes PointPillars configs."""
import argparse
import os
import warnings

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

pytestmark = pytest.mark.gpu

PCR = [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]


def _sample(sizes, seed, close=0.05):
    from det3d_b200.utils.synthetic import lidar_like_sweeps
    return lidar_like_sweeps(sizes, PCR, seed, close_fraction=close)


def _golden_sample():
    from test_ingest import _sweep_records
    g = load_golden("ingest_nusc_3sweeps")
    return _sweep_records(g)


def _per_sample(samples):
    """Each sample ingested as a batch of one, cut to its rows."""
    from det3d.datasets.pipelines.loading import ingest_sweeps
    return [ingest_sweeps(*s) for s in samples]


def _check_rows(samples, points, offsets):
    offs = offsets.cpu().tolist()
    want = _per_sample(samples)
    assert offs[0] == 0
    for b, w in enumerate(want):
        got = points[offs[b]:offs[b + 1]]
        assert got.shape == w.shape, (b, got.shape, w.shape)
        assert torch.equal(got, w), b
    return offs


def _mixed(batch, seed):
    """A batch that cycles through every sample shape of interest."""
    rng = np.random.default_rng(seed)
    kinds = [
        lambda k: _sample([int(rng.integers(500, 3000))], k),                            # key frame only
        lambda k: _sample([0], k),                                                         # a sample with no points
        lambda k: _sample([int(rng.integers(500, 3000)), int(rng.integers(500, 3000))], k),
        lambda k: _sample([int(x) for x in rng.integers(200, 1500, 10)], k),
        lambda k: _sample([int(x) for x in rng.integers(0, 700, 16)], k),                 # 16 sweeps, some tiny
        lambda k: _sample([1500, 0, 2000, 0], k),                                          # empty sweeps
        lambda k: _sample([1200, 800, 900], k, close=1.0),                                 # sweeps removed by remove_close
        lambda k: _sample([0, 0, 0], k),
    ]
    return [kinds[b % len(kinds)](seed * 100 + b) for b in range(batch)]


@pytest.mark.parametrize("batch", [1, 4, 64])
def test_rows_equal_per_sample_ingest(batch):
    from det3d.datasets.pipelines.loading import ingest_sweeps_batched
    samples = _mixed(batch, batch)
    if batch == 4:
        samples[2] = _golden_sample()
    points, offsets = ingest_sweeps_batched(samples)
    offs = _check_rows(samples, points, offsets)
    if batch > 1:
        assert any(offs[b + 1] == offs[b] for b in range(batch))                  # an empty sample took part


@pytest.mark.parametrize("n_sweeps", [1, 2, 10, 16])
def test_rows_equal_per_sample_ingest_by_sweep_count(n_sweeps):
    from det3d.datasets.pipelines.loading import ingest_sweeps_batched
    samples = [_sample([2500 + 37 * s for s in range(n_sweeps)], 40 + n_sweeps + b) for b in range(3)]
    points, offsets = ingest_sweeps_batched(samples)
    offs = _check_rows(samples, points, offsets)
    if n_sweeps > 1:
        assert offs[-1] < sum(sum(r.shape[0] for r in s[0]) for s in samples)   # remove_close dropped points


def test_golden_sample_alone_and_from_pinned_tensors():
    from det3d.datasets.pipelines.loading import ingest_sweeps_batched
    raws, tms, lags = _golden_sample()
    pinned = [torch.from_numpy(r).pin_memory() for r in raws]
    for sample in ((raws, tms, lags), (pinned, tms, lags)):
        points, offsets = ingest_sweeps_batched([sample])
        _check_rows([sample], points, offsets)


@pytest.mark.parametrize("poison", [float("nan"), 1e30])
def test_rows_past_the_live_total_are_never_read(poison):
    from det3d.datasets.pipelines.loading import BatchedIngest, check_sweep_samples, stage_raw_sweeps
    samples = _mixed(6, 3)
    stride, sizes = check_sweep_samples(samples)
    total = sum(map(sum, sizes))
    ing = BatchedIngest(len(samples), total + 5000, 96, stride)
    ing.raw.fill_(poison)
    ing.out.fill_(poison)
    ing.table.copy_(torch.from_numpy(ing.host_table(samples, sizes)))
    stage_raw_sweeps(samples, sizes, ing.raw)
    points, offsets = ing.launch()
    offs = _check_rows(samples, points, offsets)
    assert int(ing.status.item()) == 0
    assert bool(torch.isfinite(points[:offs[-1]]).all())


def _capture(ing):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ing.launch()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ing.launch()
    return graph


def test_one_graph_replays_six_tables_of_distinct_sizes():
    from det3d.datasets.pipelines.loading import BatchedIngest, check_sweep_samples, stage_raw_sweeps
    from det3d.datasets.pipelines.loading import ingest_sweeps_batched
    rng = np.random.default_rng(9)
    ing = BatchedIngest(4, 1 << 16, 64, 5)
    graph, totals = None, set()
    for k in range(6):
        samples = [_sample([int(x) for x in rng.integers(0, 1600, int(rng.integers(1, 11)))], 500 + 10 * k + b)
                   for b in range(4)]
        stride, sizes = check_sweep_samples(samples)
        totals.add(sum(map(sum, sizes)))
        want_pts, want_off = ingest_sweeps_batched(samples)
        ing.table.copy_(torch.from_numpy(ing.host_table(samples, sizes)))
        ing.raw.fill_(float("nan"))
        stage_raw_sweeps(samples, sizes, ing.raw)
        graph = graph or _capture(ing)
        graph.replay()
        assert torch.equal(ing.cloud_offsets, want_off), k
        n = int(want_off[-1])
        assert torch.equal(ing.out[:n], want_pts[:n]), k
        _check_rows(samples, ing.out, ing.cloud_offsets)
    assert len(totals) == 6


def _clamped(raw, cap):
    v = np.asarray(raw, np.int64).copy()
    v[0] = 0
    return np.minimum(np.maximum.accumulate(np.maximum(v, 0)), cap).astype(np.int32)


@pytest.mark.parametrize("case", ["offsets decreasing", "offsets past capacity", "offsets negative", "offset 0 not 0",
                                  "samples decreasing", "samples past capacity", "samples negative", "sample 0 not 0"])
def test_malformed_device_tables_are_clamped_and_reported(case):
    from det3d.datasets.pipelines.loading import BatchedIngest, check_sweep_samples, stage_raw_sweeps, sweep_table_views
    samples = [_sample([3000, 2500, 1000], 71), _sample([2000, 1500], 72), _sample([4000], 73)]
    stride, sizes = check_sweep_samples(samples)
    S, cap = 8, 16384
    host = BatchedIngest(3, cap, S, stride).host_table(samples, sizes)
    v = sweep_table_views(host, S, 3)
    off, smp = v["sweep_offsets"], v["sample_sweeps"]         # off = [0 3000 5500 6500 8500 10000 14000 ...], smp = [0 3 5 6]
    if case == "offsets decreasing":
        off[2] = 1000
    elif case == "offsets past capacity":
        off[5] = cap + 4096
    elif case == "offsets negative":
        off[1] = -7
    elif case == "offset 0 not 0":
        off[0] = 500
    elif case == "samples decreasing":
        smp[2] = 1
    elif case == "samples past capacity":
        smp[3] = S + 5
    elif case == "samples negative":
        smp[1] = -2
    elif case == "sample 0 not 0":
        smp[0] = 1
    fixed = host.copy()
    fv = sweep_table_views(fixed, S, 3)
    fv["sweep_offsets"][:] = _clamped(off, cap)
    fv["sample_sweeps"][:] = _clamped(smp, S)
    results = []
    for table in (host, fixed):
        ing = BatchedIngest(3, cap, S, stride)
        ing.raw.fill_(1e30)                    # (a clamp to the capacity reaches these rows: finite, so they compare)
        stage_raw_sweeps(samples, sizes, ing.raw)
        ing.table.copy_(torch.from_numpy(table))
        pts, offs = ing.launch()
        results.append((int(ing.status.item()), offs.clone(), pts[:int(offs[-1])].clone()))
    (st_bad, off_bad, pts_bad), (st_ok, off_ok, pts_ok) = results
    assert st_bad == 1 and st_ok == 0
    assert torch.equal(off_bad, off_ok) and torch.equal(pts_bad, pts_ok)


# ---- end to end -------------------------------------------------------------------------------------------------
def _cbgs_pipeline():
    import bench
    from det3d.torchie import Config
    from det3d_b200.apis import InferencePipeline
    wl = bench.WORKLOADS["cbgs"]
    args = argparse.Namespace(config="cbgs", wl=wl, dist="lidar_like")
    cfg = Config.fromfile(os.path.join(ROOT, "configs", wl["cfg"]))
    return InferencePipeline(cfg, model=bench.build_model(cfg, args), device="cuda")


def _pillars_nusc_pipeline(model_hook=None):
    from det3d_b200.apis import InferencePipeline
    from test_pillars_nusc import _demo_model, shipped_config
    cfg = shipped_config()
    model = _demo_model(cfg)
    if model_hook is not None:
        model_hook(model)
    return InferencePipeline(cfg, model=model, device="cuda")


@pytest.fixture(scope="module", params=["cbgs", "pillars_nusc"])
def pipe(request):
    return _cbgs_pipeline() if request.param == "cbgs" else _pillars_nusc_pipeline()


def _nusc_samples(pipe, batch, seed, per_sweep=3500, pinned=True):
    from det3d_b200.utils.synthetic import lidar_like_sweeps
    rng = np.random.default_rng(seed)
    out = []
    for b in range(batch):
        sizes = rng.integers(int(0.9 * per_sweep), per_sweep + 1, 10)
        raws, tms, lags = lidar_like_sweeps(sizes, pipe.cfg.voxel_generator.range, seed * 100 + b, close_fraction=0.02)
        out.append(([torch.from_numpy(r).pin_memory() for r in raws] if pinned else raws, tms, lags))
    return out


def _host_path(pipe, samples):
    clouds = [c.cpu().pin_memory() for c in _per_sample([([np.asarray(r) for r in s[0]], s[1], s[2]) for s in samples])]
    return pipe.infer_host(clouds).clone()


def _sweep_keys(pipe):
    return sorted(k for k in pipe._graphs if len(k) == 5)


def test_infer_sweeps_equals_per_sample_ingest_then_infer_host(pipe):
    detections = 0
    for k in range(2):
        samples = _nusc_samples(pipe, 2, 60 + k, pinned=k == 0)
        want = _host_path(pipe, samples)
        eager = pipe.infer_sweeps(samples).clone()
        graphed = pipe.infer_sweeps(samples, graphed=True).clone()
        assert torch.equal(eager, want), k
        assert torch.equal(graphed, want), k
        detections += int((want[..., -1] > 0.5).sum())
    assert detections > 0


def test_one_graph_serves_tables_of_distinct_sizes_and_a_larger_total_one_more_bucket(pipe):
    pipe._graphs.clear()
    graph, totals = None, set()
    for k in range(6):
        samples = _nusc_samples(pipe, 2, 80 + k, per_sweep=4000)       # totals in [72000, 80000]: one bucket
        totals.add(sum(r.shape[0] for s in samples for r in s[0]))
        got = pipe.infer_sweeps(samples, graphed=True).clone()
        assert torch.equal(got, pipe.infer_sweeps(samples)), k
        keys = _sweep_keys(pipe)
        assert len(keys) == 1, keys
        entry = pipe._graphs[keys[0]]
        graph = graph or entry.graph
        assert entry.graph is graph                            # captured once, replayed for every table
    assert len(totals) == 6
    (batch, bucket, table_cap, stride, n_feat), = _sweep_keys(pipe)
    assert (batch, table_cap, stride, n_feat) == (2, 32, 5, 4)
    big = _nusc_samples(pipe, 2, 90, per_sweep=bucket // 10)                    # total in (bucket, 2 * bucket)
    got = pipe.infer_sweeps(big, graphed=True).clone()
    assert torch.equal(got, _host_path(pipe, big))
    assert [k[1] for k in _sweep_keys(pipe)] == [bucket, 2 * bucket]


def test_infer_sweeps_batch_of_one_key_frame_only(pipe):
    from det3d_b200.utils.synthetic import lidar_like_sweeps
    samples = [lidar_like_sweeps([30000], pipe.cfg.voxel_generator.range, 5)]
    want = _host_path(pipe, samples)
    assert torch.equal(pipe.infer_sweeps(samples), want)
    assert torch.equal(pipe.infer_sweeps(samples, graphed=True), want)


def _raise_deblock_overflow(model):
    # deblock 0's BatchNorm on channel 7: scale 0, shift 65510 -> outside the f16 range; that channel's head weights
    # zeroed so the detections stay finite
    with torch.no_grad():
        bn = model.neck.deblocks[0][1]
        bn.weight[7] = 0.0
        bn.bias[7] = 65510.0
        for task in model.bbox_head.tasks:
            for conv in (task.conv_box, task.conv_cls):
                conv.weight[:, 7] = 0.0


@pytest.mark.parametrize("graphed", [False, True])
def test_overflow_reruns_infer_sweeps_on_tf32x3(graphed):
    pipe = _pillars_nusc_pipeline(_raise_deblock_overflow)
    assert pipe.model.fused_bev() is not None and pipe.model.math == "fp16x3"
    samples = _nusc_samples(pipe, 1, 301)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        packed = pipe.infer_sweeps(samples, graphed=graphed).clone()
    assert any("f16 range" in str(w.message) for w in caught), [str(w.message) for w in caught]
    assert pipe.model.math == "tf32x3"
    if graphed:
        assert [e.graph is not None for e in pipe._graphs.values()] == [True]  # the re-run's graph only
    assert bool(torch.isfinite(packed).all())
    assert int(pipe.overflow_flag().item()) == 0
    assert int((packed[0, :, -1] > 0.5).sum()) > 0
    assert torch.equal(packed, _host_path(pipe, samples))                      # same bits as the host path on tf32x3
