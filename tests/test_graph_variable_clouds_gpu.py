"""One CUDA graph per (batch, point-capacity bucket) serves clouds of any size: forward_graphed and
infer_host(graphed=True) return the bits of the eager forward on exactly sized points, for SECOND (B = 1), PointPillars
(B = 8, the reader that walks the voxelizer's point lists) and CBGS (B = 2)."""
import argparse
import os
import warnings

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

BATCH = {"second": 1, "pillars": 8, "cbgs": 2}


@pytest.fixture(scope="module", params=sorted(BATCH))
def setup(request):
    import bench
    from det3d.torchie import Config
    from det3d_b200.apis import InferencePipeline

    name = request.param
    args = argparse.Namespace(config=name, wl=bench.WORKLOADS[name], dist="lidar_like")
    cfg = Config.fromfile(os.path.join(ROOT, "configs", args.wl["cfg"]))
    pipe = InferencePipeline(cfg, model=bench.build_model(cfg, args), device="cuda")
    return name, cfg, pipe, args.wl["n_points"], args.wl["ndim"]


def _clouds(cfg, sizes, ndim, seed):
    from det3d_b200.utils.synthetic import lidar_like_cloud
    return [lidar_like_cloud(int(n), cfg.voxel_generator.range, ndim, seed + i) for i, n in enumerate(sizes)]


def _batches(pipe, n_points, batch, count, seed):
    """`count` batches of distinct per-cloud sizes whose totals all fall in the bucket of a full batch."""
    bucket = pipe.bucket_of(batch * n_points)
    lo = (bucket // 2) // batch + 1
    rng = np.random.default_rng(seed)
    sizes = rng.choice(np.arange(lo, n_points + 1), size=(count, batch), replace=False)
    return [s.tolist() for s in sizes], bucket


def _eager(pipe, clouds):
    offsets = np.cumsum([0] + [c.shape[0] for c in clouds]).tolist()
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    return pipe.pack(pipe.forward_device(pts, offsets)).clone(), pts, offsets


def test_one_graph_replays_batches_of_distinct_sizes(setup):
    name, cfg, pipe, n_points, ndim = setup
    batch = BATCH[name]
    pipe._graphs.clear()
    sizes, bucket = _batches(pipe, n_points, batch, 6, 11)
    graph = None
    detections = 0
    for k, s in enumerate(sizes):
        clouds = _clouds(cfg, s, ndim, 1000 + 10 * k)
        want, pts, offsets = _eager(pipe, clouds)
        got = pipe.forward_graphed(pts, offsets).clone()
        assert torch.equal(got, want), (name, s)
        assert list(pipe._graphs) == [(batch, bucket, ndim)]
        entry = pipe._graphs[(batch, bucket, ndim)]
        graph = graph or entry.graph
        assert entry.graph is graph                      # captured once, replayed for every size
        detections += int((got[..., -1] > 0.5).sum())
    assert detections > 0


def test_a_larger_batch_takes_another_bucket_with_the_same_bits(setup):
    name, cfg, pipe, n_points, ndim = setup
    batch = BATCH[name]
    pipe._graphs.clear()
    sizes, bucket = _batches(pipe, n_points, batch, 1, 12)
    want, pts, offsets = _eager(pipe, _clouds(cfg, sizes[0], ndim, 2000))
    assert torch.equal(pipe.forward_graphed(pts, offsets), want)
    big = [n_points + bucket // batch] * batch                   # total past the bucket: one more graph
    want_big, pts_big, off_big = _eager(pipe, _clouds(cfg, big, ndim, 2100))
    assert torch.equal(pipe.forward_graphed(pts_big, off_big), want_big)
    assert sorted(pipe._graphs) == [(batch, bucket, ndim), (batch, 2 * bucket, ndim)]
    # the first batch again, through its own bucket and through the larger one
    assert torch.equal(pipe.forward_graphed(pts, offsets), want)
    entry = pipe._graph_entry(batch, 2 * bucket, ndim)
    entry.points[:offsets[-1]].copy_(pts)
    assert torch.equal(pipe._replay(entry, offsets), want)
    assert len(pipe._graphs) == 2


def test_infer_host_graphed_equals_eager(setup):
    name, cfg, pipe, n_points, ndim = setup
    batch = BATCH[name]
    sizes, _bucket = _batches(pipe, n_points, batch, 3, 13)
    for k, s in enumerate(sizes):
        clouds = [torch.from_numpy(c).pin_memory() for c in _clouds(cfg, s, ndim, 3000 + 10 * k)]
        eager = pipe.infer_host(clouds).clone()
        graphed = pipe.infer_host(clouds, graphed=True).clone()
        assert torch.equal(eager, graphed), (name, s)


def test_malformed_offsets_raise_before_any_launch(setup):
    from det3d_b200 import _lib

    name, cfg, pipe, n_points, ndim = setup
    pts = torch.zeros((3000, ndim), device="cuda")
    torch.cuda.synchronize()
    launches = _lib.launch_count()
    for bad in ([0, 2000, 1000, 3000], [1, 1000, 3000], [0, 1000, 2000], [0], [], list(range(0, 3000, 45)) + [3000]):
        with pytest.raises(ValueError):
            pipe.forward_graphed(pts, bad)
    with pytest.raises(ValueError):
        pipe.infer_host([torch.zeros((10, ndim))] * 65, graphed=True)
    assert _lib.launch_count() == launches


def test_overflow_reruns_graphed_on_tf32x3():
    """nuScenes PointPillars with deblock 0's BatchNorm on channel 7 set to scale 0, shift 65510 (that channel's head
    weights zeroed, so the detections stay finite): infer_host(graphed=True) warns, switches to tf32x3, drops its graphs,
    re-runs, and returns finite detections with the flag clear."""
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import lidar_like_cloud
    from test_pillars_nusc import N_POINTS, _demo_model, shipped_config

    cfg = shipped_config()
    model = _demo_model(cfg)
    with torch.no_grad():
        bn = model.neck.deblocks[0][1]
        bn.weight[7] = 0.0
        bn.bias[7] = 65510.0
        for task in model.bbox_head.tasks:
            for conv in (task.conv_box, task.conv_cls):
                conv.weight[:, 7] = 0.0
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    assert pipe.model.fused_bev() is not None and pipe.model.math == "fp16x3"
    cloud = torch.from_numpy(lidar_like_cloud(N_POINTS, cfg.voxel_generator.range, 5, 301)).pin_memory()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        packed = pipe.infer_host([cloud], graphed=True).clone()
    assert any("f16 range" in str(w.message) for w in caught), [str(w.message) for w in caught]
    assert pipe.model.math == "tf32x3"
    assert [e.graph is not None for e in pipe._graphs.values()] == [True]      # the re-run's graph only
    assert bool(torch.isfinite(packed).all())
    assert int(pipe.overflow_flag().item()) == 0
    assert int((packed[0, :, -1] > 0.5).sum()) > 0
