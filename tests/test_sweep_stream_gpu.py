"""Device-resident sweep histories (d3b_ingest_sweeps_dev with a sweep_src table, SweepStream): the gather ingest over
sweeps scattered through a slot buffer gives the bits the ingest without sweep_src gives over the same sweeps packed
back to back, malformed sweep starts are clamped and reported, and every frame of a stream -- eager and graphed -- is
bit-identical to infer_sweeps(stream.samples()), for the CBGS and nuScenes PointPillars configs, with one captured graph
per sequence."""
import warnings

import numpy as np
import pytest
import torch

from test_ingest_batched_gpu import (_cbgs_pipeline, _golden_sample, _mixed, _pillars_nusc_pipeline,
                                     _raise_deblock_overflow, _sample)

pytestmark = pytest.mark.gpu


# ---- kernel ------------------------------------------------------------------------------------------------------
def _dev_ingest(samples, S):
    from det3d_b200.datasets.pipelines.loading import BatchedIngest, check_sweep_samples, stage_raw_sweeps
    stride, sizes = check_sweep_samples(samples)
    ing = BatchedIngest(len(samples), max(sum(map(sum, sizes)), 1), S, stride)
    ing.table.copy_(torch.from_numpy(ing.host_table(samples, sizes)))
    stage_raw_sweeps(samples, sizes, ing.raw)
    pts, offs = ing.launch()
    n = int(offs[-1])
    return pts[:n].clone(), offs.clone(), int(ing.status.item())


def _scattered(samples, S, seed, poison):
    """A gather ingest whose raw buffer holds every sweep at the start of its own slot, the slots in random order and
    one spare slot per sample; every row no sweep covers is `poison`.  Returns (ingest, sizes, sweep_src)."""
    from det3d_b200.datasets.pipelines.loading import BatchedIngest, check_sweep_samples
    stride, sizes = check_sweep_samples(samples)
    n_sweeps = sum(map(len, sizes))
    slot = max(max(max(n) for n in sizes), 1) + 37
    n_slots = n_sweeps + len(samples)
    order = np.random.default_rng(seed).permutation(n_slots)[:n_sweeps]
    ing = BatchedIngest(len(samples), n_slots * slot, S, stride, gather=True)
    ing.raw.fill_(poison)
    src, s = [], 0
    for raws, _tms, _lags in samples:
        for r in raws:
            at = int(order[s]) * slot
            if r.shape[0]:
                ing.raw[at:at + r.shape[0]].copy_(torch.as_tensor(r))
            src.append(at)
            s += 1
    return ing, sizes, src


def _gather(ing, samples, sizes, src):
    ing.table.copy_(torch.from_numpy(ing.host_table(samples, sizes, sweep_src=src)))
    pts, offs = ing.launch()
    n = int(offs[-1])
    return pts[:n].clone(), offs.clone(), int(ing.status.item())


def _table_cap(samples):
    from det3d_b200.datasets.pipelines.loading import sweep_table_capacity
    return sweep_table_capacity(sum(len(s[0]) for s in samples), len(samples))


@pytest.mark.parametrize("poison", [float("nan"), 1e30])
@pytest.mark.parametrize("batch", [1, 4, 64])
def test_gather_equals_dev_on_scattered_slots(batch, poison):
    samples = _mixed(batch, 7 + batch)
    if batch == 4:
        samples[1] = _golden_sample()
    S = _table_cap(samples)
    want_pts, want_off, st = _dev_ingest(samples, S)
    assert st == 0
    ing, sizes, src = _scattered(samples, S, batch, poison)
    got_pts, got_off, st = _gather(ing, samples, sizes, src)
    assert st == 0
    assert torch.equal(got_off, want_off)
    assert torch.equal(got_pts, want_pts)
    assert bool(torch.isfinite(got_pts).all())
    assert len(src) == 1 or src != sorted(src)                         # the slots really were out of order


@pytest.mark.parametrize("n_sweeps", [1, 2, 10, 16])
def test_gather_equals_dev_by_sweep_count(n_sweeps):
    sizes = [1500 + 211 * s for s in range(n_sweeps)]
    samples = [_sample(sizes, 900 + n_sweeps + b, close=0.05 if b else 1.0) for b in range(3)]   # sample 0: filtered out
    samples.append(_sample([0] * n_sweeps, 950))                                                   # empty sweeps only
    S = _table_cap(samples)
    want = _dev_ingest(samples, S)
    ing, sizes, src = _scattered(samples, S, n_sweeps, float("nan"))
    got = _gather(ing, samples, sizes, src)
    assert got[2] == 0 and torch.equal(got[1], want[1]) and torch.equal(got[0], want[0])


def test_golden_sample_gathered():
    samples = [_golden_sample()]
    S = _table_cap(samples)
    want = _dev_ingest(samples, S)
    ing, sizes, src = _scattered(samples, S, 5, 1e30)
    got = _gather(ing, samples, sizes, src)
    assert torch.equal(got[1], want[1]) and torch.equal(got[0], want[0])


def test_sweep_src_at_the_offsets_is_the_dev_ingest():
    """A null sweep_src and sweep_src[s] = sweep_offsets[s] give the same bits."""
    from det3d_b200.datasets.pipelines.loading import BatchedIngest, check_sweep_samples, stage_raw_sweeps
    samples = _mixed(6, 21)
    S = _table_cap(samples)
    stride, sizes = check_sweep_samples(samples)
    total = sum(map(sum, sizes))
    results = []
    for gather in (False, True):
        ing = BatchedIngest(len(samples), total + 3000, S, stride, gather=gather)
        ing.raw.fill_(float("nan"))
        stage_raw_sweeps(samples, sizes, ing.raw)
        src = np.cumsum([0] + [n for ns in sizes for n in ns])[:-1] if gather else None
        ing.table.copy_(torch.from_numpy(ing.host_table(samples, sizes, sweep_src=src)))
        pts, offs = ing.launch()
        results.append((int(ing.status.item()), offs.clone(), pts[:int(offs[-1])].clone()))
    (st_dev, off_dev, pts_dev), (st_g, off_g, pts_g) = results
    assert st_dev == 0 and st_g == 0
    assert torch.equal(off_dev, off_g) and torch.equal(pts_dev, pts_g)


@pytest.mark.parametrize("case", ["negative", "past the end", "far past the end", "and offsets past capacity"])
def test_malformed_sweep_src_is_clamped_and_reported(case):
    samples = [_sample([3000, 2500, 1000], 71), _sample([2000, 1500], 72), _sample([4000], 73)]
    S = 8
    ing, sizes, src = _scattered(samples, S, 3, 1e30)        # (a clamp may reach poisoned rows: finite, so they compare)
    cap = ing.raw_capacity
    lens = [n for ns in sizes for n in ns]
    bad = list(src)
    if case == "negative":
        bad[1] = -5
    elif case == "past the end":
        bad[2] = cap - lens[2] + 1
    elif case == "far past the end":
        bad[3] = cap + 100000
    fixed = [min(max(r, 0), cap - n) for r, n in zip(bad, lens)]
    assert fixed != bad or case == "and offsets past capacity"
    host = ing.host_table(samples, sizes, sweep_src=bad)
    if case == "and offsets past capacity":
        from det3d_b200.datasets.pipelines.loading import sweep_table_views
        v = sweep_table_views(host, S, 3, gather=True)
        v["sweep_offsets"][4] = cap + 50                         # the prefix is clamped first, then sweep_src to its lengths
        v["sweep_src"][3] = -1
    ing.table.copy_(torch.from_numpy(host))
    pts, offs = ing.launch()
    got = (int(ing.status.item()), offs.clone(), pts[:int(offs[-1])].clone())
    if case == "and offsets past capacity":
        assert got[0] == 3                                       # both bits: the offsets and a start were clamped
        return
    assert got[0] == 2
    want = _gather(ing, samples, sizes, fixed)
    assert want[2] == 0
    assert torch.equal(got[1], want[1]) and torch.equal(got[2], want[0])


# ---- stream ------------------------------------------------------------------------------------------------------
SLOT = 5000


@pytest.fixture(scope="module", params=["cbgs", "pillars_nusc"])
def pipe(request):
    return _cbgs_pipeline() if request.param == "cbgs" else _pillars_nusc_pipeline()


def _motion(rng, yaw=0.05, shift=1.5):
    a = rng.uniform(-yaw, yaw)
    m = np.eye(4)
    m[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    m[:3, 3] = rng.uniform(-shift, shift, 3) * [1, 1, 0.05]
    return m


def _sweep(rng, n, pcr, seed, kind):
    from det3d_b200.utils.synthetic import lidar_like_cloud
    p = lidar_like_cloud(int(n), pcr, 5, seed) if n else np.zeros((0, 5), np.float32)
    k = int(0.03 * p.shape[0])
    p[:k, :2] = rng.uniform(-0.99, 0.99, (k, 2)).astype(np.float32)          # inside the remove_close box
    if kind == 0:
        return torch.from_numpy(p).pin_memory()
    return p if kind == 1 else torch.from_numpy(p)                          # numpy, or a pageable tensor


def _sequence(pipe, batch, seed, resets, frames=24, K=10):
    """Runs `frames` frames of a K-slot stream of `batch` streams (one push per stream and frame, sizes redrawn every
    frame, resets = {frame: [streams]}) and checks every frame against infer_sweeps(samples())."""
    from det3d_b200.apis import SweepStream
    rng = np.random.default_rng(seed)
    pcr = pipe.cfg.voxel_generator.range
    for k in [k for k in pipe._graphs if k[0] == "stream"]:                  # (the fixture's pipeline is shared)
        del pipe._graphs[k]
    st = SweepStream(pipe, batch, K, SLOT)
    poses = [np.eye(4) for _ in range(batch)]
    times = [1.6e9 + 10 * b for b in range(batch)]
    graph, dets, filling, wrapped = None, 0, 0, False
    for f in range(frames):
        pushed = 0
        for b in resets.get(f, []):
            st.reset(b)
        for b in range(batch):
            n = 0 if (f, b) == (4, batch - 1) else int(rng.integers(1200, SLOT + 1))      # one empty key frame
            poses[b] = poses[b] @ _motion(rng)
            times[b] += 0.05 + rng.uniform(-1e-3, 1e-3)
            st.push(b, _sweep(rng, n, pcr, seed * 1000 + f * 64 + b, (f + b) % 3), poses[b], times[b])
            pushed += n * 5 * 4
        filling += sum(len(h) < K for h in st.sweeps.held)
        wrapped |= any(c > K for c in st.sweeps.count)
        eager = st.infer().clone()
        assert st.last_h2d_bytes == pushed + st._ingest.table.numel(), f
        graphed = st.infer(graphed=True).clone()
        assert st.last_h2d_bytes == st._ingest.table.numel(), f                  # the sweeps went once, with push
        samples = st.samples()
        assert [len(s[0]) for s in samples] == [len(h) for h in st.sweeps.held]
        want = pipe.infer_sweeps(samples).clone()
        assert torch.equal(eager, want), f
        assert torch.equal(graphed, want), f
        keys = [k for k in pipe._graphs if k[0] == "stream"]
        assert keys == [st.key], keys
        graph = graph or pipe._graphs[st.key].graph
        assert pipe._graphs[st.key].graph is graph, f                           # captured once for the sequence
        dets += int((want[..., -1] > 0.5).sum())
    assert dets > 0 and filling > 0 and wrapped
    return st


def test_stream_b1_equals_infer_sweeps_every_frame(pipe):
    st = _sequence(pipe, 1, 11, resets={15: [0]})
    assert st.sweeps.count == [9]


def test_stream_b4_equals_infer_sweeps_every_frame(pipe):
    st = _sequence(pipe, 4, 12, resets={5: [3], 13: [1]})
    assert st.sweeps.count == [24, 11, 24, 19]                                  # two wrapped, one reset mid-way


def test_stream_sample_layout_and_sweep_order(pipe):
    """samples() lists each stream's key frame first, then its earlier sweeps newest first."""
    from det3d_b200.apis import SweepStream
    st = SweepStream(pipe, 2, 3, 64)
    pushed = {0: [], 1: []}
    for f in range(5):
        for b in range(2):
            r = np.full((8 + f, 5), 10 * f + b, np.float32)
            st.push(b, r, np.eye(4), 0.1 * f)
            pushed[b].append(r)
    for b, (raws, tms, lags) in enumerate(st.samples()):
        assert [float(r[0, 0]) for r in raws] == [10 * f + b for f in (4, 3, 2)]
        assert all(np.array_equal(r, p) for r, p in zip(raws, pushed[b][::-1]))
        assert tms[0] is None and all(np.array_equal(t, np.eye(4)) for t in tms[1:])
        assert np.allclose(lags, [0.0, 0.1, 0.2])


@pytest.mark.parametrize("graphed", [False, True])
def test_overflow_rerun_matches_infer_sweeps_after_its_fallback(graphed):
    from det3d_b200.apis import SweepStream
    pipe = _pillars_nusc_pipeline(_raise_deblock_overflow)
    oracle = _pillars_nusc_pipeline(_raise_deblock_overflow)
    rng = np.random.default_rng(5)
    st = SweepStream(pipe, 1, 10, SLOT)
    pose, t = np.eye(4), 0.0
    for f in range(4):
        pose, t = pose @ _motion(rng), t + 0.05
        st.push(0, _sweep(rng, 4500, pipe.cfg.voxel_generator.range, 300 + f, f % 2), pose, t)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        got = st.infer(graphed=graphed).clone()
        want = oracle.infer_sweeps(st.samples(), graphed=graphed).clone()
    assert sum("f16 range" in str(w.message) for w in caught) == 2, [str(w.message) for w in caught]
    assert pipe.model.math == "tf32x3" and oracle.model.math == "tf32x3"
    assert st.sweeps.count == [4]                                               # the re-run reused the frame
    assert bool(torch.isfinite(got).all()) and int((got[0, :, -1] > 0.5).sum()) > 0
    assert torch.equal(got, want)
    assert torch.equal(st.infer(graphed=graphed), want)                         # no further fallback, same frame
    if graphed:
        assert [k for k in pipe._graphs] == [st.key]
