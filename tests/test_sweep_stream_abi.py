"""The gather form of d3b_ingest_sweeps_dev (a non-null sweep_src) and SweepStream without a GPU: the entry point's
host-side argument checks, push()'s ValueErrors, and the slot bookkeeping, transforms and lags a stream computes on the
host, against numpy."""
import numpy as np
import pytest
import torch

from det3d_b200 import _lib

# stand-ins for device pointers: never dereferenced, every call below is rejected first
_P = 0x1000


def _call(raw=_P, capacity=4096, stride=5, n_feat=4, off=_P, src=_P, samples=_P, tms=_P, lags=_P, flags=_P,
          table_cap=8, batch=2, out=_P, cloud_offsets=_P, ws=_P, ws_bytes=None):
    L = _lib.lib()
    if ws_bytes is None:
        ws_bytes = L.d3b_ingest_dev_workspace_bytes(max(capacity, 0), max(table_cap, 1))
    return L.d3b_ingest_sweeps_dev(raw, capacity, stride, n_feat, off, src, samples, tms, lags, flags, table_cap, batch,
                                   1.0, out, cloud_offsets, None, ws, ws_bytes, None)


def test_gather_null_arguments_are_rejected():
    L = _lib.lib()
    for name in ("off", "samples", "tms", "lags", "flags", "cloud_offsets", "ws"):
        assert _call(**{name: None}) == 1, name
        assert b"null" in L.d3b_last_error() and b"d3b_ingest_sweeps_dev" in L.d3b_last_error(), name
    for name in ("raw", "out"):
        assert _call(**{name: None}) == 1, name
        assert b"null buffer" in L.d3b_last_error(), name


def test_gather_bounds_and_layout_are_checked():
    L = _lib.lib()
    for batch in (0, 65):
        assert _call(batch=batch, ws_bytes=1 << 30) == 1, batch
        assert b"batch" in L.d3b_last_error()
    for table_cap, batch in ((0, 1), (17, 1), (33, 2)):
        assert _call(table_cap=table_cap, batch=batch, ws_bytes=1 << 30) == 1, (table_cap, batch)
        assert b"sweep_capacity" in L.d3b_last_error()
    for capacity in (-1, (1 << 30) + 1):
        assert _call(capacity=capacity, ws_bytes=1 << 40) == 1, capacity
        assert b"raw_capacity" in L.d3b_last_error()
    for stride, n_feat in ((3, 4), (5, 2)):
        assert _call(stride=stride, n_feat=n_feat) == 1
        assert b"layout" in L.d3b_last_error()


def test_gather_workspace():
    L = _lib.lib()
    need = L.d3b_ingest_dev_workspace_bytes(4096, 8)
    assert _call(ws_bytes=need - 1) == 4                              # D3B_ERR_WORKSPACE
    assert b"workspace" in L.d3b_last_error()


def test_gather_table_layout():
    from det3d_b200.datasets.pipelines.loading import sweep_table_bytes, sweep_table_views
    S, B = 40, 4
    assert sweep_table_bytes(S, B, gather=True) == sweep_table_bytes(S, B) + 4 * S
    buf = np.zeros(sweep_table_bytes(S, B, gather=True), np.uint8)
    v = sweep_table_views(buf, S, B, gather=True)
    assert [v[k].shape[0] for k in ("transforms", "sweep_offsets", "sample_sweeps", "sweep_src", "time_lag", "flags")] \
        == [16 * S, S + 1, B + 1, S, S, S]
    plain = sweep_table_views(np.zeros(sweep_table_bytes(S, B), np.uint8), S, B)
    assert "sweep_src" not in plain


# ---- SweepStream on the host --------------------------------------------------------------------------------------
def _stream(batch=2, history=4, slot_capacity=100, raw_stride=5):
    from det3d_b200.apis import InferencePipeline, SweepStream
    pipe = object.__new__(InferencePipeline)
    pipe.num_point_features = 5                       # every check below runs before the pipeline is touched
    return SweepStream(pipe, batch, history, slot_capacity, raw_stride)


@pytest.mark.parametrize("case", ["stream -1", "stream 2", "float64 raw", "1-D raw", "stride 4", "too many points",
                                  "3x4 pose", "flat pose", "timestamp string", "device-less object"])
def test_push_rejects_malformed_arguments(case):
    st = _stream()
    raw, pose, t, b = np.zeros((10, 5), np.float32), np.eye(4), 0.5, 0
    if case == "stream -1":
        b = -1
    elif case == "stream 2":
        b = 2
    elif case == "float64 raw":
        raw = raw.astype(np.float64)
    elif case == "1-D raw":
        raw = raw.reshape(-1)
    elif case == "stride 4":
        raw = np.zeros((10, 4), np.float32)
    elif case == "too many points":
        raw = np.zeros((101, 5), np.float32)
    elif case == "3x4 pose":
        pose = np.eye(4)[:3]
    elif case == "flat pose":
        pose = np.eye(4).reshape(16)
    elif case == "timestamp string":
        t = "0.5"
    elif case == "device-less object":
        raw = [[0.0] * 5] * 10
    with pytest.raises(ValueError):
        st.push(b, raw, pose, t)
    assert st.sweeps.count == [0, 0] and st.pending_h2d_bytes == 0 and st._ingest is None     # nothing enqueued


def test_stream_constructor_checks():
    from det3d_b200.apis import SweepStream
    pipe = _stream().pipe
    for kw in (dict(batch=0), dict(batch=65), dict(history=0), dict(history=17), dict(slot_capacity=0),
               dict(slot_capacity=1 << 30), dict(raw_stride=3), dict(n_feat=3)):
        args = dict(batch=2, history=4, slot_capacity=100, raw_stride=5, n_feat=4)
        args.update(kw)
        with pytest.raises(ValueError):
            SweepStream(pipe, **args)


def test_a_push_of_slot_capacity_points_is_accepted():
    st = _stream()
    assert st.check_push(1, torch.zeros((100, 5)), np.eye(4), 3) == 100


def _pose(rng):
    a = rng.uniform(-np.pi, np.pi)
    p = np.eye(4)
    p[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    p[:3, 3] = rng.uniform(-500, 500, 3)
    return p


def test_slot_bookkeeping_wraps_and_resets():
    from det3d_b200.datasets.pipelines.loading import SweepHistory
    K = 4
    h = SweepHistory(2, K)
    rng = np.random.default_rng(0)
    slots = {0: [], 1: []}
    for step in range(11):
        for b in range(2):
            if b == 1 and step == 6:
                h.reset(1)
                slots[1] = []
            slots[b].append(h.record(b, 10 * step + b, _pose(rng), 0.05 * step))
    assert slots[0] == [k % K for k in range(11)]
    assert slots[1] == [k % K for k in range(5)]                        # restarted at slot 0 after the reset
    frame = h.frame()
    ks0, ns0, _, _ = frame[0]
    assert ks0 == [2, 1, 0, 3] and ns0 == [100, 90, 80, 70]             # newest first, the K most recent
    ks1, ns1, _, _ = frame[1]
    assert ks1 == [0, 3, 2, 1] and ns1 == [101, 91, 81, 71]
    h.reset(0)
    with pytest.raises(ValueError, match="stream 0 has no sweep"):
        h.frame()
    h.record(0, 7, np.eye(4), 1.0)
    ks, ns, tms, lags = h.frame()[0]
    assert (ks, ns, tms, lags) == ([0], [7], [None], [0.0])             # a filling stream uses what it has


def test_transforms_and_lags_against_numpy():
    from det3d_b200.datasets.pipelines.loading import SweepHistory, fill_sweep_table, sweep_table_bytes, sweep_table_views
    rng = np.random.default_rng(3)
    K = 5
    h = SweepHistory(1, K)
    poses, times = [], []
    for step in range(8):
        poses.append(_pose(rng))
        times.append(1.7e9 + 0.05 * step + rng.uniform(0, 1e-3))
        h.record(0, 10, poses[-1], times[-1])
    ks, ns, tms, lags = h.frame()[0]
    key = np.linalg.inv(poses[-1])
    assert tms[0] is None and lags[0] == 0.0
    for j in range(1, K):
        want = key @ poses[-1 - j]
        assert tms[j].dtype == np.float64 and np.array_equal(tms[j], want), j
        assert lags[j] == times[-1] - times[-1 - j], j
    # the table rounds the lags to float32 once and flags every sweep but the key frame (transform + remove_close)
    S = 8
    buf = np.zeros(sweep_table_bytes(S, 1, gather=True), np.uint8)
    v = sweep_table_views(buf, S, 1, gather=True)
    fill_sweep_table(v, [(None, tms, lags)], [ns])
    assert np.array_equal(v["time_lag"][:K], np.asarray(lags, np.float64).astype(np.float32))
    assert v["flags"][:K].tolist() == [0, 3, 3, 3, 3]
    assert np.array_equal(v["transforms"][16:32], tms[1].reshape(16))
    assert v["sweep_offsets"][:K + 1].tolist() == [0, 10, 20, 30, 40, 50]
