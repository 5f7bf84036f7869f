"""Host side of the pipelined serving path, on the CPU: SweepHistory's slot accounting for frames left in flight, and
the whole-array to_annos / to_nusc_annos against frozen copies of their per-row forms on the committed goldens (same
keys in the same order, same Python types and dtypes, same float bits)."""
import os
import re

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def load(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


# ---- frozen per-row formatting (the forms the whole-array ones replaced) ------------------------------------------
def to_annos_per_row(results, counts, class_names):
    from det3d_b200.ops.point_cloud.kitti_results import empty_result_anno
    class_names = list(class_names)
    annos = []
    for rows, n in zip(np.asarray(results), np.asarray(counts)):
        n = int(n)
        if n == 0:
            annos.append(empty_result_anno())
            continue
        r = rows[:n]
        annos.append(dict(name=np.array([class_names[int(k)] for k in r[:, 13]]), truncated=np.zeros(n),
                          occluded=np.zeros(n, np.int64), alpha=r[:, 4].copy(), bbox=r[:, 0:4].copy(),
                          dimensions=r[:, 5:8].copy(), location=r[:, 8:11].copy(), rotation_y=r[:, 11].copy(),
                          score=r[:, 12].astype(np.float32)))
    return annos


def to_nusc_annos_per_row(results, counts, class_names, tokens, table):
    from det3d_b200.ops.point_cloud.nusc_results import META
    class_names = list(class_names)
    out = {}
    for token, rows, n in zip(tokens, np.asarray(results), np.asarray(counts)):
        r = rows[:int(n)]
        if np.isnan(r[:, 0:6]).any():
            raise ValueError("sample %r: a detection with a NaN centre or size" % (token,))
        annos = []
        for row in r.tolist():
            label = int(row[13])
            annos.append({"sample_token": token, "translation": row[0:3], "size": row[3:6], "rotation": row[6:10],
                          "velocity": row[10:12], "detection_name": class_names[label], "detection_score": row[12],
                          "attribute_name": table[label][row[14] > 0.5]})
        out[token] = annos
    return {"results": out, "meta": dict(META)}


def assert_same(a, b, where="."):
    """Equal values of the same types; dicts in the same key order; floats and arrays bit for bit."""
    assert type(a) is type(b), (where, type(a), type(b))
    if isinstance(a, dict):
        assert list(a) == list(b), where
        for k in a:
            assert_same(a[k], b[k], "%s/%s" % (where, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, "%s[%d]" % (where, i))
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), (where, a.dtype, b.dtype)
        assert not a.flags.writeable or not np.shares_memory(a, b), where
    elif isinstance(a, float):
        assert np.float64(a).tobytes() == np.float64(b).tobytes(), (where, a, b)
    else:
        assert a == b, (where, a, b)


def _scatter(rows, counts, D, width):
    results = np.zeros((len(counts), D, width))
    off = np.concatenate([[0], np.cumsum(counts)])
    for b, n in enumerate(counts):
        results[b, :n] = rows[off[b]:off[b + 1]]
    return results


# ---- KITTI ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["kitti_results_cases", "kitti_results_exact", "kitti_results_nd9"])
def test_to_annos_equals_the_per_row_form(case):
    from det3d_b200.ops.point_cloud.kitti_results import COLS, to_annos
    g = load(case)
    counts = g["counts"].astype(np.int32)
    names = [str(n) for n in g["class_names"]]
    results = _scatter(g["rows"], counts, g["packed"].shape[1], COLS)
    want = to_annos_per_row(results, counts, names)
    got = to_annos(results, counts, names)
    assert_same(got, want)
    for a in got:                                       # the arrays are copies, not views of the host rows
        assert not any(np.shares_memory(v, results) for v in a.values())


def test_to_annos_name_dtype_follows_the_kept_names():
    from det3d_b200.ops.point_cloud.kitti_results import COLS, to_annos
    names = ["Car", "Pedestrian", "Cyclist"]
    results = np.zeros((3, 4, COLS))
    results[0, :2, 13] = 0                              # only "Car": the reference's array is <U3
    results[1, :3, 13] = [2, 0, 1]
    results[2, :1, 13] = 2
    counts = np.array([2, 3, 0], np.int32)
    got = to_annos(results, counts, names)
    assert_same(got, to_annos_per_row(results, counts, names))
    assert got[0]["name"].dtype == np.dtype("<U3")


# ---- nuScenes ------------------------------------------------------------------------------------------------------
def _nusc_results(g, seed):
    """The golden's boxes as result rows [B, D, 15], the moving column drawn at random (with NaNs and values at 0.5)."""
    n = g["score"].shape[0]
    moving = np.random.default_rng(seed).choice([0.0, 1.0, 0.5, np.nan, 0.75], n)
    rows = np.concatenate([g["translation"], g["size"], g["rotation"], g["velocity"], g["score"][:, None],
                           g["label"][:, None].astype(np.float64), moving[:, None]], 1)
    return _scatter(rows, g["counts"].astype(np.int32), g["packed"].shape[1], 15)


@pytest.mark.parametrize("case", ["nusc_results_cases", "nusc_results_exact"])
def test_to_nusc_annos_equals_the_per_row_form(case):
    from det3d_b200.ops.point_cloud.nusc_results import attribute_table, to_nusc_annos
    g = load(case)
    names, tokens = [str(n) for n in g["class_names"]], [str(t) for t in g["tokens"]]
    table = attribute_table(names)
    results = _nusc_results(g, 7)
    counts = g["counts"].astype(np.int32)
    want = to_nusc_annos_per_row(results, counts, names, tokens, table)
    assert_same(to_nusc_annos(results, counts, names, tokens, table), want)
    assert_same(to_nusc_annos(results, counts, names, tokens), want)
    # the returned str objects are the class names and attributes themselves, as the per-row form's
    got = to_nusc_annos(results, counts, names, tokens, table)
    boxes = [a for t in tokens for a in got["results"][t]]
    assert boxes and all(any(a["detection_name"] is n for n in names) for a in boxes)


def test_to_nusc_annos_nan_check_is_per_sample():
    from det3d_b200.ops.point_cloud.nusc_results import attribute_table, to_nusc_annos
    names = ["car", "pedestrian"]
    results = np.zeros((2, 3, 15))
    results[0, :, 13] = [1, 0, 1]
    results[1, 2, 0] = np.nan                           # past sample 1's count first, then inside it
    for counts in ([3, 2], [3, 3]):
        counts = np.array(counts, np.int32)
        try:
            want = to_nusc_annos_per_row(results, counts, names, ["a", "b"], attribute_table(names))
        except ValueError as e:
            with pytest.raises(ValueError, match=re.escape(str(e))):
                to_nusc_annos(results, counts, names, ["a", "b"])
        else:
            assert_same(to_nusc_annos(results, counts, names, ["a", "b"]), want)


# ---- SweepHistory slot accounting ----------------------------------------------------------------------------------
def _push(h, b, rows=10):
    h.check_free(b)
    return h.record(b, rows, np.eye(4), float(h.count[b]))


def test_default_history_refuses_to_overwrite_an_unfinished_frames_slot():
    from det3d_b200.datasets.pipelines.loading import SweepHistory
    K = 3
    h = SweepHistory(1, K)
    assert h.slots == K
    for _ in range(K):
        _push(h, 0)
    held = h.acquire(h.frame())
    assert sorted(held) == [(0, 0), (0, 1), (0, 2)]
    with pytest.raises(ValueError, match="slot 0"):
        h.check_free(0)                                 # every slot is read by the unfinished frame
    h.release(held)
    assert _push(h, 0) == 0                             # free again once the frame has finished


@pytest.mark.parametrize("k", [2, 3, 4])
def test_in_flight_slots_let_k_frames_run(k):
    """With K + k - 1 slots a stream can be pushed and submitted with k frames in flight, one push per frame, forever;
    with k frames unfinished a push is refused."""
    from det3d_b200.datasets.pipelines.loading import SweepHistory
    K = 4
    h = SweepHistory(2, K, K + k - 1)
    pending = []
    for f in range(5 * (K + k)):
        while len(pending) > k - 1:                     # collect the oldest before pushing
            h.release(pending.pop(0))
        for b in range(2):
            _push(h, b)
        frame = h.frame()
        assert all(len(set(ks)) == len(ks) == min(f + 1, K) for ks, _n, _t, _l in frame)
        pending.append(h.acquire(frame))
        if len(pending) == k and f + 1 >= K + k - 1:            # every slot is read by one of the k
            with pytest.raises(ValueError, match="unfinished"):
                h.check_free(0)
    for held in pending:
        h.release(held)
    assert all(c == 0 for r in h.readers for c in r)


def test_reset_respects_held_slots_and_streams_are_independent():
    from det3d_b200.datasets.pipelines.loading import SweepHistory
    h = SweepHistory(2, 2, 3)
    for b in range(2):
        _push(h, b)
        _push(h, b)
    held = h.acquire(h.frame())                          # slots 0 and 1 of both streams
    h.reset(1)
    with pytest.raises(ValueError, match="stream 1"):
        h.check_free(1)                                  # a reset stream restarts at slot 0, still held
    assert _push(h, 0) == 2                              # stream 0's slot 2 is free
    with pytest.raises(ValueError, match="stream 0"):
        h.check_free(0)
    h.release(held)
    assert _push(h, 1) == 0 and _push(h, 0) == 0


def test_fewer_slots_than_the_history_are_refused():
    from det3d_b200.datasets.pipelines.loading import SweepHistory
    with pytest.raises(ValueError, match="cannot hold"):
        SweepHistory(1, 4, 3)
