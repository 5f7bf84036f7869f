"""KITTI result rows on the CPU: the checker (oracle/kitti_results.py) against the goldens the reference's own functions
produced (tests/golden/make_golden_kitti_results.py), the exact golden bit for bit, the host side of the device path
(calibration table, anno formatting, the per-calibration cache) and the argument checks of d3b_kitti_results_dev, which
return before any CUDA call.  The device kernel is checked against the same goldens in test_kitti_results_gpu.py."""
import collections
import os

import numpy as np
import pytest

from oracle import kitti_results as okr

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CASES = ("kitti_results_cases", "kitti_results_nd9", "kitti_results_exact")
EXACT_COLS = [5, 6, 7, 11, 12, 13]            # dimensions, rotation_y, score, label: copies of float32 values


def load(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def frames(g):
    """Per frame: (packed rows [D, nd + 3], table, the reference's kept rows [n, 14], the recorded margins [D])."""
    off = np.concatenate([[0], np.cumsum(g["counts"])])
    for b in range(g["packed"].shape[0]):
        yield g["packed"][b], g["tables"][b], g["rows"][off[b]:off[b + 1]], g["margin"][b]


def kept_by_oracle(packed, nd, table):
    rows, keep, _aux = okr.kernel_order(packed, nd, table)
    bound, _margin = okr.error_bound(packed, nd, table)
    return rows[keep], bound[keep], keep


def assert_within(got, want, bound, what):
    with np.errstate(invalid="ignore"):
        ok = (got == want) | (np.isnan(got) & np.isnan(want)) | (np.abs(got - want) <= bound)
    assert ok.all(), "%s: %d values outside the bound, worst %s" % (
        what, int((~ok).sum()), np.max(np.where(ok, 0, np.abs(got - want) / np.maximum(bound, 1e-300))))


def test_goldens_hold_the_cases():
    g = load("kitti_results_cases")
    counts, valid = g["counts"], (g["packed"][..., 9] > 0.5).sum(1)
    assert counts[5] == 0 and valid[5] == 0                   # no valid detection
    assert counts[6] == 0 and valid[6] > 0                    # every detection filtered
    assert valid[7] == g["packed"].shape[1]                   # D full
    assert np.isnan(g["packed"][4, :21, :7]).any() and np.isinf(g["packed"][4, :21, :7]).any()
    assert np.all(g["margin"] > 1), "every golden decision is farther from the image bound than the error bound"


@pytest.mark.parametrize("case", CASES)
def test_oracle_equals_the_reference_within_the_bound(case):
    g = load(case)
    nd = int(g["nd"])
    for b, (packed, table, want, margin) in enumerate(frames(g)):
        got, bound, keep = kept_by_oracle(packed, nd, table)
        if case != "kitti_results_exact":       # (its boxes sit on the bounds on purpose; its values are exact)
            assert np.all(margin[packed[:, nd + 2] > 0.5] > 1)
        assert got.shape == want.shape, (case, b, got.shape, want.shape)     # same kept set, same order
        assert np.array_equal(got[:, EXACT_COLS].view(np.uint64), want[:, EXACT_COLS].view(np.uint64)), (case, b)
        assert_within(got[:, :4], want[:, :4], bound[:, :4], "%s frame %d bbox" % (case, b))
        assert_within(got[:, 4], want[:, 4], bound[:, 4], "%s frame %d alpha" % (case, b))
        assert_within(got[:, 8:11], want[:, 8:11], bound[:, 8:11], "%s frame %d location" % (case, b))


def test_exact_golden_bit_for_bit():
    g = load("kitti_results_exact")
    for b, (packed, table, want, _margin) in enumerate(frames(g)):
        got, bound, _keep = kept_by_oracle(packed, 7, table)
        assert got.shape == want.shape, b
        cols = [0, 1, 2, 3, 5, 6, 7, 8, 9, 10, 11, 12, 13]
        assert np.array_equal(got[:, cols], want[:, cols]), b               # == (a zero's sign aside)
        assert_within(got[:, 4], want[:, 4], bound[:, 4], "alpha")


@pytest.mark.parametrize("variant", okr.VARIANTS)
def test_exact_golden_tells_each_variant_from_the_reference(variant):
    g = load("kitti_results_exact")
    changed = 0
    for packed, table, want, _margin in frames(g):
        rows, keep = okr.variant_rows(packed, 7, table, variant)
        got = rows[keep]
        changed += got.shape != want.shape or not np.array_equal(got[:, :4], want[:, :4])
    assert changed >= 1


def test_exact_golden_has_image_boxes_on_every_edge():
    g = load("kitti_results_exact")
    hits = collections.Counter()
    for packed, table, _want, _margin in frames(g):
        _rows, _keep, a = okr.kernel_order(packed, 7, table)
        H, W = table[28], table[29]
        hits["u0 = W"] += int((a["u"].min(1) == W).sum())
        hits["v0 = H"] += int((a["v"].min(1) == H).sum())
        hits["u1 = 0"] += int((a["u"].max(1) == 0).sum())
        hits["v1 = 0"] += int((a["v"].max(1) == 0).sum())
    assert all(hits[k] > 0 for k in ("u0 = W", "v0 = H", "u1 = 0", "v1 = 0")), hits


def test_float32_steps_equal_the_reference_rotation():
    """rotation_y is the reference's float32 limit_period, bit for bit, at k * 2pi and +-pi +-1..4 ulps."""
    g = load("kitti_results_cases")
    packed, _table, want, _margin = list(frames(g))[3]
    b = okr.f32_steps(packed[packed[:, 9] > 0.5], 7)
    assert np.array_equal(b[:, 6].astype(np.float64).view(np.uint64), want[:, 11].view(np.uint64))


@pytest.mark.parametrize("case", CASES)
def test_calibration_table_is_numpy_matmul(case):
    from det3d_b200.ops.point_cloud.kitti_results import calib_table
    g = load(case)
    for b in range(g["tables"].shape[0]):
        cal = dict(rect=g["rect"][b], Trv2c=g["Trv2c"][b], P2=g["P2"][b], image_shape=g["image_shape"][b])
        assert np.array_equal(calib_table(cal).view(np.uint64), g["tables"][b].view(np.uint64))
        assert np.array_equal(okr.calib_table(**cal).view(np.uint64), g["tables"][b].view(np.uint64))


@pytest.mark.parametrize("case", CASES)
def test_to_annos_gives_the_reference_keys_and_dtypes(case):
    from det3d_b200.ops.point_cloud.kitti_results import to_annos
    g = load(case)
    nd, B, D = int(g["nd"]), g["packed"].shape[0], g["packed"].shape[1]
    results = np.zeros((B, D, okr.COLS))
    off = np.concatenate([[0], np.cumsum(g["counts"])])
    for b in range(B):
        results[b, :g["counts"][b]] = g["rows"][off[b]:off[b + 1]]
    annos = to_annos(results, g["counts"], list(g["class_names"]))
    names = list(g["class_names"])
    for b, a in enumerate(annos):
        cal = dict(rect=g["rect"][b], Trv2c=g["Trv2c"][b], P2=g["P2"][b], image_shape=g["image_shape"][b])
        ref = okr.reference_annos(g["packed"][b], nd, cal, names)
        assert list(a) == list(ref)
        for k in ref:
            assert a[k].dtype == ref[k].dtype and a[k].shape == ref[k].shape, (case, b, k)
        assert list(a["name"]) == list(g["names"][off[b]:off[b + 1]])
        assert np.array_equal(a["score"], ref["score"], equal_nan=True)
        assert np.array_equal(a["rotation_y"], ref["rotation_y"], equal_nan=True)


def test_calibration_table_cache_is_keyed_on_bytes():
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import kitti_like_calib
    pipe = object.__new__(InferencePipeline)
    pipe._kitti_tables = collections.OrderedDict()
    cal = kitti_like_calib(3)
    t0 = pipe.kitti_calib_table(cal)
    assert pipe.kitti_calib_table(dict(cal)) is t0 and len(pipe._kitti_tables) == 1
    cal32 = {k: (np.asarray(v, np.float32) if k != "image_shape" else v) for k, v in cal.items()}
    t1 = pipe.kitti_calib_table(cal32)
    assert len(pipe._kitti_tables) == 2 and t1 is not t0
    assert np.array_equal(t0[:16], (cal["rect"] @ cal["Trv2c"]).reshape(-1))


# ---- d3b_kitti_results_dev: argument errors before any CUDA call ------------------------------------------------------
_P = 0x1000                   # stand-in for a device pointer: never dereferenced, every call below is rejected first


def _call(det=_P, calib=_P, batch=2, max_det=100, nd=7, results=_P, counts=_P):
    from det3d_b200 import _lib
    return _lib.lib().d3b_kitti_results_dev(det, calib, batch, max_det, nd, results, counts, None)


def _err():
    from det3d_b200 import _lib
    return _lib.lib().d3b_last_error()


def test_abi_null_arguments():
    for name in ("calib", "counts"):
        assert _call(**{name: None}) == 1, name
        assert b"null argument" in _err()
    for name in ("det", "results"):
        assert _call(**{name: None}) == 1, name
        assert b"null buffer" in _err()


def test_abi_batch_and_max_det_bounds():
    for batch in (0, -1, 65):
        assert _call(batch=batch) == 1 and b"batch" in _err()
    for max_det in (-1, (1 << 20) + 1):
        assert _call(max_det=max_det) == 1 and b"max_det" in _err()


def test_abi_nd_other_than_7_or_9_is_not_built():
    for nd in (-1, 0, 6, 8, 10):
        assert _call(nd=nd) == 3 and b"nd" in _err()                    # D3B_ERR_UNSUPPORTED


def test_host_arguments_are_checked():
    import torch
    from det3d_b200.datasets.kitti import convert_detection_to_kitti_annos
    from det3d_b200.ops.point_cloud.kitti_results import KittiResults
    from det3d_b200.utils.synthetic import kitti_like_calib
    with pytest.raises(ValueError):
        convert_detection_to_kitti_annos(torch.zeros((1, 4, 10)), [kitti_like_calib(0)], ["Car"])   # host tensor
    for b in (0, 65):
        with pytest.raises(ValueError):
            KittiResults(b, "cpu")
