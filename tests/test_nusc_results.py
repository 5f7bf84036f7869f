"""nuScenes result rows on the CPU: the checker (oracle/nusc_results.py) against the goldens the reference's own conversion
code produced (tests/golden/make_golden_nusc_results.py), the exact golden bit for bit, the variants it tells apart, the
host side of the device path (pose table, attribute table, nusc_annos formatting, the per-record cache, argument checks)
and the argument checks of d3b_nusc_results_dev, which return before any CUDA call.  The device kernel is checked
against the same goldens in test_nusc_results_gpu.py."""
import collections
import os

import numpy as np
import pytest

from oracle import nusc_results as onr

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CASES = ("nusc_results_cases", "nusc_results_exact")
U = 2.0 ** -53


def load(name):
    return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def records(g):
    return [{"calibrated_sensor": {"translation": list(g["cs_translation"][b]), "rotation": list(g["cs_rotation"][b])},
             "ego_pose": {"translation": list(g["ego_translation"][b]), "rotation": list(g["ego_rotation"][b])}}
            for b in range(g["packed"].shape[0])]


def fallback(g):
    """{class: its most frequent attribute} as the golden's (class, moving) table implies it: the still attribute
    where the still rule names none, else the moving one (pedestrian; bus is ruled both ways)."""
    return {str(n): str(m if n in onr.STILL else s)
            for n, s, m in zip(g["class_names"], g["attr_still"], g["attr_moving"])}


def golden_rows(g):
    """The reference's boxes as rows [n, 15] (moving from the attribute is not recoverable: column 14 is NaN)."""
    n = g["score"].shape[0]
    return np.concatenate([g["translation"], g["size"], g["rotation"], g["velocity"], g["score"][:, None],
                           g["label"][:, None].astype(np.float64), np.full((n, 1), np.nan)], 1)


def per_sample(g):
    off = np.concatenate([[0], np.cumsum(g["counts"])])
    rows = golden_rows(g)
    recs = records(g)
    for b in range(g["packed"].shape[0]):
        yield (b, g["packed"][b], g["tables"][b], recs[b], rows[off[b]:off[b + 1]],
               list(g["attributes"][off[b]:off[b + 1]]), g["margin"][b])


def assert_within(got, want, bound, what):
    ok = (got == want) | (np.abs(got - want) <= bound)
    assert ok.all(), "%s: %d values outside the bound, worst ratio %s" % (
        what, int((~ok).sum()), np.max(np.where(ok, 0, np.abs(got - want) / np.maximum(bound, 1e-300))))


def test_goldens_hold_the_cases():
    g = load("nusc_results_cases")
    valid = (g["packed"][..., 11] > 0.5).sum(1)
    assert list(g["counts"]) == list(valid)
    assert 0 in g["counts"] and g["packed"].shape[1] in g["counts"]       # an empty sample, a full one
    assert set(g["label"].tolist()) == set(range(10))
    assert np.isnan(g["packed"][0][g["packed"][0][:, 11] <= 0.5, 0]).any()  # invalid rows carry NaN
    speeds = np.abs(g["margin"][2][:96])
    assert np.all(speeds > 1) and np.all(g["margin"][g["packed"][..., 11] > 0.5] > 1)
    # both moving and still boxes straddle the 0.2 threshold
    assert {"vehicle.moving", "vehicle.parked"} <= set(g["attributes"][g["counts"][:2].sum():g["counts"][:3].sum()])


@pytest.mark.parametrize("case", CASES)
def test_oracle_reference_equals_the_lifted_reference(case):
    g = load(case)
    exact = case == "nusc_results_exact"
    names = list(g["class_names"])
    annos = onr.reference_annos(g["packed"], records(g), list(g["tokens"]), names, fallback(g))
    assert list(annos["results"]) == list(g["tokens"])
    for b, packed, table, rec, want, attrs, _m in per_sample(g):
        boxes = annos["results"][g["tokens"][b]]
        assert len(boxes) == want.shape[0]
        got = np.array([a["translation"] + a["size"] + a["rotation"] + a["velocity"]
                        + [a["detection_score"], names.index(a["detection_name"]), np.nan] for a in boxes]
                       ).reshape(-1, 15)
        assert [a["attribute_name"] for a in boxes] == attrs
        assert np.array_equal(got[:, 3:6], want[:, 3:6]) and np.array_equal(got[:, 12:14], want[:, 12:14])
        if exact:
            assert np.array_equal(got[:, :12], want[:, :12]), b
        else:
            bound, _margin = onr.error_bound(packed, table, rec)
            kept = packed[:, 11] > 0.5
            for cols, what in ((slice(0, 3), "translation"), (slice(6, 10), "rotation"), (slice(10, 12), "velocity")):
                assert_within(got[:, cols], want[:, cols], bound[kept][:, cols], "%s sample %d %s" % (case, b, what))


@pytest.mark.parametrize("case", CASES)
def test_kernel_order_equals_the_reference_within_the_bound(case):
    g = load(case)
    names = list(g["class_names"])
    for b, packed, table, rec, want, attrs, margin in per_sample(g):
        rows, valid, _a = onr.kernel_order(packed, table)
        bound, m = onr.error_bound(packed, table, rec)
        assert np.array_equal(m, margin)
        assert np.all(margin[valid] > 1), "a speed decision inside the error bound"
        got = rows[valid]
        assert got.shape[0] == want.shape[0]
        assert np.array_equal(got[:, 3:6], want[:, 3:6]) and np.array_equal(got[:, 12:14], want[:, 12:14])
        assert onr.attributes(got, names, fallback(g)) == attrs
        assert_within(got[:, :12], want[:, :12], bound[valid][:, :12], "%s sample %d" % (case, b))
        if case == "nusc_results_exact":
            assert np.array_equal(got[:, :12], want[:, :12]), b


@pytest.mark.parametrize("variant", onr.VARIANTS)
def test_exact_golden_tells_each_variant_from_the_reference(variant):
    g = load("nusc_results_exact")
    names = list(g["class_names"])
    changed = 0
    for _b, packed, table, _rec, want, attrs, _m in per_sample(g):
        rows, vattrs = onr.variant_output(packed, table, names, fallback(g), variant)
        bound, _margin = onr.error_bound(packed, table)
        valid = packed[:, 11] > 0.5
        changed += int((np.abs(rows[valid][:, :12] - want[:, :12]) > bound[valid][:, :12]).any(1).sum())
        changed += sum(a != b for a, b in zip([v for v, k in zip(vattrs, valid) if k], attrs))
    assert changed >= 1


def test_attribute_table_is_the_reference_rule():
    from det3d_b200.ops.point_cloud.nusc_results import attribute_table
    for case in CASES:
        g = load(case)
        table = attribute_table(list(g["class_names"]))
        assert [t[0] for t in table] == list(g["attr_still"])
        assert [t[1] for t in table] == list(g["attr_moving"])
    t = dict(zip(g["class_names"], table))
    assert t["barrier"] == ("cycle.with_rider", "cycle.with_rider")
    assert t["traffic_cone"] == ("cycle.with_rider", "cycle.with_rider")
    assert t["car"] == ("vehicle.parked", "vehicle.moving")
    with pytest.raises(ValueError):
        attribute_table(["car", "Car"])


@pytest.mark.parametrize("case", CASES)
def test_pose_table_is_the_stand_in_rotation_matrix(case):
    from det3d_b200.ops.point_cloud.nusc_results import pose_table
    g = load(case)
    for b, rec in enumerate(records(g)):
        assert np.array_equal(pose_table(rec).view(np.uint64), onr.pose_table(rec).view(np.uint64))
        assert np.array_equal(pose_table(rec).view(np.uint64), g["tables"][b].view(np.uint64))


def test_pose_table_agrees_with_scipy():
    from scipy.spatial.transform import Rotation

    from det3d_b200.ops.point_cloud.nusc_results import pose_table
    g = load("nusc_results_cases")
    for rec in records(g):
        t = pose_table(rec)
        for R, q in ((t[0:9], t[24:28]), (t[12:21], t[28:32])):
            # scipy normalises q; pyquaternion leaves a q with |1 - q . q| < 1e-14 as it is, which scales R by q . q
            nu = abs(1.0 - np.dot(q, q))
            want = Rotation.from_quat([q[1], q[2], q[3], q[0]]).as_matrix().reshape(-1)
            assert np.all(np.abs(R - want) <= 4 * U + nu * np.abs(want)), np.abs(R - want).max() / U
        # the Hamilton product of the stand-in (pyquaternion's __mul__) is scipy's composition
        qc, qp = t[24:28], t[28:32]
        prod = (onr.Quaternion(qp) * onr.Quaternion(qc)).q
        want = (Rotation.from_quat([qp[1], qp[2], qp[3], qp[0]]) * Rotation.from_quat([qc[1], qc[2], qc[3], qc[0]])
                ).as_quat(canonical=False)
        want = np.array([want[3], want[0], want[1], want[2]])
        want = want if np.dot(want, prod) > 0 else -want
        nu = abs(1.0 - np.dot(qc, qc)) + abs(1.0 - np.dot(qp, qp))
        assert np.all(np.abs(prod - want) <= 4 * U + nu), np.abs(prod - want).max() / U


def test_pose_table_rejects_bad_records():
    from det3d_b200.ops.point_cloud.nusc_results import pose_table
    ok = records(load("nusc_results_cases"))[0]
    bad = [None, {"ego_pose": ok["ego_pose"]}, {"calibrated_sensor": {"rotation": [1, 0, 0, 0]}, "ego_pose": ok["ego_pose"]}]
    for k in ("calibrated_sensor", "ego_pose"):
        for field, value in (("rotation", [1.0, 0.0, np.nan, 0.0]), ("rotation", [1.0 + 2e-6, 0, 0, 0]),
                             ("rotation", [0.5, 0.5, 0.5]), ("translation", [1.0, np.inf, 0.0]),
                             ("translation", [1.0, 2.0])):
            r = {kk: dict(vv) for kk, vv in ok.items()}
            r[k][field] = value
            bad.append(r)
    for r in bad:
        with pytest.raises(ValueError):
            pose_table(r)
    r = {kk: dict(vv, extra="ignored") for kk, vv in ok.items()}
    r["token"] = "abc"
    assert np.array_equal(pose_table(r), pose_table(ok))
    r["ego_pose"]["rotation"] = list(np.array(ok["ego_pose"]["rotation"]) * (1 + 5e-7))       # normalised
    assert np.allclose(pose_table(r), pose_table(ok), rtol=0, atol=1e-12)


@pytest.mark.parametrize("case", CASES)
def test_to_nusc_annos_gives_the_reference_format(case):
    from det3d_b200.ops.point_cloud.nusc_results import COLS, to_nusc_annos
    g = load(case)
    names, tokens = [str(n) for n in g["class_names"]], [str(t) for t in g["tokens"]]
    B, D = g["packed"].shape[:2]
    results = np.zeros((B, D, COLS))
    for b, packed, table, _rec, _want, _attrs, _m in per_sample(g):
        rows, valid, _a = onr.kernel_order(packed, table)
        results[b, :int(valid.sum())] = rows[valid]
    got = to_nusc_annos(results, g["counts"], names, tokens)
    ref = onr.reference_annos(g["packed"], records(g), tokens, names, fallback(g))
    assert list(got) == ["results", "meta"] == list(ref) and got["meta"] == ref["meta"]
    assert list(got["results"]) == tokens
    for t in tokens:
        assert len(got["results"][t]) == len(ref["results"][t])
        for a, r in zip(got["results"][t], ref["results"][t]):
            assert list(a) == list(r)
            assert all(type(a[k]) is type(r[k]) for k in r)
            assert all(type(v) is float for k in ("translation", "size", "rotation", "velocity") for v in a[k])
            assert [a[k] for k in ("sample_token", "size", "detection_name", "detection_score", "attribute_name")] == \
                   [r[k] for k in ("sample_token", "size", "detection_name", "detection_score", "attribute_name")]


def test_to_nusc_annos_rejects_nan_centres_and_sizes():
    from det3d_b200.ops.point_cloud.nusc_results import to_nusc_annos
    results = np.zeros((2, 3, 15))
    results[1, 1, 4] = np.nan
    with pytest.raises(ValueError, match="tok1"):
        to_nusc_annos(results, np.array([3, 2]), ["car"], ["tok0", "tok1"])
    assert len(to_nusc_annos(results, np.array([3, 1]), ["car"], ["tok0", "tok1"])["results"]["tok1"]) == 1


def test_pose_table_cache_is_keyed_on_bytes():
    from det3d_b200.apis import InferencePipeline
    pipe = object.__new__(InferencePipeline)
    pipe._nusc_tables = collections.OrderedDict()
    recs = records(load("nusc_results_cases"))
    t0 = pipe.nusc_pose_table(recs[0])
    assert pipe.nusc_pose_table({k: dict(v) for k, v in recs[0].items()}) is t0 and len(pipe._nusc_tables) == 1
    t1 = pipe.nusc_pose_table(recs[1])
    assert t1 is not t0 and len(pipe._nusc_tables) == 2
    with pytest.raises(ValueError):
        pipe.nusc_pose_table({"ego_pose": recs[0]["ego_pose"]})


def test_host_arguments_are_checked():
    import torch

    from det3d_b200.apis.pipeline import _NuscStep
    from det3d_b200.datasets.nuscenes import convert_detection_to_nusc_annos
    from det3d_b200.ops.point_cloud.nusc_results import NuscResults, check_tokens
    recs = records(load("nusc_results_cases"))
    names = ["car"]
    with pytest.raises(ValueError):
        convert_detection_to_nusc_annos(torch.zeros((1, 4, 12)), recs[:1], ["t"], names)      # host tensor
    for b in (0, 65):
        with pytest.raises(ValueError):
            NuscResults(b, "cpu")
    for tokens in (["a"], ["a", "a"], ["a", 3], ("a", b"b")):
        with pytest.raises(ValueError):
            check_tokens(tokens, 2)
    assert check_tokens(("a", "b"), 2) == ["a", "b"]

    class Coder:
        n_dim = 9

    class Head:
        box_coder = Coder()

    class Model:
        bbox_head = Head()

    class Cfg:
        tasks = [dict(class_names=["car", "pedestrian"])]

    pipe = type("P", (), {})()
    pipe.model, pipe.cfg, pipe.device = Model(), Cfg(), torch.device("cpu")
    pipe.class_names = lambda: ["car", "pedestrian"]
    pipe.nusc_pose_table = lambda r: onr.pose_table(r)
    _NuscStep(pipe, 2, recs[:2], ["a", "b"])                                    # well formed
    for poses, tokens in ((None, ["a", "b"]), (recs[:2], None), (recs[:1], ["a", "b"]), (recs[:2], ["a"]),
                          (recs[:2], ["a", "a"]), (recs[:2], ["a", 1])):
        with pytest.raises(ValueError):
            _NuscStep(pipe, 2, poses, tokens)
    pipe.class_names = lambda: ["car", "Pedestrian"]
    with pytest.raises(ValueError):
        _NuscStep(pipe, 2, recs[:2], ["a", "b"])
    pipe.class_names = lambda: ["car", "pedestrian"]
    Coder.n_dim = 7                                                             # CBGS Lyft: no velocity
    with pytest.raises(ValueError):
        _NuscStep(pipe, 2, recs[:2], ["a", "b"])


# ---- d3b_nusc_results_dev: argument errors before any CUDA call -------------------------------------------------------
_P = 0x1000                   # stand-in for a device pointer: never dereferenced, every call below is rejected first


def _call(det=_P, poses=_P, batch=2, max_det=100, nd=9, results=_P, counts=_P):
    from det3d_b200 import _lib
    return _lib.lib().d3b_nusc_results_dev(det, poses, batch, max_det, nd, results, counts, None)


def _err():
    from det3d_b200 import _lib
    return _lib.lib().d3b_last_error()


def test_abi_null_arguments():
    for name in ("poses", "counts"):
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


def test_abi_nd_other_than_9_is_not_built():
    for nd in (-1, 0, 7, 8, 10):
        assert _call(nd=nd) == 3 and b"nd" in _err()                    # D3B_ERR_UNSUPPORTED
