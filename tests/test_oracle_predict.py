"""CPU checks of the predict oracle (oracle/predict_cpu.py) that tests/test_predict_task_gpu.py compares the device
predict against: its standup conversion is pinned to the reference's own functions, and its general restatement gives
what the e2e tests' predict_sample_task gives where both apply."""
import numpy as np
import torch

from conftest import load_golden


def test_standup_boxes_match_reference():
    """center_to_corner_box2d + corner_to_standup_nd (the boxes the axis-aligned NMS compares) against the
    reference's functions run on the same fp32 inputs (tests/golden/make_golden_predict_standup.py)."""
    from oracle.predict_cpu import center_to_corner_box2d, corner_to_standup_nd
    g = load_golden("predict_standup")
    corners = center_to_corner_box2d(torch.from_numpy(g["centers"]), torch.from_numpy(g["dims"]),
                                     torch.from_numpy(g["angles"]))
    standup = corner_to_standup_nd(corners)
    # corner order and rotation sense must be the reference's; the last bit of a two-term dot product may depend on
    # the CPU's FMA use inside einsum
    scale = np.abs(g["centers"]).max(1) + np.abs(g["dims"]).max(1)
    tol = 4 * np.finfo(np.float32).eps * scale
    assert corners.shape == g["corners"].shape
    assert (np.abs(corners.numpy() - g["corners"]).max((1, 2)) <= tol).all()
    assert (np.abs(standup.numpy() - g["standup"]).max(1) <= tol).all()


def _head(seed, A, n_cls, code, nd):
    rng = np.random.default_rng(seed)
    cls = torch.from_numpy(rng.normal(-2.0, 1.5, size=(A, n_cls)).astype(np.float32))
    enc = torch.from_numpy((rng.normal(size=(A, code)) * 0.2).astype(np.float32))
    dirs = torch.from_numpy(rng.normal(size=(A, 2)).astype(np.float32))
    anchors = np.zeros((A, nd), np.float32)
    anchors[:, 0] = rng.uniform(0.0, 70.0, A)
    anchors[:, 1] = rng.uniform(-40.0, 40.0, A)
    anchors[:, 2] = -1.0
    anchors[:, 3:6] = [1.6, 3.9, 1.56]
    anchors[:, nd - 1] = rng.choice([0.0, np.pi / 2], A)
    return cls, enc, dirs, torch.from_numpy(anchors)


def test_reference_reproduces_predict_sample_task():
    """The rotated-NMS, thresholded, range-masked case both oracles state: same boxes, scores and labels."""
    from oracle.predict_cpu import predict_sample_task, predict_task_reference
    test_cfg = dict(score_threshold=0.3, post_center_limit_range=[0.0, -39.68, -5.0, 69.12, 39.68, 5.0],
                    nms=dict(nms_pre_max_size=1000, nms_post_max_size=100, nms_iou_threshold=0.5))
    for seed, n_cls, vec in ((0, 1, True), (1, 2, True), (2, 3, False)):
        cls, enc, dirs, anchors = _head(seed, 4000, n_cls, 7 + int(vec), 7)
        bx, sc, lb = predict_sample_task(cls, enc, dirs, anchors, test_cfg, vec, direction_offset=0.3)
        got = predict_task_reference(cls, enc, dirs, anchors, 0.3, 1000, 100, 0.5, True,
                                     test_cfg["post_center_limit_range"], 0.3, vec)
        m = got["valid"]
        assert bx.shape[0] >= 20 and int(m.sum()) == bx.shape[0]
        assert np.array_equal(got["boxes"][m], bx.numpy())
        assert np.array_equal(got["scores"][m], sc.numpy())
        assert np.array_equal(got["labels"][m], lb.numpy())


def test_reference_label_rule_and_nan():
    """Labels come from the first maximal fp32 SCORE (logits 20 and 25 both score 1.0f: label 0), and an anchor with
    a NaN logit in any class is dropped by a positive threshold."""
    from oracle.predict_cpu import predict_task_reference
    cls = torch.tensor([[20.0, 25.0], [1.0, 3.0], [float("nan"), 5.0], [4.0, float("nan")], [0.5, 0.25]])
    enc = torch.zeros((5, 7))
    anchors = torch.tensor([[10.0 * i, 0.0, 0.0, 1.0, 2.0, 1.0, 0.0] for i in range(5)])
    got = predict_task_reference(cls, enc, None, anchors, 0.5, 5, 5, 0.5)
    assert got["nms_in"].tolist() == [0, 1, 4]
    assert got["labels"].tolist() == [0, 1, 0]
    got = predict_task_reference(cls, enc, None, anchors, 0.0, 5, 5, 0.5, use_rotate_nms=False)
    assert sorted(got["nms_in"].tolist()) == [0, 1, 2, 3, 4]      # no filter at threshold 0
