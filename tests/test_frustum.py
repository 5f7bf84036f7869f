"""KITTI camera-frustum crop on the host side (no GPU needed): the float64 planes of camera_frustum_planes and the CPU
oracle's keep masks against the reference's own functions (tests/golden/frustum_kitti_*.npz, make_golden_frustum.py),
and Preprocess(remove_outside_points=True) built from the stock configs."""
import os

import numpy as np
import pytest

from conftest import ROOT, load_golden

CASES = ("scans", "adversarial")


def _calib(g, b):
    return dict(rect=g["rect"][b], Trv2c=g["Trv2c"][b], P2=g["P2"][b], image_shape=g["image_shape"][b])


@pytest.mark.parametrize("case", CASES)
def test_camera_frustum_planes_equal_the_reference_bit_for_bit(case):
    from det3d_b200.core.bbox.box_np_ops import camera_frustum_planes
    g = load_golden("frustum_kitti_" + case)
    for b in range(g["planes"].shape[0]):
        c = _calib(g, b)
        got = camera_frustum_planes(c["rect"], c["Trv2c"], c["P2"], c["image_shape"])
        assert got.dtype == np.float64 and got.shape == (6, 4)
        assert np.array_equal(got.view(np.uint64), g["planes"][b].view(np.uint64)), b


@pytest.mark.parametrize("case", CASES + ("rounding",))
def test_oracle_masks_equal_the_reference(case):
    from oracle.frustum import keep_mask
    g = load_golden("frustum_kitti_" + case)
    off = g["offsets"]
    for b in range(off.shape[0] - 1):
        pts = g["points"][off[b]:off[b + 1]]
        assert np.array_equal(keep_mask(pts, g["planes"][b]), g["mask"][off[b]:off[b + 1]]), b


@pytest.mark.parametrize("variant", ["fma_chain_yx", "fma_chain_xy", "fma_d_first", "d_first", "right_assoc", "pairwise",
                                     "strict_gt"])
def test_rounding_golden_tells_every_other_evaluation_from_the_reference(variant):
    """The reference rounds every product and sum on its own, left to right, and drops a point at s >= 0.  An
    FMA-contracted chain (what a compiler may emit for x*n0 + y*n1 + z*n2 + d), another summation order or a `>` test
    decides differently on some points of frustum_kitti_rounding.npz, so a kernel built any of those ways fails the
    device test on that golden."""
    from oracle.frustum import variant_keep_mask
    g = load_golden("frustum_kitti_rounding")
    off = g["offsets"]
    differ = 0
    for b in range(off.shape[0] - 1):
        pts = g["points"][off[b]:off[b + 1]]
        differ += int((variant_keep_mask(pts, g["planes"][b], variant) != g["mask"][off[b]:off[b + 1]]).sum())
    assert differ >= 4, differ


def test_plane_cache_keeps_float32_and_float64_calibrations_apart():
    import collections

    from det3d_b200.apis import InferencePipeline
    from det3d_b200.core.bbox.box_np_ops import camera_frustum_planes
    from det3d_b200.utils.synthetic import kitti_like_calib
    pipe = object.__new__(InferencePipeline)
    pipe._planes = collections.OrderedDict()
    c64 = kitti_like_calib(3)
    c32 = {k: (v.astype(np.float32) if k != "image_shape" else v) for k, v in c64.items()}
    for cal in (c64, c32, c64):
        want = camera_frustum_planes(cal["rect"], cal["Trv2c"], cal["P2"], cal["image_shape"])
        assert np.array_equal(pipe.frustum_planes(cal).view(np.uint64), want.view(np.uint64))
    assert len(pipe._planes) == 2


def _plane_values(g):
    """s of every (point, plane) of the adversarial golden, in the reference's order."""
    off, out = g["offsets"], []
    with np.errstate(invalid="ignore"):
        for b in range(off.shape[0] - 1):
            p = g["points"][off[b]:off[b + 1], :3].astype(np.float64)
            out.append(np.stack([((p[:, 0] * n[0] + p[:, 1] * n[1]) + p[:, 2] * n[2]) + n[3] for n in g["planes"][b]], 1))
    return np.concatenate(out)


def test_adversarial_golden_covers_the_boundary_cases():
    """At least one s is exactly 0 (outside: the reference tests s >= 0), NaN / inf coordinates are present and NaN ones
    are kept, points sit within a few ulps of every plane, and both outcomes occur."""
    g = load_golden("frustum_kitti_adversarial")
    s = _plane_values(g)
    pts, mask = g["points"], g["mask"]
    assert (s == 0).any()
    zero_rows = (s == 0).any(1)
    assert not mask[zero_rows].any()
    nan_rows = np.isnan(pts[:, :3]).any(1)
    assert nan_rows.sum() >= 3 and mask[nan_rows].all()
    assert np.isinf(pts[:, :3]).any()
    scale = np.abs(g["planes"][..., :3]).max()
    assert (np.abs(s) < 1e-9 * scale).sum() >= 100
    assert 0.2 < mask.mean() < 0.8


KITTI_STOCK = ["examples/second/configs/kitti_car_vfev3_spmiddlefhd_rpn1_mghead_syncbn.py",
               "examples/second/configs/kitti_all_vfev3_spmiddlefhd_rpn1_mghead_syncbn.py",
               "examples/point_pillars/configs/kitti_point_pillars_mghead_syncbn.py"]
OTHER_STOCK = [("examples/cbgs/configs/nusc_all_vfev3_spmiddleresnetfhd_rpn2_mghead_syncbn.py", "NuScenesDataset"),
               ("examples/cbgs/configs/lyft_all_vfev3_spmiddleresnetfhd_rpn2_mghead_syncbn.py", "LyftDataset")]


def _stock(rel):
    from boundary_golden import reference_config
    from boundary_golden_more import reference_config_more
    try:
        return reference_config(rel)
    except KeyError:
        return reference_config_more(rel)


def _test_pipeline_with_crop(rel):
    """The stock config's test_pipeline (as the reference's file parses) with remove_outside_points=True in its
    Preprocess step, built through PIPELINES."""
    from det3d.datasets.pipelines import Compose
    cfg = _stock(rel)
    steps = []
    for s in cfg.test_pipeline:
        s = dict(s)
        if s["type"] == "Preprocess":
            s["cfg"] = dict(s["cfg"], remove_outside_points=True)
        steps.append(s)
    return Compose(steps)


@pytest.mark.parametrize("rel", KITTI_STOCK)
def test_preprocess_with_remove_outside_points_builds_from_the_kitti_configs(rel):
    pipe = _test_pipeline_with_crop(rel)
    pre = [t for t in pipe.transforms if type(t).__name__ == "Preprocess"]
    assert len(pre) == 1 and pre[0].remove_outside_points is True


@pytest.mark.parametrize("rel,dataset", OTHER_STOCK)
def test_preprocess_remove_outside_points_raises_without_a_calibration(rel, dataset):
    """The reference's `assert calib is not None`: nuScenes and Lyft samples carry no camera calibration."""
    pipe = _test_pipeline_with_crop(rel)
    pre = next(t for t in pipe.transforms if type(t).__name__ == "Preprocess")
    pts = np.zeros((4, 5), np.float32)
    res = dict(type=dataset, lidar=dict(points=pts, combined=pts), metadata={})
    with pytest.raises(ValueError, match="calib"):
        pre(res, {})
