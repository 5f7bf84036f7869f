"""SECOND KITTI three-class and CBGS Lyft on the host side: the reference's stock files load unchanged and build the same
models as the shipped subsets (configs/second_kitti_all.py, configs/cbgs_lyft.py); the Lyft anchors equal the
reference's bit for bit; the Lyft LoadPointCloudFromFile follows the reference's read_file; the generalised oracles
(tests/oracle_tasks.py) give the original oracles' outputs on the configs those cover."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from boundary_golden_more import reference_config_more
from conftest import ROOT, load_golden

KITTI_ALL = "examples/second/configs/kitti_all_vfev3_spmiddlefhd_rpn1_mghead_syncbn.py"
LYFT = "examples/cbgs/configs/lyft_all_vfev3_spmiddleresnetfhd_rpn2_mghead_syncbn.py"


def _shipped(name):
    from det3d.torchie import Config
    return Config.fromfile(os.path.join(ROOT, "configs", name))


@pytest.mark.parametrize("rel,shipped,n_tasks,fused_cols", [(KITTI_ALL, "second_kitti_all.py", 3, 60),
                                                             (LYFT, "cbgs_lyft.py", 5, 148)])
def test_reference_config_loads_unchanged_and_matches_the_shipped_subset(rel, shipped, n_tasks, fused_cols):
    from det3d.models import build_detector

    cfg, mine = reference_config_more(rel), _shipped(shipped)
    model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    m2 = build_detector(mine.model, train_cfg=None, test_cfg=mine.test_cfg)
    assert type(model).__name__ == type(m2).__name__ == "VoxelNet"
    a, b = model.state_dict(), m2.state_dict()
    assert list(a) == list(b) and all(a[k].shape == b[k].shape for k in a)
    for key in ("test_cfg", "voxel_generator", "target_assigner"):
        assert cfg[key].to_dict() == mine[key].to_dict(), key
    assert cfg.assigner.out_size_factor == mine.assigner.out_size_factor == 8
    assert len(model.bbox_head.tasks) == n_tasks
    cols = 0
    for t in model.bbox_head.tasks:
        cols += sum(m.out_channels for m in (t.conv_box, t.conv_cls, t.conv_dir))
    assert cols == fused_cols
    for k in ("direction_offset", "encode_rad_error_by_sin"):
        assert cfg.model.bbox_head[k] == mine.model.bbox_head[k]
    if rel == LYFT:
        assert tuple(a["backbone.middle_conv.0.weight"].shape) == (3, 3, 3, 3, 16)     # SubM 3 -> 16
        assert cfg.model.reader.num_input_features == 3 and model.bbox_head.box_n_dim == 7
        assert model.bbox_head.num_classes == [1, 1, 2, 1, 2]
        assert model.bbox_head.direction_offset == 0.785
    else:
        assert tuple(a["backbone.middle_conv.0.weight"].shape) == (3, 3, 3, 4, 16)
        assert len(model.backbone.fused().plan) == 14
        assert cfg.voxel_generator.max_voxel_num == 40000


def test_fused_bev_takes_both_rpns():
    from det3d.models import build_detector
    from det3d_b200.ops.spconv import bev

    for name in ("second_kitti_all.py", "cbgs_lyft.py"):
        cfg = _shipped(name)
        model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
        assert bev.rpn_is_fusable16(model.neck), name


def test_lyft_anchors_match_reference_golden():
    from det3d_b200.core.anchor.anchor_generator import anchors_for_tasks, create_anchors_3d_range

    g = load_golden("anchors_lyft")
    cfg = _shipped("cbgs_lyft.py")
    for ag in cfg.target_assigner.anchor_generators:
        name = ag["class_name"]
        a = create_anchors_3d_range([1, 252, 252], ag["anchor_ranges"], ag["sizes"], ag["rotations"]).reshape(-1, 7)
        assert a.dtype == np.float32 and list(a.shape) == g[name + "_shape"].tolist() == [127008, 7]
        assert np.array_equal(a[g[name + "_sample_idx"]], g[name + "_sample"]), name
        assert np.array_equal([a.astype(np.float64).sum(), (a.astype(np.float64) ** 2).sum()], g[name + "_checksum"]), name
    tasks = anchors_for_tasks(cfg.target_assigner, [2016, 2016, 40], 8)
    assert [t.shape for t in tasks] == [(127008, 7), (127008, 7), (254016, 7), (127008, 7), (254016, 7)]
    # a two-class task holds, per cell, its first class's two rotations, then its second's (preprocess.py:355-378)
    moto = tasks[2].reshape(252 * 252, 4, 7)
    idx = g["motorcycle_sample_idx"]
    assert np.array_equal(moto[idx // 2, idx % 2], g["motorcycle_sample"])
    idx = g["bicycle_sample_idx"]
    assert np.array_equal(moto[idx // 2, 2 + idx % 2], g["bicycle_sample"])


def _reference_read_file(path, num_point_feature=4):
    """loading.py:17-31 of the reference, restated."""
    points = np.fromfile(path, dtype=np.float32)
    s = points.shape[0]
    if s % 5 != 0:
        points = points[: s - (s % 5)]
    return points.reshape(-1, 5)[:, :num_point_feature]


def test_lyft_load_point_cloud_follows_read_file(tmp_path):
    from det3d.datasets.pipelines import Compose

    rng = np.random.default_rng(5)
    raw = rng.normal(size=5 * 1234 + 3).astype(np.float32)           # a trailing partial record of 3 floats
    path = tmp_path / "LIDAR_TOP.bin"
    raw.tofile(path)
    pipe = Compose(reference_config_more(LYFT).test_pipeline)
    load = pipe.transforms[0]
    res, info = load({"lidar": {}, "metadata": {}}, {"ref_info": {"LIDAR_TOP": {"lidar_path": str(path)}}})
    pts = res["lidar"]["points"]
    assert res["type"] == "LyftDataset"
    assert pts.dtype == np.float32 and pts.shape == (1234, 4)
    assert np.array_equal(pts, _reference_read_file(str(path)))
    assert np.array_equal(pts, raw[:5 * 1234].reshape(-1, 5)[:, :4])
    # the host steps after it take the Lyft sample; Voxelization runs on the device (tests/test_stock_configs_more_gpu.py)
    for t in pipe.transforms[1:3]:
        res, info = t(res, info)
    assert res["mode"] == "val" and res["lidar"]["points"] is pts
    assign = pipe.transforms[4]
    assert [a.shape[0] for a in assign.anchors(pipe.transforms[3].voxel_generator.grid_size)] == \
        [127008, 127008, 254016, 127008, 254016]


def test_stock_test_pipelines_build():
    from det3d.datasets.pipelines import Compose

    for rel in (KITTI_ALL, LYFT):
        pipe = Compose(reference_config_more(rel).test_pipeline)
        assert [type(t).__name__ for t in pipe.transforms] == ["LoadPointCloudFromFile", "LoadPointCloudAnnotations",
                                                               "Preprocess", "Voxelization", "AssignTarget", "Reformat"]


# ---------------------------------------------------------------------------------------------------------------------
# the generalised oracles on the configs the original ones cover
# ---------------------------------------------------------------------------------------------------------------------

def _random_heads(cfg, sd, anchors, H, W, B, seed):
    """Seeded head outputs in the oracles' NHWC layout, scaled so that a few percent of the anchors pass."""
    g = torch.Generator().manual_seed(seed)
    heads = []
    for t, a in enumerate(anchors):
        na = a.shape[0] // (H * W)
        d = {}
        for key, name in (("conv_box", "box"), ("conv_cls", "cls"), ("conv_dir", "dir")):
            w = "bbox_head.tasks.%d.%s.weight" % (t, key)
            if w in sd:
                c = sd[w].shape[0]
                x = torch.randn((B, H, W, c), generator=g) * (0.1 if name == "box" else 1.0)
                if name == "cls":
                    x -= 2.5
                d[name] = x
        assert d["box"].shape[-1] % na == 0
        heads.append(d)
    return heads


def test_second_tasks_oracle_reproduces_second_cpu_bit_for_bit():
    from det3d.models import build_detector
    from det3d_b200.core.anchor.anchor_generator import anchors_for_tasks
    from oracle.second_cpu import SecondCPU
    from oracle_tasks import SecondTasksCPU

    cfg = _shipped("second_kitti_car.py")
    torch.manual_seed(0)
    sd = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).state_dict()
    anchors = anchors_for_tasks(cfg.target_assigner, [1408, 1600, 40], 8)
    old, new = SecondCPU(cfg, sd, anchors), SecondTasksCPU(cfg, sd, anchors)
    x = torch.relu(torch.randn((2, 128, 200, 176), generator=torch.Generator().manual_seed(3)))
    for k in ("conv_box", "conv_cls", "conv_dir"):
        new.sd["bbox_head.tasks.0.%s.weight" % k] = old.sd["bbox_head.tasks.0.%s.weight" % k] = \
            torch.randn_like(old.sd["bbox_head.tasks.0.%s.weight" % k]) * 0.05
    box, cls, dirs = old.head(x)
    assert all(torch.equal(u, v) for u, v in zip((box, cls, dirs), new.task_head(x, 0)))
    cls = cls + 1.5
    want = old.predict(box, cls, dirs)
    got = new.predict_tasks([(box, cls, dirs)])
    assert sum(w["box3d_lidar"].shape[0] for w in want) > 20
    for w, g in zip(want, got):
        for k in ("box3d_lidar", "scores", "label_preds"):
            assert w[k].dtype == g[k].dtype and torch.equal(w[k], g[k]), k


def test_cbgs_tasks_oracle_reproduces_cbgs_cpu_bit_for_bit():
    from det3d.models import build_detector
    from det3d_b200.core.anchor.anchor_generator import anchors_for_tasks
    from oracle.cbgs_cpu import CbgsCPU
    from oracle_tasks import CbgsTasksCPU

    cfg = _shipped("cbgs_nusc.py")
    sd = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).state_dict()
    anchors = anchors_for_tasks(cfg.target_assigner, [1024, 1024, 40], 8)
    old, new = CbgsCPU(cfg, sd, anchors), CbgsTasksCPU(cfg, sd, anchors)
    heads = _random_heads(cfg, old.sd, old.anchors, 128, 128, 2, 7)
    want, got = old.predict_tasks(heads), new.predict_tasks(heads)
    assert sum(w["box3d_lidar"].shape[0] for w in want) > 20
    for w, g in zip(want, got):
        for k in ("box3d_lidar", "scores", "label_preds"):
            assert w[k].dtype == g[k].dtype and torch.equal(w[k], g[k]), k


def test_generalised_oracles_on_the_new_configs():
    """Label offsets and the Lyft direction offset: each task's detections carry its labels, and a Lyft box's angle is
    flipped by pi exactly when (angle - 0.785 > 0) disagrees with its direction label."""
    from det3d.models import build_detector
    from det3d_b200.core.anchor.anchor_generator import anchors_for_tasks
    from oracle.predict_cpu import predict_sample_task
    from oracle_tasks import CbgsTasksCPU, SecondTasksCPU

    cfg = _shipped("second_kitti_all.py")
    sd = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).state_dict()
    anchors = anchors_for_tasks(cfg.target_assigner, [1408, 1600, 40], 8)
    cpu = SecondTasksCPU(cfg, sd, anchors)
    heads = _random_heads(cfg, cpu.sd, cpu.anchors, 200, 176, 1, 11)
    for h in heads:
        h["cls"] += 1.0
    got = cpu.predict_tasks([(h["box"], h["cls"], h["dir"]) for h in heads])[0]
    assert set(got["label_preds"].tolist()) == {0, 1, 2}
    assert torch.equal(got["label_preds"], got["label_preds"].sort()[0])

    cfg = _shipped("cbgs_lyft.py")
    sd = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).state_dict()
    anchors = anchors_for_tasks(cfg.target_assigner, [2016, 2016, 40], 8)
    cpu = CbgsTasksCPU(cfg, sd, anchors)
    heads = _random_heads(cfg, cpu.sd, cpu.anchors, 252, 252, 1, 12)
    got = cpu.predict_tasks(heads)[0]
    assert set(got["label_preds"].tolist()) <= set(range(7)) and {0, 1, 4} <= set(got["label_preds"].tolist())
    # task 2 (motorcycle / bicycle, labels 2 and 3) restated with the offset: equal
    h, a = heads[2], cpu.anchors[2]
    bx, sc, lb = predict_sample_task(h["cls"][0].reshape(-1, 2), h["box"][0].reshape(-1, 7), h["dir"][0].reshape(-1, 2), a,
                                     cfg.test_cfg, False, direction_offset=0.785)
    m = (got["label_preds"] == 2) | (got["label_preds"] == 3)
    assert torch.equal(got["box3d_lidar"][m], bx) and torch.equal(got["label_preds"][m], lb + 2)
    plain = predict_sample_task(h["cls"][0].reshape(-1, 2), h["box"][0].reshape(-1, 7), h["dir"][0].reshape(-1, 2), a,
                                cfg.test_cfg, False)[0]
    assert not torch.equal(plain, bx), "the direction offset changes some flips on this draw"
