"""PointPillars reader (SURVEY 8f.3): oracle and host mirror vs the reference's own outputs (golden), and the
fused CUDA reader / scatter / end-to-end pipeline vs the oracle."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

PILLAR_VS = [0.16, 0.16, 4.0]
PILLAR_PCR = [0, -39.68, -3, 69.12, 39.68, 1]


def _golden():
    g = load_golden("pillars_kitti_3k")
    sd = {"reader." + k[3:]: torch.from_numpy(g[k]) for k in g if k.startswith("sd.")}
    return g, sd


def _pillars(points):
    from oracle import voxel as ovoxel
    return ovoxel.points_to_voxel(points, np.array(PILLAR_VS, np.float32), np.array(PILLAR_PCR, np.float32), 100, True, 12000)


def test_oracle_reader_matches_reference_golden():
    from oracle.pillars_cpu import pillar_features, pillar_scatter
    g, sd = _golden()
    voxels, coors, nums = _pillars(g["points"])
    assert np.array_equal(coors, g["coors"][:, 1:]) and np.array_equal(nums, g["num_points"])
    assert nums.max() == 100 and (nums == 99).any()          # a full pillar (no padded slot) and a nearly full one
    feats = pillar_features(sd, voxels, nums, g["coors"], PILLAR_VS, PILLAR_PCR)
    assert float(np.abs(feats.numpy() - g["features"]).max()) <= 1e-5
    # the float64 evaluation (the error model's reference, tests/pillar_error_model.py) is the same operation: it
    # differs from the reference's fp32 outputs by fp32 rounding only, a few ulps of their largest magnitude
    feats64 = pillar_features(sd, voxels, nums, g["coors"], PILLAR_VS, PILLAR_PCR, dtype=torch.float64)
    assert feats64.dtype == torch.float64
    ulp = float(np.spacing(np.abs(g["features"]).max()))
    assert float(np.abs(feats64.numpy() - g["features"]).max()) <= 4 * ulp
    canvas = pillar_scatter(torch.from_numpy(g["features"]), g["coors"], 1, 432, 496)
    assert tuple(canvas.shape) == tuple(g["canvas_shape"])
    flat = canvas.numpy().reshape(64, -1)
    assert np.array_equal(np.nonzero(np.abs(flat).sum(0))[0], g["canvas_cols"])
    assert np.allclose([flat.astype(np.float64).sum(), (flat.astype(np.float64) ** 2).sum()], g["canvas_checksum"], rtol=1e-12)


def test_host_mirror_module_matches_reference_golden():
    """The registry module (same parameter names as the reference) loads the reference's state_dict and its
    module-by-module torch forward reproduces the reference output."""
    from det3d.models.readers import PillarFeatureNet
    g, sd = _golden()
    net = PillarFeatureNet(num_input_features=4, num_filters=[64], voxel_size=PILLAR_VS, pc_range=PILLAR_PCR).eval()
    net.load_state_dict({k[len("reader."):]: v for k, v in sd.items()}, strict=True)
    voxels, _, nums = _pillars(g["points"])
    with torch.no_grad():
        out = net.forward_torch(torch.from_numpy(voxels), torch.from_numpy(nums), torch.from_numpy(g["coors"]))
    assert float(np.abs(out.numpy() - g["features"]).max()) <= 1e-5
    if not torch.cuda.is_available():
        from det3d_b200._lib import D3BError
        with pytest.raises((D3BError, RuntimeError, AssertionError)):      # no CPU fallback behind the fused entry
            net.forward_fused(torch.from_numpy(voxels), torch.from_numpy(nums), torch.from_numpy(g["coors"]))


@pytest.mark.gpu
def test_fused_reader_and_scatter_match_golden():
    from det3d.models.readers import PillarFeatureNet, PointPillarsScatter
    from det3d_b200.ops.point_cloud.voxelize import Voxelizer
    g, sd = _golden()
    net = PillarFeatureNet(num_input_features=4, num_filters=[64], voxel_size=PILLAR_VS, pc_range=PILLAR_PCR).eval()
    net.load_state_dict({k[len("reader."):]: v for k, v in sd.items()}, strict=True)
    net = net.cuda()
    vox = Voxelizer(PILLAR_VS, PILLAR_PCR, 100, 12000, want_voxels=True, want_mean=False)(torch.from_numpy(g["points"]).cuda(), None)
    m = int(vox["counts"][0])
    assert m == g["coors"].shape[0]
    assert np.array_equal(vox["coors"][:m].cpu().numpy(), g["coors"])
    with torch.no_grad():
        feats = net(vox["voxels"], vox["num_points"], vox["coors"], n_dev=vox["counts"][1:2])
    assert feats.shape[0] == 12000 and float(feats[m:].abs().max()) == 0.0       # rows past the live count are zero
    assert float(np.abs(feats[:m].cpu().numpy() - g["features"]).max()) <= 1e-4   # north_star tolerance
    with torch.no_grad():
        canvas = PointPillarsScatter(num_input_features=64)(feats, vox["coors"], 1, [432, 496, 1], n_dev=vox["counts"][1:2])
    flat = canvas.cpu().numpy().reshape(64, -1)
    assert np.array_equal(np.nonzero(np.abs(flat).sum(0))[0], g["canvas_cols"])
    assert np.allclose([flat.astype(np.float64).sum(), (flat.astype(np.float64) ** 2).sum()], g["canvas_checksum"], rtol=1e-5)


@pytest.mark.gpu
def test_pointpillars_pipeline_matches_cpu_restatement():
    """BASELINE configs[2] at its stated size: 20k-point clouds, batch 8, uniform clouds that hit the 12000-pillar cap
    (the reference `break`).  Device pipeline vs the CPU restatement stage by stage, STRICT: indices and point lists
    bit-exact, pillar features / RPN / head outputs <= 1e-4 abs, detections identical to the oracle's predict on the same
    head outputs, and the detection set equal to the from-scratch oracle's up to near-tied candidates (counted)."""
    from det3d.models import build_detector
    from det3d.torchie import Config
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud, uniform_cloud
    from oracle.pillars_cpu import PillarsCPU

    cfg = Config.fromfile(os.path.join(ROOT, "configs", "pointpillars_kitti_car.py"))
    torch.manual_seed(0)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 0)
    calibrate_demo_weights_(model, cfg, [uniform_cloud(20000, cfg.voxel_generator.range, 4, 70),
                                         lidar_like_cloud(20000, cfg.voxel_generator.range, 4, 71)], 0, pass_fraction=0.02)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    assert type(pipe.model.fused_bev()).__name__ == "FusedBevStack"        # [3,5,5] RPN with strides + ConvTranspose on own kernels
    cpu = PillarsCPU(cfg, sd, [a.cpu().numpy() for a in pipe._anchors])
    B = 8
    clouds = [uniform_cloud(20000, cfg.voxel_generator.range, 4, 7 + i) if i % 2 == 0 else
              lidar_like_cloud(20000, cfg.voxel_generator.range, 4, 7 + i) for i in range(B)]
    stages = {}
    want = cpu.forward(clouds, stages)
    assert (stages["coors"][:, 0] == 0).sum() == 12000                      # the reference `break` at max_voxels

    packed = pipe.infer_host([torch.from_numpy(c) for c in clouds])
    got = pipe.unpack(packed)
    assert int(pipe.overflow_flag().item()) == 0
    offsets = [20000 * i for i in range(B + 1)]
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    from det3d_b200.ops.point_cloud.voxelize import Voxelizer
    vg = cfg.voxel_generator
    assert pipe._reader_takes_lists and pipe.voxelizer.want_voxels is False     # the serving path never builds [M,100,4]
    full = Voxelizer(vg.voxel_size, vg.range, vg.max_points_in_voxel, vg.max_voxel_num, want_voxels=True, want_mean=False)
    vox = full(pts, offsets)
    m = int(vox["counts"][B])
    assert np.array_equal(vox["coors"][:m].cpu().numpy(), stages["coors"])
    assert np.array_equal(vox["num_points"][:m].cpu().numpy(), stages["nums"])
    assert np.array_equal(vox["voxels"][:m].cpu().numpy(), stages["voxels"])
    with torch.no_grad():
        feats = pipe.model.reader(vox["voxels"], vox["num_points"], vox["coors"], n_dev=vox["counts"][B:B + 1])
        # the reader fused with the voxelizer (point-index lists instead of the voxel tensor): the same bits
        lean = pipe.voxelizer(pts, offsets)
        assert lean["voxels"] is None and torch.equal(lean["coors"][:m], vox["coors"][:m])
        fused = pipe.model.reader.forward_lists(dict(lean["point_lists"], counts=lean["counts"]), lean["num_points"],
                                                lean["coors"], lean["coors"].shape[0], lean["counts"][B:B + 1])
        assert torch.equal(fused[:m], feats[:m])
        planes = pipe.model.backbone.forward_planes(feats, vox["coors"], B, [int(g) for g in pipe.grid_size], n_dev=vox["counts"][B:B + 1])
        preds = {k: v.clone().cpu() for k, v in pipe.model.fused_bev().run(planes)[0].items()}
    assert float((feats[:m].cpu() - stages["pillar_feats"]).abs().max()) <= 1e-4
    assert float(stages["rpn"].abs().max()) < 100.0, "calibration failed: features are not O(1)"
    for key, ref in (("cls_preds", stages["cls"]), ("box_preds", stages["box"]), ("dir_cls_preds", stages["dirs"])):
        e = float((preds[key] - ref).abs().max())
        assert e <= 1e-4, "%s: abs error %g" % (key, e)
    o = cpu.predict(preds["box_preds"], preds["cls_preds"], preds["dir_cls_preds"])
    thr, pre = cfg.test_cfg.score_threshold, cfg.test_cfg.nms.nms_pre_max_size
    total = 0
    for b in range(B):
        assert got[b]["box3d_lidar"].shape == o[b]["box3d_lidar"].shape, "sample %d" % b
        if o[b]["box3d_lidar"].shape[0]:
            assert float((got[b]["box3d_lidar"] - o[b]["box3d_lidar"]).abs().max()) <= 1e-5
            assert float((got[b]["scores"] - o[b]["scores"]).abs().max()) <= 1e-6
        total += o[b]["box3d_lidar"].shape[0]
        sc = torch.sigmoid(stages["cls"][b].reshape(-1))
        top = sc[sc >= thr].sort(descending=True)[0][:pre]
        fragile = int(((top[:-1] - top[1:]) < 2e-6).sum()) + int(((sc - thr).abs() < 2e-6).sum())
        w, gdet = want[b]["box3d_lidar"], got[b]["box3d_lidar"]
        for a_, b_ in ((w, gdet), (gdet, w)):
            miss = 0
            if a_.shape[0]:
                miss = a_.shape[0] if b_.shape[0] == 0 else int(((a_[:, None, :] - b_[None, :, :]).abs().max(-1)[0].min(1)[0] > 1e-3).sum())
            assert miss <= fragile, "sample %d: %d detections differ with %d near-tied candidates" % (b, miss, fragile)
    assert total >= 40
