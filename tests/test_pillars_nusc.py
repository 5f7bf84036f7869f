"""nuScenes PointPillars (examples/point_pillars/configs/nusc_all_point_pillars_mghead_syncbn.py): the stock config
loads unchanged and builds the shipped one's model, its RPN -- whose first deblock is Conv2d(64, 128, 2, stride=2) --
runs on the FP16x3 BEV kernels, and the device pipeline matches the CPU restatement (oracle/pillars_nusc_cpu.py)."""
import copy
import gzip
import json
import os
import re
import warnings

import numpy as np
import pytest
import torch
from torch import nn

from boundary_golden import GOLDEN, decode
from conftest import ROOT

REL = "examples/point_pillars/configs/nusc_all_point_pillars_mghead_syncbn.py"
B = 4                 # samples_per_gpu of the reference config
N_POINTS = 35000


def reference_config():
    """The reference's own file as Config.fromfile parsed it (tests/golden/make_golden_pillars_nusc.py)."""
    from det3d.torchie import Config

    with gzip.open(os.path.join(GOLDEN, "reference_config_pillars_nusc.json.gz"), "rt") as fh:
        return Config(decode(json.load(fh)[REL]), filename=None)


def shipped_config():
    from det3d.torchie import Config

    return Config.fromfile(os.path.join(ROOT, "configs", "pointpillars_nusc.py"))


def test_reference_config_loads_unchanged_and_builds_the_shipped_model():
    from det3d.models import build_detector
    from det3d_b200.ops.spconv.bev import rpn_is_fusable16

    cfg, mine = reference_config(), shipped_config()
    model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    m2 = build_detector(mine.model, train_cfg=None, test_cfg=mine.test_cfg)
    assert type(model).__name__ == "PointPillars" and len(model.bbox_head.tasks) == 6
    a, b = model.state_dict(), m2.state_dict()
    assert list(a) == list(b) and all(a[k].shape == b[k].shape for k in a)
    assert tuple(a["neck.deblocks.0.0.weight"].shape) == (128, 64, 2, 2)
    assert tuple(a["neck.deblocks.2.0.weight"].shape) == (256, 128, 2, 2)      # ConvTranspose2d: [C_in, C_out, k, k]
    assert tuple(a["reader.pfn_layers.0.linear.weight"].shape) == (64, 10)
    for key in ("test_cfg", "voxel_generator", "target_assigner"):
        assert cfg[key].to_dict() == mine[key].to_dict(), key
    assert cfg.assigner.out_size_factor == mine.assigner.out_size_factor == 4
    assert isinstance(model.neck.deblocks[0][0], nn.Conv2d)
    assert rpn_is_fusable16(model.neck) and rpn_is_fusable16(m2.neck)


def test_rpn_is_fusable16_takes_only_the_built_strided_deblocks():
    from det3d_b200.models.necks.rpn import RPN
    from det3d_b200.ops.spconv.bev import rpn_is_fusable16

    def rpn(us):
        return RPN([1, 1], [1, 2], [64, 128], us, [128, 128], 64)

    assert rpn_is_fusable16(rpn([0.5, 1]))            # Conv2d(k = s = 2), then 1x1
    assert rpn_is_fusable16(rpn([0.25, 0.5]))         # Conv2d(k = s = 4), Conv2d(k = s = 2)
    assert rpn_is_fusable16(rpn([1 / 3, 2 / 3]))      # Conv2d(k = s = 3), Conv2d(k = s = round(1.5) = 2)
    assert not rpn_is_fusable16(rpn([0.2, 0.4]))      # Conv2d(k = s = 5) is not built
    for change in (dict(padding=(1, 1)), dict(dilation=(2, 2)), dict(groups=2)):
        r = rpn([0.5, 1])
        conv = r.deblocks[0][0]
        for k, v in change.items():
            setattr(conv, k, v)
        assert not rpn_is_fusable16(r), change
    r = rpn([0.5, 1])
    r.deblocks[0][0] = nn.Conv2d(64, 128, 2, stride=1, bias=False)
    assert not rpn_is_fusable16(r)


# ---------------------------------------------------------------------------------------------------------------------
# on the GPU
# ---------------------------------------------------------------------------------------------------------------------

def _demo_model(cfg):
    from det3d.models import build_detector
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud

    torch.manual_seed(2)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 2)
    calibrate_demo_weights_(model, cfg, [lidar_like_cloud(N_POINTS, cfg.voxel_generator.range, 5, 60 + i) for i in range(2)],
                            2, pass_fraction=0.01)
    return model


@pytest.fixture(scope="module")
def setup():
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import lidar_like_cloud

    cfg = shipped_config()
    model = _demo_model(cfg)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    clouds = [lidar_like_cloud(N_POINTS, cfg.voxel_generator.range, 5, 300 + i) for i in range(B)]
    return cfg, pipe, sd, clouds


def _unmatched(want_boxes, got_boxes, tol):
    if want_boxes.shape[0] == 0:
        return 0
    if got_boxes.shape[0] == 0:
        return int(want_boxes.shape[0])
    d = (want_boxes[:, None, :] - got_boxes[None, :, :]).abs().max(-1)[0]
    return int((d.min(1)[0] > tol).sum())


@pytest.mark.gpu
def test_pipeline_matches_cpu_restatement(setup):
    """Four 35k-point 5-feature clouds, stage by stage against the CPU restatement: voxel indices and counts bit-exact,
    pillar features, RPN and head outputs <= 1e-4 abs (the latter two against the torch modules in float64), device
    detections identical to the oracle's predict on the same head outputs, and the detection set equal to the
    from-scratch oracle's up to near-tied candidates (counted)."""
    from det3d_b200.ops.point_cloud.voxelize import Voxelizer
    from oracle.pillars_nusc_cpu import PillarsNuscCPU

    cfg, pipe, sd, clouds = setup
    model = pipe.model
    bev = model.fused_bev()
    assert type(bev).__name__ == "FusedBevStack"
    cpu = PillarsNuscCPU(cfg, sd, [a.cpu().numpy() for a in pipe._anchors])
    stages = {}
    want = cpu.forward(clouds, stages)

    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    offsets = [N_POINTS * i for i in range(B + 1)]
    det = pipe.forward_device(pts, offsets)
    assert det["boxes"].shape == (B, 6 * 83, 9)
    got = pipe.unpack(pipe.pack(det).cpu())
    assert int(pipe.overflow_flag().item()) == 0

    vg = cfg.voxel_generator
    full = Voxelizer(vg.voxel_size, vg.range, vg.max_points_in_voxel, vg.max_voxel_num, want_voxels=True, want_mean=False)
    vox = full(pts, offsets)
    m = int(vox["counts"][B])
    assert m == stages["coors"].shape[0] and int(vox["counts"][0]) > 5000
    assert np.array_equal(vox["coors"][:m].cpu().numpy(), stages["coors"])
    assert np.array_equal(vox["num_points"][:m].cpu().numpy(), stages["nums"])
    grid = [int(g) for g in pipe.grid_size]
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            feats = model.reader(vox["voxels"], vox["num_points"], vox["coors"], n_dev=vox["counts"][B:B + 1])
            dense = model.backbone(feats, vox["coors"], B, grid, n_dev=vox["counts"][B:B + 1])
            planes = model.backbone.forward_planes(feats, vox["coors"], B, grid, n_dev=vox["counts"][B:B + 1])
            preds = [{k: v.clone() for k, v in d.items()} for d in bev.run(planes)]
            rpn = bev._bufs[("concat",)].to_f32().permute(0, 3, 1, 2)
            neck64 = copy.deepcopy(model.neck).double()
            rpn64 = neck64(dense.double())
            ref = copy.deepcopy(model.bbox_head).double()(rpn64)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    assert float((feats[:m].cpu() - stages["pillar_feats"]).abs().max()) <= 1e-4
    assert float(stages["dense"].abs().max()) < 100.0 and float(stages["rpn"].abs().max()) < 100.0, \
        "calibration failed: features are not O(1)"
    e = float((rpn.double() - rpn64).abs().max())
    assert e <= 1e-4, "RPN output: abs error %g vs the float64 modules" % e
    for t in range(6):
        assert set(preds[t]) == set(ref[t])
        for key in ref[t]:
            e = float((preds[t][key].double() - ref[t][key]).abs().max())
            assert e <= 1e-4, "task %d %s: abs error %g vs the float64 modules" % (t, key, e)

    heads = [{"box": p["box_preds"].cpu(), "cls": p["cls_preds"].cpu()} for p in preds]
    o = cpu.predict_tasks(heads)
    thr, pre = cfg.test_cfg.score_threshold, cfg.test_cfg.nms.nms_pre_max_size
    total = 0
    for b in range(B):
        gb, wb = got[b]["box3d_lidar"], o[b]["box3d_lidar"]
        assert gb.shape == wb.shape, "sample %d: %d detections vs %d from the oracle" % (b, gb.shape[0], wb.shape[0])
        if wb.shape[0]:
            assert float((gb - wb).abs().max()) <= 1e-5
            assert float((got[b]["scores"] - o[b]["scores"]).abs().max()) <= 1e-6
        assert torch.equal(got[b]["label_preds"], o[b]["label_preds"])
        total += wb.shape[0]
        fragile = 0
        for h in stages["heads"]:
            sc = torch.sigmoid(h["cls"][b].reshape(-1))
            top = sc[sc >= thr].sort(descending=True)[0][:pre]
            fragile += int(((top[:-1] - top[1:]) < 2e-6).sum()) + int(((sc - thr).abs() < 2e-6).sum())
        w = want[b]["box3d_lidar"]
        missing, extra = _unmatched(w, gb, 1e-3), _unmatched(gb, w, 1e-3)
        assert missing <= fragile and extra <= fragile, \
            "sample %d: %d missing, %d extra with %d near-tied candidates" % (b, missing, extra, fragile)
    assert total >= 40


_VENDOR_KERNEL = re.compile(r"cudnn|cublas|xmma|cutlass|gemm|winograd|convolve|fprop|dgrad|wgrad|fft[12]d|conv2d",
                            re.IGNORECASE)


@pytest.mark.gpu
def test_forward_launches_no_vendor_convolution(setup):
    """One eager forward under torch.profiler: no cuDNN / cuBLAS convolution or GEMM kernel; every convolution is one of
    the project's own kernels (d3b::...)."""
    from torch.profiler import ProfilerActivity, profile

    cfg, pipe, sd, clouds = setup
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    offsets = [N_POINTS * i for i in range(B + 1)]
    pipe.forward_device(pts, offsets)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pipe.forward_device(pts, offsets)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    ours = {n for n in names if "d3b" in n}
    assert any("bev_conv16" in n for n in ours), sorted(names)
    vendor = sorted(n for n in names - ours if _VENDOR_KERNEL.search(n))
    assert not vendor, "vendor convolution / GEMM kernels on the forward: %s" % vendor


@pytest.mark.gpu
def test_graph_replay_and_batch_composition(setup):
    """forward_graphed returns the bits of forward_device, and a cloud's detections do not depend on its batch mates."""
    cfg, pipe, sd, clouds = setup
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    offsets = [N_POINTS * i for i in range(B + 1)]
    eager = pipe.pack(pipe.forward_device(pts, offsets)).clone()
    graphed = pipe.forward_graphed(pts, offsets).clone()
    assert torch.equal(eager, graphed)
    c = [torch.from_numpy(x).pin_memory() for x in clouds]
    alone = pipe.infer_host([c[0]]).clone()
    mixed = pipe.infer_host([c[2], c[0], c[3]]).clone()
    assert int((alone[0, :, -1] > 0.5).sum()) > 0
    assert torch.equal(alone[0], mixed[1])
    assert torch.equal(alone[0], eager[0].cpu())


@pytest.mark.gpu
def test_overflow_in_the_strided_deblock_reruns_on_the_torch_modules(setup):
    """Deblock 0's folded BatchNorm on one channel set to scale 0, shift 65510: every output of that channel is 65510
    exactly, past the f16 range (its hi plane still rounds to the finite 65504).  The channel's head weights are zero,
    so the detections stay finite.  The Conv2d(k = s = 2) epilogue raises the flag, infer_host warns, switches to
    tf32x3 and re-runs through the torch modules; the result is finite and the flag clear."""
    from det3d.models import build_detector
    from det3d_b200.apis import InferencePipeline

    cfg, _pipe, sd, clouds = setup
    model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    model.load_state_dict(sd)
    model.eval()
    with torch.no_grad():
        bn = model.neck.deblocks[0][1]                        # deblock 0 writes concat channels [0, 128)
        bn.weight[7] = 0.0
        bn.bias[7] = 65510.0
        for task in model.bbox_head.tasks:
            for conv in (task.conv_box, task.conv_cls):
                conv.weight[:, 7] = 0.0
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    assert pipe.model.fused_bev() is not None and pipe.model.math == "fp16x3"
    cloud = torch.from_numpy(clouds[1]).pin_memory()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        packed = pipe.infer_host([cloud]).clone()
    assert any("f16 range" in str(w.message) for w in caught), [str(w.message) for w in caught]
    assert pipe.model.math == "tf32x3"
    assert bool(torch.isfinite(packed).all())
    assert int(pipe.overflow_flag().item()) == 0
    assert int((packed[0, :, -1] > 0.5).sum()) > 0
