"""End-to-end SECOND forward (config 2 of BASELINE.json) on the GPU vs the CPU restatement of
the reference path (oracle/second_cpu.py), stage by stage."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup():
    from det3d.models import build_detector
    from det3d.torchie import Config
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud
    from oracle.second_cpu import SecondCPU

    cfg = Config.fromfile(os.path.join(ROOT, "configs", "second_kitti_car.py"))
    torch.manual_seed(0)
    # random weights made to behave like trained ones: BatchNorm statistics matched to the activations (features stay
    # O(1), so the north_star's 1e-4 ABSOLUTE tolerance is meaningful), ~3 % of the anchors above the 0.3 threshold
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 0)
    calib = [lidar_like_cloud(20000, cfg.voxel_generator.range, 4, 900 + i) for i in range(2)]
    calibrate_demo_weights_(model, cfg, calib, 0)
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    cpu = SecondCPU(cfg, model.state_dict(), [a.cpu().numpy() for a in pipe._anchors])
    return cfg, pipe, cpu


def _unmatched(want_boxes, got_boxes, tol):
    """Number of `want` rows without a `got` row within `tol` (max-abs over the box)."""
    if want_boxes.shape[0] == 0:
        return 0
    if got_boxes.shape[0] == 0:
        return int(want_boxes.shape[0])
    d = (want_boxes[:, None, :] - got_boxes[None, :, :]).abs().max(-1)[0]
    return int((d.min(1)[0] > tol).sum())


@pytest.mark.parametrize("dist,n", [("lidar", 20000), ("uniform", 20000)])
def test_forward_matches_cpu_restatement(setup, dist, n):
    """BASELINE configs[1], stage by stage against the CPU restatement of the reference path, STRICT:
    indices bit-exact, features <= 1e-4 abs, head outputs <= 1e-4 abs, and the detection list equal to the oracle's."""
    from det3d_b200.utils.synthetic import lidar_like_cloud, uniform_cloud
    cfg, pipe, cpu = setup
    pts = (lidar_like_cloud if dist == "lidar" else uniform_cloud)(n, cfg.voxel_generator.range, 4, 1)
    stages = {}
    want = cpu.forward([pts], stages)[0]

    dev_pts = torch.from_numpy(pts).cuda()
    vox = pipe.voxelizer(dev_pts, [0, n])
    m = int(vox["counts"][0])
    assert m == stages["coors"].shape[0]
    assert np.array_equal(vox["coors"][:m].cpu().numpy(), stages["coors"])                 # bit-exact indices
    assert np.array_equal(vox["num_points"][:m].cpu().numpy(), stages["nums"])
    feats_cpu = stages["voxels"].sum(1) / stages["nums"][:, None].astype(np.float32)
    assert np.allclose(vox["mean"][:m].cpu().numpy(), feats_cpu, rtol=0, atol=1e-6)

    model = pipe.model
    grid = [int(g) for g in pipe.grid_size]
    with torch.no_grad():
        dense = model.backbone(vox["mean"], vox["coors"], 1, grid, n_dev=vox["counts"][1:2]).cpu()
        planes = model.backbone.forward_planes(vox["mean"], vox["coors"], 1, grid, n_dev=vox["counts"][1:2])
        preds = model.fused_bev().run(planes)[0]
        heads = {k: v.clone().cpu() for k, v in preds.items()}
    assert float(stages["dense"].abs().max()) < 100.0, "calibration failed: features are not O(1)"
    err = float((dense - stages["dense"]).abs().max())
    print("%s: dense max |x| %.3g, abs error %.3g" % (dist, float(stages["dense"].abs().max()), err))
    assert err <= 1e-4, "dense feature map: abs error %g" % err                              # north_star: 1e-4 ABS
    for key, ref in (("cls_preds", stages["cls"]), ("box_preds", stages["box"]), ("dir_cls_preds", stages["dirs"])):
        e = float((heads[key] - ref).abs().max())
        print("%s: %s max |x| %.3g, abs error %.3g" % (dist, key, float(ref.abs().max()), e))
        assert e <= 1e-4, "%s: abs error %g" % (key, e)

    # the encoder is deterministic: two runs of the whole path give the same bits
    p1 = pipe.pack(pipe.forward_device(dev_pts, [0, n])).clone()
    p2 = pipe.pack(pipe.forward_device(dev_pts, [0, n])).clone()
    assert torch.equal(p1, p2)
    assert int(pipe.overflow_flag().item()) == 0
    got = pipe.unpack(p1.cpu())[0]

    # (a) device predict == the ORACLE's predict (mg_head.py:697-1085 restated on the CPU) on the same head outputs:
    #     same detections, same order
    o = cpu.predict(heads["box_preds"], heads["cls_preds"], heads["dir_cls_preds"])[0]
    assert o["box3d_lidar"].shape[0] >= 10, "degenerate workload: no detections"
    assert got["box3d_lidar"].shape == o["box3d_lidar"].shape
    assert float((got["box3d_lidar"] - o["box3d_lidar"]).abs().max()) <= 1e-5            # libm vs CUDA exp / atan2 ulps
    assert float((got["scores"] - o["scores"]).abs().max()) <= 1e-6
    # (b) against the oracle run from the raw points: the detection SET is identical, except where two candidates'
    #     scores are closer than the 1e-6-level difference between the two implementations (counted, not ignored)
    sc = torch.sigmoid(stages["cls"].reshape(-1))
    top = sc[sc >= cfg.test_cfg.score_threshold].sort(descending=True)[0][: cfg.test_cfg.nms.nms_pre_max_size]
    fragile = int(((top[:-1] - top[1:]) < 2e-6).sum()) + int(((sc - cfg.test_cfg.score_threshold).abs() < 2e-6).sum())
    missing = _unmatched(want["box3d_lidar"], got["box3d_lidar"], 1e-3)
    extra = _unmatched(got["box3d_lidar"], want["box3d_lidar"], 1e-3)
    assert want["box3d_lidar"].shape[0] >= 10
    assert missing <= fragile and extra <= fragile, "detections differ (%d missing, %d extra) with only %d near-tied candidates" % (
        missing, extra, fragile)


def test_tf32x3_fallback_path_and_overflow_guard(setup):
    """The tf32x3 kernels stay selectable (`set_math("tf32x3")`) and are where a forward is re-run when a feature
    leaves the f16 range: same detections as the FP16x3 path, the same bits run to run, and the guard trips (instead of
    saturating) on huge inputs."""
    from det3d_b200.ops.spconv import conv16
    from det3d_b200.utils.synthetic import lidar_like_cloud
    cfg, pipe, cpu = setup
    cloud = torch.from_numpy(lidar_like_cloud(12000, cfg.voxel_generator.range, 4, 77))
    a = pipe.unpack(pipe.infer_host([cloud]).clone())[0]
    pipe.model.set_math("tf32x3")
    try:
        packed = pipe.infer_host([cloud]).clone()
        again = pipe.infer_host([cloud]).clone()
    finally:
        pipe.model.set_math("fp16x3")
    assert torch.equal(packed, again)        # output-stationary kernels: fixed summation order, no atomics
    b = pipe.unpack(packed)[0]
    # the tf32x3 output-stationary kernels chain hundreds of truncating tensor-core accumulations without correction
    # (relative bias -1.4e-6 for a 3x3x3 C_in 64 sparse layer, -7.4e-6 for a 3x3 C_in 128 dense one, on an H100 80GB HBM3
    # at 400 W: profiles/h100_trunc_bias.txt; bounded in
    # test_conv_error_model_gpu.py::test_tf32x3_output_stationary_beyond_f16_range):
    # near-tied candidates may swap, so this fallback is only required to agree closely
    n = a["box3d_lidar"].shape[0]
    assert n >= 5 and _unmatched(a["box3d_lidar"], b["box3d_lidar"], 2e-3) <= max(1, n // 10)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    conv16.Planes.from_f32(torch.full((4, 8), 7.0e4, device="cuda"), flag)
    assert int(flag.item()) == 1


def test_host_api_and_batching(setup):
    from det3d_b200.utils.synthetic import lidar_like_cloud
    cfg, pipe, cpu = setup
    clouds = [torch.from_numpy(lidar_like_cloud(6000 + 500 * i, cfg.voxel_generator.range, 4, 10 + i)).pin_memory()
              for i in range(3)]
    packed = pipe.infer_host(clouds)
    assert packed.shape[0] == 3 and packed.shape[2] == 10
    singles = [pipe.infer_host([c]).clone() for c in clouds]
    for b in range(3):
        a, s = pipe.unpack(packed)[b], pipe.unpack(singles[b])[0]
        assert a["box3d_lidar"].shape == s["box3d_lidar"].shape
        assert torch.allclose(a["box3d_lidar"], s["box3d_lidar"], atol=1e-4)
        assert torch.allclose(a["scores"], s["scores"], atol=1e-5)


def test_detections_do_not_depend_on_batch_composition(setup):
    """A cloud's detections are the same BITS whatever else shares its batch (sparse tiles straddle clouds: the
    accumulation order of a row must not depend on its tile mates) -- what makes the sharded multi-GPU run
    (tools/dist_infer.py --check) reproduce the single-rank result exactly."""
    from det3d_b200.utils.synthetic import lidar_like_cloud
    cfg, pipe, cpu = setup
    c = [torch.from_numpy(lidar_like_cloud(9000 + 700 * i, cfg.voxel_generator.range, 4, 40 + i)).pin_memory() for i in range(4)]
    alone = pipe.infer_host([c[0]]).clone()
    ab = pipe.infer_host([c[0], c[1]]).clone()
    cad = pipe.infer_host([c[2], c[0], c[3]]).clone()
    assert int((alone[0, :, -1] > 0.5).sum()) > 0
    assert torch.equal(alone[0], ab[0])
    assert torch.equal(alone[0], cad[1])


def test_model_predict_api(setup):
    """VoxelNet.forward(example, return_loss=False) with reference-style inputs (voxels [M,5,4])."""
    from det3d.core.input.voxel_generator import VoxelGenerator
    from det3d_b200.utils.synthetic import lidar_like_cloud
    cfg, pipe, cpu = setup
    vg = cfg.voxel_generator
    gen = VoxelGenerator(vg.voxel_size, vg.range, vg.max_points_in_voxel, vg.max_voxel_num)
    pts = lidar_like_cloud(5000, vg.range, 4, 3)
    voxels, coors, num = gen.generate(pts)
    coors = np.concatenate([np.zeros((coors.shape[0], 1), np.int32), coors], 1)           # collate_kitti
    example = dict(voxels=torch.from_numpy(voxels).cuda(), coordinates=torch.from_numpy(coors).cuda(),
                   num_points=torch.from_numpy(num).cuda(), num_voxels=torch.tensor([voxels.shape[0]]),
                   shape=[gen.grid_size], anchors=pipe.anchors(1))
    with torch.no_grad():
        out = pipe.model(example, return_loss=False)
    assert len(out) == 1 and set(out[0]) >= {"box3d_lidar", "scores", "label_preds"}
    ref = pipe.unpack(pipe.infer_host([torch.from_numpy(pts)]))[0]
    assert out[0]["box3d_lidar"].shape[0] == ref["box3d_lidar"].shape[0]
    assert torch.allclose(out[0]["box3d_lidar"].cpu(), ref["box3d_lidar"], atol=1e-4)


def test_fused_bev_path_matches_cudnn_path(setup):
    """RPN + heads through the channels-last wgmma kernels vs the module's torch/cuDNN fp32 forward."""
    from det3d_b200.utils.synthetic import lidar_like_cloud
    cfg, pipe, cpu = setup
    model = pipe.model
    assert model.fused_bev() is not None
    pts = torch.from_numpy(lidar_like_cloud(20000, cfg.voxel_generator.range, 4, 5)).cuda()
    vox = pipe.voxelizer(pts, [0, 20000])
    grid = [int(g) for g in pipe.grid_size]
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            planes = model.backbone.forward_planes(vox["mean"], vox["coors"], 1, grid, n_dev=vox["counts"][1:2])
            dense = model.backbone(vox["mean"], vox["coors"], 1, grid, n_dev=vox["counts"][1:2])
            # the same values in the two layouts, bit for bit (the FP16x3 encoder is deterministic)
            assert torch.equal(planes.to_f32().permute(0, 3, 1, 2), dense)
            fused = model.fused_bev().run(planes)
            ref = model.bbox_head(model.neck(dense))
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    for key in ("box_preds", "cls_preds", "dir_cls_preds"):
        a, r = fused[0][key], ref[0][key]
        assert a.shape == r.shape
        # fp32 cuDNN vs 3xTF32: both fp32-accurate; compare relative to the tensor's magnitude
        assert float((a - r).abs().max()) <= 1e-4 * max(1.0, float(r.abs().max())), key


def test_cbgs_nuscenes_config():
    """BASELINE configs[3] shape: CBGS (SpMiddleResNetFHD with residual blocks, two-block RPN with a stride-2 block and a
    ConvTranspose deblock, 6 task heads, 9-dim boxes with angle-vector encoding), 35k-point 5-feature clouds, 4 clouds
    per GPU as in the 32-over-8 sharding.  RPN + heads run on the FP16x3 TMA kernels and are checked against the module's
    fp32 cuDNN forward; the device predict is checked against the CPU restatement of MultiGroupHead.predict on the same
    head outputs: identical detections.  (The sparse encoder at this shape is pinned against the float64 oracle, stage by
    stage and layer by layer, in test_encoder_deployed_gpu; the 32-cloud multi-GPU run in test_multi_gpu.)"""
    from det3d.models import build_detector
    from det3d.torchie import Config
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud
    from oracle.predict_cpu import predict_sample_task

    cfg = Config.fromfile(os.path.join(ROOT, "configs", "cbgs_nusc.py"))
    torch.manual_seed(1)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 1)
    calibrate_demo_weights_(model, cfg, [lidar_like_cloud(35000, cfg.voxel_generator.range, 5, 50 + i) for i in range(2)], 1,
                            pass_fraction=0.01)
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    B = 4
    assert type(pipe.model.fused_bev()).__name__ == "FusedBevStack"        # strided RPN + ConvTranspose on own kernels
    clouds = [lidar_like_cloud(35000, cfg.voxel_generator.range, 5, s) for s in range(B)]
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    offsets = [35000 * i for i in range(B + 1)]
    det = pipe.forward_device(pts, offsets)
    assert det["boxes"].shape == (B, 6 * 83, 9) and int(det["valid"].sum()) > 20
    got = pipe.unpack(pipe.pack(det).cpu())
    assert int(pipe.overflow_flag().item()) == 0

    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            vox = pipe.voxelizer(pts, offsets)
            counts = vox["counts"].cpu().numpy()
            assert counts[B] == counts[:B].sum() and counts[0] > 10000
            grid = [int(g) for g in pipe.grid_size]
            planes = model.backbone.forward_planes(vox["mean"], vox["coors"], B, grid, n_dev=vox["counts"][B:B + 1])
            dense = model.backbone(vox["mean"], vox["coors"], B, grid, n_dev=vox["counts"][B:B + 1])
            assert torch.equal(planes.to_f32().permute(0, 3, 1, 2), dense)
            preds = [{k: v.clone() for k, v in d.items()} for d in model.fused_bev().run(planes)]
            # reference: the torch modules themselves (necks/rpn.py, mg_head.py) evaluated in float64 -- cuDNN's fp32
            # algorithms (Winograd / FFT picks) are themselves ~1e-4 away from it after 13 layers, reported below
            import copy
            ref = copy.deepcopy(model.bbox_head).double()(copy.deepcopy(model.neck).double()(dense.double()))
            ref32 = model.bbox_head(model.neck(dense))
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    assert float(dense.abs().max()) < 100.0
    worst, worst32 = 0.0, 0.0
    for t in range(6):
        assert set(preds[t]) == set(ref[t])
        for key in ref[t]:
            e = float((preds[t][key].double() - ref[t][key]).abs().max())
            worst, worst32 = max(worst, e), max(worst32, float((ref32[t][key].double() - ref[t][key]).abs().max()))
            assert e <= 1e-4, "task %d %s: abs error %g vs the float64 modules" % (t, key, e)
    print("cbgs RPN+heads max abs error vs float64: FP16x3 kernels %.3g, fp32 cuDNN %.3g" % (worst, worst32))

    flag = 0
    want = [dict(b=[], s=[], l=[]) for _ in range(B)]
    for task_id, p in enumerate(preds):
        anchors = pipe._anchors[task_id].cpu()
        n_cls = model.bbox_head.num_classes[task_id]
        for b in range(B):
            bx, sc, lb = predict_sample_task(p["cls_preds"][b].reshape(-1, n_cls).cpu(), p["box_preds"][b].reshape(-1, 10).cpu(),
                                             p["dir_cls_preds"][b].reshape(-1, 2).cpu() if "dir_cls_preds" in p else None,
                                             anchors, cfg.test_cfg, True)
            want[b]["b"].append(bx); want[b]["s"].append(sc); want[b]["l"].append(lb + flag)
        flag += n_cls
    total = 0
    for b in range(B):
        wb, ws, wl = torch.cat(want[b]["b"]), torch.cat(want[b]["s"]), torch.cat(want[b]["l"])
        gb, gs, gl = got[b]["box3d_lidar"], got[b]["scores"], got[b]["label_preds"]
        assert gb.shape == wb.shape, "sample %d: %d detections vs %d from the oracle" % (b, gb.shape[0], wb.shape[0])
        assert float((gb - wb).abs().max()) <= 1e-5 and float((gs - ws).abs().max()) <= 1e-6 and torch.equal(gl, wl)
        total += wb.shape[0]
    assert total >= 40


def test_fused_predict_kernels_match_torch_ops(setup):
    """d3b_predict_task (radix-select top-k, decode of the selected anchors, NMS, finalize) vs the same
    algorithm written with torch ops: identical boxes / scores / labels / validity."""
    from det3d_b200.utils.synthetic import lidar_like_cloud
    cfg, pipe, cpu = setup
    model = pipe.model
    for seed in (3, 4):
        pts = torch.from_numpy(lidar_like_cloud(20000, cfg.voxel_generator.range, 4, seed)).cuda()
        vox = pipe.voxelizer(pts, [0, 20000])
        with torch.no_grad():
            planes = model.backbone.forward_planes(vox["mean"], vox["coors"], 1, [int(g) for g in pipe.grid_size],
                                                   n_dev=vox["counts"][1:2])
            preds = model.fused_bev().run(planes)
            example = dict(anchors=pipe.anchors(1))
            a = model.bbox_head.predict_device(example, preds, cfg.test_cfg)
            t = model.bbox_head.predict_device(example, preds, cfg.test_cfg, use_torch_ops=True)
        va, vt = a["valid"][0], t["valid"][0]
        assert int(vt.sum()) >= 10
        assert torch.equal(va, vt)
        assert torch.equal(a["boxes"][0][va], t["boxes"][0][vt])          # same fp32 op sequence -> bit-identical
        assert torch.equal(a["scores"][0][va], t["scores"][0][vt])
        assert torch.equal(a["labels"][0][va], t["labels"][0][vt])


@pytest.mark.parametrize("hw", [3000, 40000])
def test_topk_handles_ties_and_constants(hw):
    """All-equal scores (the degenerate case): lowest anchor indices win, deterministically.  hw=3000: the whole
    pivot bin is sorted in shared memory; hw=40000: it exceeds the sort capacity -> radix select over composites."""
    import ctypes as C
    from det3d_b200 import _lib
    B, na = 2, 2
    cls = torch.zeros((B, 1, hw, na), device="cuda")
    cls[1] = -5.0
    cls[1, 0, 100:110, :] = 5.0
    box = torch.zeros((B, 1, hw, na * 7), device="cuda")
    anchors = torch.rand((hw * na, 7), device="cuda") * 10 + 1
    q = _lib.PredictParams()
    q.cls, q.cls_row_stride, q.cls_col0 = cls.data_ptr(), na, 0
    q.box, q.box_row_stride, q.box_col0 = box.data_ptr(), na * 7, 0
    q.dir = None
    q.anchors = anchors.data_ptr()
    q.batch, q.hw, q.na, q.n_cls, q.code, q.nd = B, hw, na, 1, 7, 7
    q.use_rotate_nms, q.pre_max, q.post_max = 1, 1000, 1000
    q.nms_iou_threshold, q.score_threshold = 2.0, 0.3       # IoU never reaches 2 -> NMS keeps every candidate
    q.has_range = 0
    ws = torch.empty(_lib.lib().d3b_predict_workspace_bytes(C.byref(q)), dtype=torch.uint8, device="cuda")
    packed = torch.zeros((B, 1000, 10), device="cuda")
    counts = torch.zeros(B, dtype=torch.int32, device="cuda")
    st = _lib.lib().d3b_predict_task(C.byref(q), packed.data_ptr(), 1000, 0, counts.data_ptr(), ws.data_ptr(), ws.numel(),
                                    torch.cuda.current_stream().cuda_stream)
    _lib.check(st)
    assert counts.tolist() == [1000, 20]                    # sample 0: 0.5 >= 0.3 for all; sample 1: only the 20 raised logits
    got0 = packed[0, :, :3]
    assert torch.equal(got0, anchors[:1000, :3])            # ties -> first 1000 anchors, in index order
    assert torch.equal(packed[1, :20, :3], anchors[200:220, :3])
