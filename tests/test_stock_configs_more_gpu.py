"""SECOND KITTI three-class (configs/second_kitti_all.py) and CBGS Lyft (configs/cbgs_lyft.py) end to end on the device
path, at their deployed shapes, held to the criteria of test_encoder_deployed_gpu / test_e2e_gpu:

* KITTI three-class: B = 2 clouds of 20k LiDAR-like points; three single-class tasks, 60 fused head columns.
* Lyft: B = 2, a 60k-point LiDAR-like cloud and a 100k-point cloud spread over the whole +-100.8 m range that fills
  max_voxel_num = 80000 (the voxelizer's `break`).  The reader keeps 3 of the 4 point columns, read in place by the
  first sparse layer (SubM 3 -> 16); the BEV map is 252 x 252 x 256, the RPN runs at 252^2 and 126^2 (widths that are not
  multiples of the 8-column tile), the ConvTranspose deblock writes 126 -> 252, and tasks 2 and 4 have 254,016 anchors.

Per config: voxels, every level's coordinates, neighbour map and tile masks bit-exact; the BEV map within 1e-4 abs of the
float64 encoder; RPN and heads within 1e-4 of the float64 modules; detections equal to the oracle predict on the device
heads and to the from-scratch oracle (tests/oracle_tasks.py) up to counted near-ties; graph replay bit-identical to the
eager forward; detections independent of batch composition; no cuDNN / cuBLAS kernel in the forward; an injected f16
overflow re-runs and still matches the oracle.  Plus: every Lyft encoder layer against the FP16x3 error model on its
deployed rulebook, the dense layers at 252^2 / 126^2 against theirs, and d3b_predict_task at A = 254,016.
"""
import copy
import os
import re
import warnings

import numpy as np
import pytest
import torch

import test_conv_error_model_gpu as tem
import test_encoder_deployed_gpu as ted
import test_f16_guard_gpu as tfg
import test_predict_task_gpu as tpt
from conftest import ROOT

pytestmark = pytest.mark.gpu

TOL = 1e-4
N_LYFT = (60000, 100000)
_VENDOR_KERNEL = re.compile(r"cudnn|cublas|xmma|cutlass|gemm|winograd|convolve|fprop|dgrad|wgrad|fft[12]d|conv2d",
                            re.IGNORECASE)


def _config(name):
    from det3d.torchie import Config
    return Config.fromfile(os.path.join(ROOT, "configs", name))


def _clouds(name, cfg):
    from det3d_b200.utils.synthetic import lidar_like_cloud, uniform_cloud
    r = cfg.voxel_generator.range
    if name == "kitti_all":
        return [lidar_like_cloud(20000, r, 4, 1), lidar_like_cloud(20000, r, 4, 2)]
    return [lidar_like_cloud(N_LYFT[0], r, 4, 3), uniform_cloud(N_LYFT[1], r, 4, 4)]


def _model(name):
    """Seeded demo weights with BatchNorm statistics and head scales calibrated on two clouds (as test_e2e_gpu)."""
    from det3d.models import build_detector
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud
    from oracle_tasks import CbgsTasksCPU, SecondTasksCPU
    cfg = _config("second_kitti_all.py" if name == "kitti_all" else "cbgs_lyft.py")
    seed = 0 if name == "kitti_all" else 1
    torch.manual_seed(seed)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), seed)
    n = 20000 if name == "kitti_all" else 80000
    calibrate_demo_weights_(model, cfg, [lidar_like_cloud(n, cfg.voxel_generator.range, 4, 900 + i) for i in range(2)],
                            seed, pass_fraction=0.03 if name == "kitti_all" else 0.01)
    return cfg, model, SecondTasksCPU if name == "kitti_all" else CbgsTasksCPU


def _run(cfg, pipe, cpu, name):
    from det3d_b200.ops.spconv import conv16
    clouds = _clouds(name, cfg)
    B = len(clouds)
    stages = {}
    want = cpu.forward(clouds, stages)
    dense64, levels64, _ = cpu.backbone(stages["voxels"], stages["coors"], stages["nums"], B, dtype=torch.float64,
                                        return_levels=True)
    model = pipe.model
    grid = [int(g) for g in pipe.grid_size]
    with torch.no_grad():
        pts = torch.from_numpy(np.concatenate(clouds)).cuda()
        offsets = np.cumsum([0] + [c.shape[0] for c in clouds]).tolist()
        vox = pipe.voxelizer(pts, offsets)
        counts = vox["counts"].clone()
        mean = vox["mean"].clone()
        feats = model.reader(mean, None)                # the deployed read: a strided view for Lyft's 3 columns
        planes = model.backbone.forward_planes(feats, vox["coors"], B, grid, n_dev=counts[B:B + 1])
        bev = planes.to_f32()
        kept = conv16.Planes(planes.shape, "cuda")
        kept.buf.copy_(planes.buf)
        steps = ted._snapshot(model.backbone.fused())
        fb = model.fused_bev()
        preds = [{k: v.clone() for k, v in d.items()} for d in fb.run(planes)]
        rpn = fb._bufs[("concat",)].to_f32() if ("concat",) in fb._bufs else None
        got = pipe.unpack(pipe.pack(pipe.forward_device(pts, offsets)).cpu())
    return dict(name=name, B=B, clouds=clouds, samples=None, stages=stages, want=want, dense64=dense64,
                levels64=levels64, counts=counts.cpu().numpy(), coors=vox["coors"][:int(counts[B])].cpu().numpy(),
                mean=mean[:int(counts[B])].cpu(), feats=feats, planes=kept, bev=bev, steps=steps, preds=preds,
                rpn=rpn, got=got, pts=pts, offsets=offsets, flag=int(pipe.overflow_flag().item()))


@pytest.fixture(scope="module")
def deployed():
    """config name -> (cfg, pipe, oracle, run), each built and run once."""
    from det3d_b200.apis import InferencePipeline
    cache = {}

    def get(name):
        if name not in cache:
            cfg, model, oracle = _model(name)
            sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
            pipe = InferencePipeline(cfg, model=model, device="cuda")
            cpu = oracle(cfg, sd, [a.cpu().numpy() for a in pipe._anchors])
            cache[name] = (cfg, pipe, cpu, sd, _run(cfg, pipe, cpu, name))
        return cache[name]
    return get


CONFIGS = ["kitti_all", "lyft"]


def test_shapes_at_deployment(deployed):
    """The shapes of the issue's table: anchors per task, fused head columns, BEV grid."""
    cfg, pipe, _cpu, _sd, run = deployed("kitti_all")
    assert [int(a.shape[0]) for a in pipe._anchors] == [70400] * 3
    assert tuple(run["planes"].shape) == (2, 200, 176, 128)
    cfg, pipe, _cpu, _sd, run = deployed("lyft")
    assert [int(a.shape[0]) for a in pipe._anchors] == [127008, 127008, 254016, 127008, 254016]
    assert all(a.shape[1] == 7 for a in pipe._anchors)
    assert tuple(run["planes"].shape) == (2, 252, 252, 256)
    assert run["feats"].shape[1] == 3 and run["feats"].stride(0) == 4, "the reader must not copy the mean"
    assert run["rpn"] is not None and tuple(run["rpn"].shape) == (2, 252, 252, 512)


@pytest.mark.parametrize("name", CONFIGS)
def test_stage_by_stage_vs_float64_oracle(deployed, name):
    from oracle.predict_cpu import predict_sample_task
    cfg, pipe, cpu, _sd, run = deployed(name)
    B, model = run["B"], pipe.model
    ted._check_voxels(run)
    per_sample = run["counts"][:B]
    print("%s: voxels per sample %s" % (name, per_sample.tolist()))
    if name == "lyft":
        assert per_sample[1] == cfg.voxel_generator.max_voxel_num and per_sample[0] < cfg.voxel_generator.max_voxel_num
    ted._check_levels(run)

    dense64 = run["dense64"].cuda()
    assert float(dense64.abs().max()) < 100.0, "calibration failed: features are not O(1)"
    err = float((run["bev"].permute(0, 3, 1, 2).double() - dense64).abs().max())
    errs = ted._chain_errors(run)
    print("%s: BEV max abs error vs float64 %.3g; per layer %s" % (name, err, " ".join("%.2g" % e for e in errs)))
    assert err <= TOL, "BEV map: abs error %g vs the float64 oracle" % err

    # RPN + heads: on the device's own map vs the float64 modules (the dense kernels alone), and on the oracle's map
    # (the whole chain; held to the fp32 oracle's own error + 1e-4 where that exceeds 1e-4)
    preds, stages = run["preds"], run["stages"]
    bev64 = run["bev"].permute(0, 3, 1, 2).double()
    neck64, head64 = copy.deepcopy(model.neck).double(), copy.deepcopy(model.bbox_head).double()
    with torch.no_grad():
        rpn64 = neck64(dense64)
        ref = head64(rpn64)
        ref_own = head64(neck64(bev64))
    o32_key = {"box_preds": "box", "cls_preds": "cls", "dir_cls_preds": "dir"}
    rows = []
    for t in range(len(ref)):
        assert set(preds[t]) == set(ref[t])
        rows += [("task %d %s" % (t, k), preds[t][k], ref[t][k], ref_own[t][k], stages["heads"][t][o32_key[k]].cuda())
                 for k in ref[t]]
    worst = 0.0
    for what, got_t, want_t, own_t, o32_t in rows:
        e_chain = float((got_t.double() - want_t).abs().max())
        e_own = float((got_t.double() - own_t).abs().max())
        e_o32 = float((o32_t.double() - want_t).abs().max())
        worst = max(worst, e_own)
        assert e_own <= TOL, "%s: abs error %g vs the float64 modules on the device's map" % (what, e_own)
        bound = TOL if e_o32 <= TOL else e_o32 + TOL
        assert e_chain <= bound, "%s: abs error %g vs the float64 chain (fp32 oracle: %g)" % (what, e_chain, e_o32)
    print("%s: heads max abs error vs float64 on the device's map %.3g" % (name, worst))

    # detections == the oracle predict on the device heads, and == the from-scratch oracle up to counted near-ties
    assert run["flag"] == 0
    got, want = run["got"], run["want"]
    thr, pre = cfg.test_cfg.score_threshold, cfg.test_cfg.nms.nms_pre_max_size
    offset = float(cfg.model["bbox_head"]["direction_offset"])
    total = 0
    for b in range(B):
        boxes, scores, labels, flag = [], [], [], 0
        for t, p in enumerate(preds):
            n_cls = model.bbox_head.num_classes[t]
            bx, sc, lb = predict_sample_task(p["cls_preds"][b].reshape(-1, n_cls).cpu(), p["box_preds"][b].reshape(-1, 7).cpu(),
                                             p["dir_cls_preds"][b].reshape(-1, 2).cpu(), pipe._anchors[t].cpu(), cfg.test_cfg,
                                             False, direction_offset=offset)
            boxes.append(bx); scores.append(sc); labels.append(lb + flag)
            flag += n_cls
        wb, ws, wl = torch.cat(boxes), torch.cat(scores), torch.cat(labels)
        gb = got[b]["box3d_lidar"]
        assert gb.shape == wb.shape, "sample %d: %d detections vs %d from the oracle predict" % (b, gb.shape[0], wb.shape[0])
        assert torch.equal(got[b]["label_preds"], wl)
        if wb.shape[0]:
            assert float((gb - wb).abs().max()) <= 1e-5 and float((got[b]["scores"] - ws).abs().max()) <= 1e-6
        total += wb.shape[0]
        fragile = 0
        for h in stages["heads"]:
            sc = torch.sigmoid(h["cls"][b].reshape(-1))
            top = sc[sc >= thr].sort(descending=True)[0][:pre]
            fragile += int(((top[:-1] - top[1:]) < 2e-6).sum()) + int(((sc - thr).abs() < 2e-6).sum())
        w = want[b]["box3d_lidar"]
        missing, extra = ted._unmatched(w, gb, 1e-3), ted._unmatched(gb, w, 1e-3)
        print("%s sample %d: %d detections, oracle %d, %d missing, %d extra, %d near-tied, labels %s" % (
            name, b, gb.shape[0], w.shape[0], missing, extra, fragile, sorted(set(wl.tolist()))))
        assert missing <= fragile and extra <= fragile
    assert total >= 40
    assert len({int(x) for b in range(B) for x in got[b]["label_preds"]}) >= 3, "detections from several tasks"


@pytest.mark.parametrize("name", CONFIGS)
def test_graph_replay_and_batch_composition(deployed, name):
    cfg, pipe, _cpu, _sd, run = deployed(name)
    clouds = [torch.from_numpy(c).pin_memory() for c in run["clouds"]]
    eager = pipe.infer_host(clouds).clone()
    graphed = pipe.infer_host(clouds, graphed=True).clone()
    fg = pipe.forward_graphed(run["pts"], run["offsets"]).clone().cpu()
    D = 300 if name == "kitti_all" else 400
    assert tuple(eager.shape) == (2, D, 10)
    assert torch.equal(graphed, eager) and torch.equal(fg, eager)
    assert torch.equal(eager, pipe.pack(pipe.forward_device(run["pts"], run["offsets"])).cpu())
    alone = [pipe.infer_host([c]).clone() for c in clouds]
    swapped = pipe.infer_host([clouds[1], clouds[0]], graphed=True).clone()
    for b in range(2):
        assert int((alone[b][0, :, -1] > 0.5).sum()) > 0
        assert torch.equal(alone[b][0], eager[b]) and torch.equal(swapped[1 - b], eager[b])
    assert int(pipe.overflow_flag().item()) == 0 and pipe.model.math == "fp16x3"


@pytest.mark.parametrize("name", CONFIGS)
def test_forward_launches_no_vendor_kernel(deployed, name):
    from torch.profiler import ProfilerActivity, profile
    cfg, pipe, _cpu, _sd, run = deployed(name)
    pipe.forward_device(run["pts"], run["offsets"])
    torch.cuda.synchronize()
    # two forwards per trace: a trace can lack the device records of its first operations (see
    # test_frustum_gpu.test_graphed_forward_runs_no_vendor_kernel), and spconv_first16 runs right after the voxelizer
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            pipe.forward_device(run["pts"], run["offsets"])
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    ours = {n for n in names if "d3b" in n}
    assert any("bev_conv16" in n for n in ours) and any("spconv_first16" in n for n in ours), sorted(names)
    vendor = sorted(n for n in names - ours if _VENDOR_KERNEL.search(n))
    assert not vendor, "vendor kernels on the forward: %s" % vendor


@pytest.mark.parametrize("name", CONFIGS)
def test_injected_overflow_reruns_and_matches_the_oracle(deployed, name):
    """As test_f16_guard_gpu: a BatchNorm channel pushed past the f16 range in the sparse encoder (its consumers' weights
    on it zeroed) raises the flag; infer_host warns, switches to tf32x3 and re-runs; the result matches the oracle."""
    cfg, _pipe, cpu, sd, run = deployed(name)
    clouds = [run["clouds"][0]]

    def calibrated(_config):
        return cfg, sd, clouds, type(cpu)
    inject = tfg._inject_sparse(1, 3) if name == "kitti_all" else tfg._inject_cbgs_residual_chain
    config = "second" if name == "kitti_all" else "cbgs"       # _compare's tf32x3 tolerance for both
    ok, report, st = tfg._run_site(calibrated, config, inject, tfg.OVERFLOW, graphed=True)
    assert st["warned"] and st["math"] == "tf32x3" and st["flag"] == 0 and st["finite"], report
    assert ok, "re-run detections differ from the oracle: %s" % report


# ---------------------------------------------------------------------------------------------------------------------
# Lyft: every encoder layer on its deployed rulebook, the dense layers at 252^2 / 126^2, the predict at A = 254,016
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("layer", range(21))
def test_lyft_layer_vs_error_model_on_deployed_rulebook(deployed, layer):
    *_, run = deployed("lyft")
    # test_encoder_deployed_gpu's per-layer check, fed this run (its `deployed` argument only has to return it)
    ted.test_layer_vs_error_model_on_deployed_rulebook(lambda _name: (None, None, None, run), "cbgs", layer)


LYFT_DENSE = [
    # b, h, w, c_in, c_out, ks, stride, pad, up: block 0 (3x3 at 252^2), block 1's strided entry and 3x3 at 126^2,
    # deblock 0 (1x1 at 252^2), deblock 1 (ConvTranspose 126 -> 252), a head (1x1 512 -> 148 fused columns)
    (2, 252, 252, 256, 128, 3, 1, 1, 1),
    (2, 252, 252, 128, 128, 3, 1, 1, 1),
    (2, 252, 252, 128, 256, 3, 2, 1, 1),
    (2, 126, 126, 256, 256, 3, 1, 1, 1),
    (2, 252, 252, 128, 256, 1, 1, 0, 1),
    (2, 126, 126, 256, 256, 1, 1, 0, 2),
]


@pytest.mark.parametrize("b,h,w,c_in,c_out,ks,stride,pad,up", LYFT_DENSE)
def test_lyft_dense_layers_vs_error_model(b, h, w, c_in, c_out, ks, stride, pad, up):
    tem.test_dense_fp16x3_error_model(b, h, w, c_in, c_out, ks, stride, pad, up)


def test_lyft_deployed_layers_match_the_dense_shapes(deployed):
    """LYFT_DENSE lists the layers the deployed Lyft RPN runs."""
    *_, run = deployed("lyft")
    _cfg, pipe, *_ = deployed("lyft")
    layers = dict(pipe.model.fused_bev().layers())
    shapes = {(L.c_in, L.c_out_total, L.ksize, L.stride, L.up) for L in layers.values()}
    for _b, _h, _w, c_in, c_out, ks, stride, _pad, up in LYFT_DENSE:
        assert (c_in, c_out, ks, stride, up) in shapes, (c_in, c_out, ks, stride, up, sorted(shapes))


def test_predict_task_at_254016_anchors():
    """d3b_predict_task against predict_task_reference at Lyft's largest task: 252 x 252 cells x 4 anchors, two classes,
    7-dim boxes, direction classifier with offset 0.785, score 0.1, IoU 0.2, pre 1000 / post 80, label offset 5."""
    T = tpt._gen_task(seed=21, B=2, hw=252 * 252, na=4, n_cls=2, nd=7, dir=True, offset=0.785, rot=True, iou=0.2,
                      thr=0.1, pre=1000, post=80, has_range=True, label_offset=5)
    dev = tpt._Dev(T, 2, 8, 16, 3)
    packed, counts = tpt._run(dev)
    tpt._check_task(T, packed, counts)
    assert min(counts.tolist()) > 0


def test_lyft_test_pipeline_runs_through_pipelines(tmp_path):
    """The stock Lyft test_pipeline, as the reference's file parses, from a LIDAR_TOP file to anchors."""
    from boundary_golden_more import reference_config_more
    from det3d.datasets.pipelines import Compose
    cfg = reference_config_more("examples/cbgs/configs/lyft_all_vfev3_spmiddleresnetfhd_rpn2_mghead_syncbn.py")
    from det3d_b200.utils.synthetic import lidar_like_cloud
    pts = lidar_like_cloud(5000, cfg.voxel_generator.range, 5, 7)
    path = tmp_path / "top.bin"
    pts.tofile(path)
    pipe = Compose(cfg.test_pipeline)
    res = {"lidar": {"type": "lidar"}, "metadata": {}, "mode": "val"}
    info = {"ref_info": {"LIDAR_TOP": {"lidar_path": str(path)}}}
    for t in pipe.transforms[:-1]:
        res, info = t(res, info)
    assert np.array_equal(res["lidar"]["points"], pts[:, :4])
    vox = res["lidar"]["voxels"]
    assert list(vox["shape"]) == [2016, 2016, 40] and vox["voxels"].shape[2] == 4 and vox["num_voxels"][0] > 0
    assert [a.shape[0] for a in res["lidar"]["targets"]["anchors"]] == [127008, 127008, 254016, 127008, 254016]
