"""The sparse encoders at the shapes they are deployed at, against a float64 oracle.

(a) CBGS stage by stage, strict, on four 35k-point 5-feature LiDAR-like clouds and on four 10-sweep samples (one of
    which fills max_voxel_num = 60000): voxels bit-exact; every level's coordinates, rulebook and tile masks bit-exact;
    the BEV map within 1e-4 abs of the float64 oracle (oracle/spconv.py in float64); the RPN and heads within 1e-4 of the
    float64 torch modules fed the device's map, and fed the ORACLE's map within 1e-4 (or, where the fp32 oracle itself
    misses 1e-4, within its own error + 1e-4); detections equal to the oracle predict on the device heads and to the
    from-scratch oracle up to counted near-ties; graph replay bit-identical to eager.

(b) Every encoder layer of SECOND (B = 2) and CBGS (B = 4) in isolation against the FP16x3 error model
    (test_conv_error_model_gpu), on the rulebooks of the deployed run.  LiDAR rulebooks are ragged: most 128-row tiles
    lack some kernel offsets, so tiles run different numbers of pipeline slots and packed slot groups are only partly
    present -- the situation uniformly random test sites (every tile holds every offset) never reach.  The test asserts
    that raggedness, so a change of data generator cannot quietly turn it back into the easy case.
"""
import copy
import os
import types

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_conv_error_model_gpu import U, _os16_pack, check_against_model, check_epilogue, sparse_ref

pytestmark = pytest.mark.gpu

TOL = 1e-4              # BASELINE.json north_star: float features within 1e-4 abs
B_CBGS = 4
N_CBGS = 35000
SWEEP_SIZES = (3000, 4000, 5000, 7500)      # records per sweep of each sample; 10 x 7500 fills 60000 voxels


# ---------------------------------------------------------------------------------------------------------------------
# models, oracle runs and deployed runs (module-scoped, built on first use)
# ---------------------------------------------------------------------------------------------------------------------

def _config(name):
    from det3d.torchie import Config
    return Config.fromfile(os.path.join(ROOT, "configs", name))


def _cbgs_model(sweeps=False):
    """Seeded and calibrated as in test_e2e_gpu.test_cbgs_nuscenes_config; with sweeps=True the BatchNorm statistics come
    from merged 10-sweep samples instead of single frames.

    A CBGS model is trained on 10-sweep input, and its BatchNorm layers keep its features O(1) on such input.  Single-frame
    statistics do not: ten merged sweeps fill about three times as many voxels, each SubM site has more active neighbours,
    and the BEV map and RPN output of the single-frame model reach 56 and 82 on the multi-sweep workload.  There an
    absolute 1e-4 is below what fp32 resolves: the fp32 CPU oracle's own RPN output is 2.6e-4 from the float64 one
    (measured with this file's workloads on an H100 80GB HBM3 at 700 W)."""
    from det3d.models import build_detector
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud, lidar_like_sweeps
    from oracle.cbgs_cpu import CbgsCPU
    from oracle.ingest import merge_sweeps
    cfg = _config("cbgs_nusc.py")
    r = cfg.voxel_generator.range
    torch.manual_seed(1)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 1)
    if sweeps:
        calib = [merge_sweeps(*lidar_like_sweeps([5000] * 10, r, 50 + i)) for i in range(2)]
    else:
        calib = [lidar_like_cloud(N_CBGS, r, 5, 50 + i) for i in range(2)]
    calibrate_demo_weights_(model, cfg, calib, 1, pass_fraction=0.01)
    return cfg, model, CbgsCPU


def _second_model():
    """Seeded and calibrated as in test_e2e_gpu.setup."""
    from det3d.models import build_detector
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud
    from oracle.second_cpu import SecondCPU
    cfg = _config("second_kitti_car.py")
    torch.manual_seed(0)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 0)
    calibrate_demo_weights_(model, cfg, [lidar_like_cloud(20000, cfg.voxel_generator.range, 4, 900 + i) for i in range(2)], 0)
    return cfg, model, SecondCPU


def _snapshot(fused):
    """(layer, rulebook) of every step of the last run, the rulebooks copied: a later run rewrites them in place."""
    from det3d_b200.ops.spconv import core
    copies, steps = {}, []
    for L, rb, _build in fused._state["steps"]:
        c = copies.get(id(rb))
        if c is None:
            lv = rb.out_level
            out = core.SparseLevel(lv.coors.clone(), lv.n.clone(), lv.cap, lv.spatial, lv.batch)
            c = copies[id(rb)] = core.Rulebook(rb.nbr.clone(), rb.tile_mask.clone(), rb.ksize, out, None, rb.kind)
        steps.append((L, c))
    return steps


def _workload(name, cfg):
    """-> (oracle clouds, samples or None) of a named workload."""
    from det3d_b200.utils.synthetic import lidar_like_cloud, lidar_like_sweeps, uniform_cloud
    from oracle.ingest import merge_sweeps
    r = cfg.voxel_generator.range
    if name == "second":
        return [lidar_like_cloud(20000, r, 4, 1), uniform_cloud(20000, r, 4, 1)], None
    if name == "cbgs_clouds":
        return [lidar_like_cloud(N_CBGS, r, 5, s) for s in range(B_CBGS)], None
    samples = [lidar_like_sweeps([n] * 10, r, 500 + b) for b, n in enumerate(SWEEP_SIZES)]
    return [merge_sweeps(*s) for s in samples], samples


def _run(cfg, pipe, cpu, name):
    """The oracle (fp32 from scratch, and the float64 encoder with its per-layer record) and the deployed device run of
    one workload."""
    from det3d_b200.datasets.pipelines.loading import ingest_sweeps_batched
    from det3d_b200.ops.spconv import conv16
    clouds, samples = _workload(name, cfg)
    B = len(clouds)
    stages = {}
    if name == "second":              # only the encoder is needed: voxelize, no RPN / predict
        stages["voxels"], stages["coors"], stages["nums"] = cpu.voxelize(clouds)
        want = None
    else:
        want = cpu.forward(clouds, stages)
    dense64, levels64, _ = cpu.backbone(stages["voxels"], stages["coors"], stages["nums"], B, dtype=torch.float64,
                                        return_levels=True)
    model = pipe.model
    grid = [int(g) for g in pipe.grid_size]
    with torch.no_grad():
        if samples is None:
            pts = torch.from_numpy(np.concatenate(clouds)).cuda()
            offsets = np.cumsum([0] + [c.shape[0] for c in clouds]).tolist()
        else:
            pts, offsets = ingest_sweeps_batched(samples, 1.0, 4, "cuda")
        vox = pipe.voxelizer(pts, offsets)
        counts = vox["counts"].clone()
        feats = vox["mean"].clone()
        planes = model.backbone.forward_planes(feats, vox["coors"], B, grid, n_dev=counts[B:B + 1])
        bev = planes.to_f32()
        kept = conv16.Planes(planes.shape, "cuda")          # the encoder's own buffer is rewritten by the next run
        kept.buf.copy_(planes.buf)
        steps = _snapshot(model.backbone.fused())
        run = dict(name=name, B=B, clouds=clouds, samples=samples, stages=stages, want=want, dense64=dense64,
                   levels64=levels64, counts=counts.cpu().numpy(), coors=vox["coors"][:int(counts[B])].cpu().numpy(),
                   mean=feats[:int(counts[B])].cpu(), feats=feats, planes=kept, bev=bev, steps=steps)
        if want is not None:
            fb = model.fused_bev()
            run["preds"] = [{k: v.clone() for k, v in d.items()} for d in fb.run(planes)]
            run["rpn"] = fb._bufs[("concat",)].to_f32()
            if samples is None:
                run["got"] = pipe.unpack(pipe.pack(pipe.forward_device(pts, offsets)).cpu())
                run["pts"], run["offsets"] = pts, offsets
            else:
                run["got"] = pipe.unpack(pipe.infer_sweeps(samples).clone())
            run["flag"] = int(pipe.overflow_flag().item())
    return run


@pytest.fixture(scope="module")
def deployed():
    """workload name -> (cfg, pipe, oracle, run of _run), each model built and each workload run once."""
    from det3d_b200.apis import InferencePipeline
    models, runs = {}, {}

    def get(name):
        cname = {"second": "second", "cbgs_clouds": "cbgs", "cbgs_sweeps": "cbgs_sweeps"}[name]
        if cname not in models:
            cfg, model, oracle = _second_model() if cname == "second" else _cbgs_model(sweeps=cname == "cbgs_sweeps")
            sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
            pipe = InferencePipeline(cfg, model=model, device="cuda")
            models[cname] = (cfg, pipe, oracle(cfg, sd, [a.cpu().numpy() for a in pipe._anchors]))
        if name not in runs:
            runs[name] = _run(*models[cname], name)
        return models[cname] + (runs[name],)
    return get


# ---------------------------------------------------------------------------------------------------------------------
# shared checks
# ---------------------------------------------------------------------------------------------------------------------

def _tile_bits(nbr, n):
    """Tile masks (bit k: offset k occurs in the 128-row tile) recomputed from an oracle nbr [K, n]."""
    k_vol = nbr.shape[0]
    nt = (n + 127) // 128
    ok = np.zeros((k_vol, nt * 128), bool)
    ok[:, :n] = nbr[:, :n] >= 0
    present = ok.reshape(k_vol, nt, 128).any(2)
    return (present.astype(np.int64) << np.arange(k_vol)[:, None]).sum(0)


def _check_levels(run):
    """Every step's output coordinates, row count, neighbour map and tile masks equal the oracle's bit for bit."""
    assert len(run["steps"]) == len(run["levels64"])
    seen = set()
    for i, ((L, rb), rec) in enumerate(zip(run["steps"], run["levels64"])):
        assert rb.k_vol == rec["nbr"].shape[0] and (rb.kind == "subm") == (rec["kind"] == "subm"), i
        if id(rb) in seen:
            continue
        seen.add(id(rb))
        n = rec["coors"].shape[0]
        assert int(rb.out_level.n[0]) == n and int(rb.out_level.n[1]) == n, "layer %d: %d rows vs %d" % (
            i, int(rb.out_level.n[0]), n)
        assert rb.out_level.spatial == tuple(rec["spatial"]), i
        assert np.array_equal(rb.out_level.coors[:n].cpu().numpy(), rec["coors"]), "layer %d: coordinates" % i
        assert np.array_equal(rb.nbr[:, :n].cpu().numpy().astype(np.int64), rec["nbr"]), "layer %d: rulebook" % i
        got = rb.tile_mask[:(n + 127) // 128].cpu().numpy().astype(np.int64) & 0xFFFFFFFF
        assert np.array_equal(got, _tile_bits(rec["nbr"], n)), "layer %d: tile masks" % i


def _check_voxels(run):
    st, B = run["stages"], run["B"]
    m = int(run["counts"][B])
    assert run["counts"][:B].sum() == m == st["coors"].shape[0]
    assert np.array_equal(run["coors"], st["coors"]) and np.array_equal(run["counts"][:B], np.bincount(st["coors"][:, 0], minlength=B))
    c = st["voxels"].shape[2]
    mean = st["voxels"].sum(1) / st["nums"][:, None].astype(np.float32)
    assert float(np.abs(run["mean"].numpy()[:, :c] - mean).max()) <= 1e-6


def _chain_errors(run):
    """Re-run the deployed chain layer by layer (the fused encoder's kernels, weights and rulebooks, every output kept)
    -> max |device - float64 oracle| per layer.  The last output scattered to BEV planes must give the deployed planes'
    bits, so these are the errors of the deployed run."""
    from det3d_b200.ops.spconv import conv16
    x, identity, errs = run["feats"], None, []
    for (L, rb), rec in zip(run["steps"], run["levels64"]):
        if L.save_identity:
            identity = x
        out = conv16.Planes((rb.out_level.cap, L.conv.out_channels), "cuda")
        conv16.sparse_conv16(x, rb, L.cw16, out, residual=identity if L.residual else None)
        n = rec["coors"].shape[0]
        errs.append(float((out.to_f32()[:n].double() - rec["output"].cuda()).abs().max()))
        x = out
    final = run["steps"][-1][1].out_level
    planes = conv16.Planes(run["planes"].shape, "cuda", zero=True)
    conv16.sparse_to_bev16(x, final, planes)
    assert torch.equal(planes.buf, run["planes"].buf), "the layer-by-layer replay is not the deployed computation"
    return errs


def _unmatched(want_boxes, got_boxes, tol):
    if want_boxes.shape[0] == 0:
        return 0
    if got_boxes.shape[0] == 0:
        return int(want_boxes.shape[0])
    d = (want_boxes[:, None, :] - got_boxes[None, :, :]).abs().max(-1)[0]
    return int((d.min(1)[0] > tol).sum())


# ---------------------------------------------------------------------------------------------------------------------
# (a) CBGS stage by stage
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("workload", ["cbgs_clouds", "cbgs_sweeps"])
def test_cbgs_stage_by_stage_vs_float64_oracle(deployed, workload):
    from oracle.predict_cpu import predict_sample_task
    cfg, pipe, cpu, run = deployed(workload)
    B, model = run["B"], pipe.model
    vg = cfg.voxel_generator
    _check_voxels(run)
    per_sample = run["counts"][:B]
    print("%s: voxels per sample %s, rows per level %s" % (workload, per_sample.tolist(),
                                                          [r["coors"].shape[0] for r in run["levels64"][::5]]))
    if workload == "cbgs_sweeps":          # the reference's `break` at max_voxel_num is reached, and only there
        assert (per_sample == vg.max_voxel_num).any() and (per_sample < vg.max_voxel_num).any()
    _check_levels(run)

    # the BEV map (C * D = 256 channels) against the float64 oracle; the chain's per-layer errors for the record
    dense64 = run["dense64"].cuda()
    assert dense64.shape[1] == 256 and float(dense64.abs().max()) < 100.0, "calibration failed: features are not O(1)"
    err = float((run["bev"].permute(0, 3, 1, 2).double() - dense64).abs().max())
    err32 = float((run["stages"]["dense"].double().cuda() - dense64).abs().max())
    errs = _chain_errors(run)
    print("%s: BEV max abs error vs float64 %.3g (fp32 oracle %.3g); per layer %s" % (
        workload, err, err32, " ".join("%.2g" % e for e in errs)))
    assert err <= TOL, "BEV map: abs error %g vs the float64 oracle" % err

    # RPN + heads from the device planes vs the float64 modules, (i) on the oracle's map: the whole chain, and (ii) on the
    # device's own map: the dense kernels alone.  The RPN amplifies its input's rounding (about 4.5x here), so (i) is
    # held to 1e-4 wherever the fp32 oracle itself -- its RPN and heads on its own fp32 map -- is within 1e-4 of float64,
    # and otherwise to the fp32 oracle's own error plus 1e-4.  (ii) is always held to 1e-4.
    preds, stages = run["preds"], run["stages"]
    bev64 = run["bev"].permute(0, 3, 1, 2).double()
    neck64, head64 = copy.deepcopy(model.neck).double(), copy.deepcopy(model.bbox_head).double()
    with torch.no_grad():
        rpn64 = neck64(dense64)
        ref = head64(rpn64)
        rpn_own = neck64(bev64)
        ref_own = head64(rpn_own)
    rpn = run["rpn"].permute(0, 3, 1, 2).double()
    rows = [("RPN", rpn, rpn64, rpn_own, stages["rpn"].cuda())]
    o32_key = {"box_preds": "box", "cls_preds": "cls", "dir_cls_preds": "dir"}
    for t in range(len(ref)):
        assert set(preds[t]) == set(ref[t])
        rows += [("task %d %s" % (t, k), preds[t][k], ref[t][k], ref_own[t][k], stages["heads"][t][o32_key[k]].cuda())
                 for k in ref[t]]
    worst = dict(chain=0.0, own=0.0, o32=0.0)
    for what, got_t, want_t, own_t, o32_t in rows:
        e_chain = float((got_t.double() - want_t).abs().max())
        e_own = float((got_t.double() - own_t).abs().max())
        e_o32 = float((o32_t.double() - want_t).abs().max())
        for k, v in (("chain", e_chain), ("own", e_own), ("o32", e_o32)):
            worst[k] = max(worst[k], v)
        if what == "RPN":
            print("%s: RPN max |x| %.3g" % (workload, float(want_t.abs().max())))
        assert e_own <= TOL, "%s: abs error %g vs the float64 modules on the device's map" % (what, e_own)
        bound = TOL if e_o32 <= TOL else e_o32 + TOL
        assert e_chain <= bound, "%s: abs error %g vs the float64 chain (fp32 oracle: %g)" % (what, e_chain, e_o32)
    print("%s: RPN + heads max abs error vs float64: chain %.3g, on the device's own map %.3g, fp32 oracle %.3g" % (
        workload, worst["chain"], worst["own"], worst["o32"]))

    # device detections == the oracle predict on the device heads (same order), and == the from-scratch oracle's set up
    # to counted near-ties
    got, want, stages = run["got"], run["want"], run["stages"]
    assert run["flag"] == 0
    thr, pre = cfg.test_cfg.score_threshold, cfg.test_cfg.nms.nms_pre_max_size
    total = 0
    for b in range(B):
        boxes, scores, labels, flag = [], [], [], 0
        for task_id, p in enumerate(preds):
            n_cls = model.bbox_head.num_classes[task_id]
            bx, sc, lb = predict_sample_task(p["cls_preds"][b].reshape(-1, n_cls).cpu(), p["box_preds"][b].reshape(-1, 10).cpu(),
                                             p["dir_cls_preds"][b].reshape(-1, 2).cpu() if "dir_cls_preds" in p else None,
                                             pipe._anchors[task_id].cpu(), cfg.test_cfg, True)
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
        missing, extra = _unmatched(w, gb, 1e-3), _unmatched(gb, w, 1e-3)
        print("%s sample %d: %d detections, oracle %d, %d missing, %d extra, %d near-tied" % (
            workload, b, gb.shape[0], w.shape[0], missing, extra, fragile))
        assert missing <= fragile and extra <= fragile, \
            "sample %d: %d missing, %d extra with %d near-tied candidates" % (b, missing, extra, fragile)
    assert total >= 40

    # graph replay == eager, flag clear
    if run["samples"] is None:
        clouds = [torch.from_numpy(c).pin_memory() for c in run["clouds"]]
        eager = pipe.infer_host(clouds).clone()
        graphed = pipe.infer_host(clouds, graphed=True).clone()
        assert torch.equal(eager, pipe.pack(pipe.forward_device(run["pts"], run["offsets"])).cpu())
    else:
        eager = pipe.infer_sweeps(run["samples"]).clone()
        graphed = pipe.infer_sweeps(run["samples"], graphed=True).clone()
    assert torch.equal(graphed, eager)
    assert torch.equal(pipe.unpack(eager)[0]["box3d_lidar"], got[0]["box3d_lidar"])
    assert int(pipe.overflow_flag().item()) == 0 and pipe.model.math == "fp16x3"


# ---------------------------------------------------------------------------------------------------------------------
# (b) every layer against the FP16x3 error model, on the deployed rulebooks
# ---------------------------------------------------------------------------------------------------------------------

RUN_OF = {"second": "second", "cbgs": "cbgs_clouds"}
N_LAYERS = {"second": 14, "cbgs": 21}
LAYERS = [(c, i) for c in ("second", "cbgs") for i in range(N_LAYERS[c])]

# Share of 128-row tiles that lack at least one kernel offset, per rulebook in plan order (level 0 SubM, then each
# strided conv and the SubM of its level).  Measured with the CPU oracle on these workloads:
#   SECOND  0.884 0.281 0.204 0.165 0.163 0.080 0.391 0.166
#   CBGS    1.000 0.775 0.747 0.721 0.711 0.543 0.540 0.987
# The bounds keep about 60 % of each.
MIN_RAGGED = {"second": [0.5, 0.15, 0.12, 0.1, 0.1, 0.045, 0.2, 0.1],
              "cbgs": [0.6, 0.45, 0.45, 0.4, 0.4, 0.3, 0.3, 0.6]}
MIN_PARTIAL_GROUPS = 20      # (tile, slot group) pairs with some but not all offsets present, per packed layer


def _layer_operands(run, i):
    L, rb = run["steps"][i]
    rec = run["levels64"][i]
    c_in, c_out = L.conv.in_channels, L.conv.out_channels
    w = L.conv.weight.detach().float().reshape(-1, c_in, c_out).contiguous().cuda()
    x = rec["input"].float().cuda().contiguous()            # the float64 oracle's input, rounded to fp32
    return L, rb, rec, w, x, rec["coors"].shape[0]


@pytest.mark.parametrize("config,layer", LAYERS, ids=["%s-L%02d" % t for t in LAYERS])
def test_layer_vs_error_model_on_deployed_rulebook(deployed, config, layer):
    from det3d_b200.ops.spconv import conv16
    *_, run = deployed(RUN_OF[config])
    L, rb, rec, w, x, n_out = _layer_operands(run, layer)
    assert np.array_equal(rb.nbr[:, :n_out].cpu().numpy().astype(np.int64), rec["nbr"])
    what = "%s layer %d (%s, C_in %d -> %d, k_vol %d, %d rows)" % (config, layer, rec["conv"], w.shape[1], w.shape[2],
                                                                 w.shape[0], n_out)
    cap, c_out = rb.out_level.cap, w.shape[2]
    raw = torch.full((cap, c_out), float("nan"), device="cuda")
    cw = conv16.ConvWeights16(w)
    if cw.fp32_input:
        # FFMA chains (test_sparse_first_layer_fp32_input): |got - y| <= L u (1 + L u) M, L = 7 C_in + 2
        conv16.sparse_conv16(x, rb, cw, None, out_f32=raw)
        idx = rb.nbr[:, :n_out].long()
        y = torch.zeros((n_out, c_out), dtype=torch.float64, device="cuda")
        m = torch.zeros_like(y)
        for k in range(w.shape[0]):
            ok = idx[k] >= 0
            y[ok] += x.double()[idx[k][ok]] @ w.double()[k]
            m[ok] += x.double().abs()[idx[k][ok]] @ w.double().abs()[k]
        lc = 7 * w.shape[1] + 2
        tol = lc * U * (1 + lc * U) * m
        worst = float(((raw[:n_out].double() - y).abs() / tol.clamp_min(1e-300)).max())
        assert worst <= 1.0, "%s: error reaches %.3g of the FFMA bound" % (what, worst)
        ref = types.SimpleNamespace(yh=y, elem_tol=lambda: tol)
        x_in = x
    else:
        planes = conv16.Planes.from_f32(x)
        conv16.sparse_conv16(planes, rb, cw, None, out_f32=raw)
        ref = sparse_ref(x, planes, w, cw.w_exp, rb.nbr, n_out)
        stats = check_against_model(raw[:n_out], ref, cw.w_exp, what)
        worst = stats["worst"]
        x_in = planes
    assert bool(torch.isnan(raw[n_out:]).all()), "%s: rows past the live count were written" % what
    print("%s: worst |got - yh| / bound %.3f" % (what, worst))

    # the fused epilogue of the deployed layer: bias, folded BatchNorm, the oracle's identity, ReLU; planes to 22 bits
    res = conv16.Planes.from_f32(rec["identity"].float().cuda()) if L.residual else None
    assert (res is None) == (rec["identity"] is None)
    out = conv16.Planes((cap, c_out), "cuda")
    out32 = torch.empty((cap, c_out), device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    e = L.cw16
    conv16.sparse_conv16(x_in, rb, e, out, residual=res, out_f32=out32, overflow=flag)
    assert int(flag.item()) == 0
    bias = e.bias if e.bias is not None else torch.zeros(c_out, device="cuda")
    check_epilogue(out32[:n_out], out.to_f32()[:n_out], ref, bias, e.scale, e.shift, e.relu,
                   res=None if res is None else res.to_f32(), what=what)


@pytest.mark.parametrize("config", ["second", "cbgs"])
def test_deployed_rulebooks_are_ragged(deployed, config):
    """The property that makes the per-layer test worth having: at every level a share of the tiles lacks some offset
    (slot counts vary from tile to tile), and on every packed layer (C_in 16 / 32) some slot groups are partly present."""
    *_, run = deployed(RUN_OF[config])
    rbs, fracs = [], []
    for L, rb in run["steps"]:
        n = int(rb.out_level.n[0])
        mask = rb.tile_mask[:(n + 127) // 128].cpu().numpy().astype(np.int64) & 0xFFFFFFFF
        full = (1 << rb.k_vol) - 1
        if all(rb is not r for r in rbs):
            rbs.append(rb)
            fracs.append(float((mask != full).mean()))
        pack = _os16_pack(L.conv.in_channels, rb.k_vol)
        if pack > 1:
            partial = 0
            for g in range(0, rb.k_vol, pack):
                grp = ((1 << min(pack, rb.k_vol - g)) - 1) << g
                partial += int(((mask & grp) != 0).sum() - ((mask & grp) == grp).sum())
            print("%s C_in %d pack %d: %d partly present slot groups" % (config, L.conv.in_channels, pack, partial))
            assert partial >= MIN_PARTIAL_GROUPS, "%s: C_in %d, only %d partly present slot groups" % (
                config, L.conv.in_channels, partial)
    print("%s: share of tiles lacking an offset per rulebook: %s" % (config, " ".join("%.3f" % f for f in fracs)))
    assert len(fracs) == len(MIN_RAGGED[config])
    for j, (f, lo) in enumerate(zip(fracs, MIN_RAGGED[config])):
        assert f >= lo, "%s rulebook %d: only %.3f of the tiles lack an offset (bound %.3f)" % (config, j, f, lo)


@pytest.mark.parametrize("config", ["second", "cbgs"])
def test_error_model_rejects_swapped_offsets(deployed, config):
    """Host-side discrimination: a kernel that read offset 22's neighbour rows for offset 4 and vice versa (different
    slot groups when packed) must fail the bound on the first packed layer, the C_in 16 SubM of level 0."""
    from det3d_b200.ops.spconv import conv16
    *_, run = deployed(RUN_OF[config])
    L, rb, rec, w, x, n_out = _layer_operands(run, 1)
    assert w.shape[:2] == (27, 16)
    planes = conv16.Planes.from_f32(x)
    cw = conv16.ConvWeights16(w)
    raw = torch.empty((rb.out_level.cap, w.shape[2]), device="cuda")
    conv16.sparse_conv16(planes, rb, cw, None, out_f32=raw)
    check_against_model(raw[:n_out], sparse_ref(x, planes, w, cw.w_exp, rb.nbr, n_out), cw.w_exp, "unswapped")
    swapped = rb.nbr[:, :n_out].clone()
    swapped[[4, 22]] = swapped[[22, 4]]
    bad = sparse_ref(x, planes, w, cw.w_exp, swapped, n_out)
    with pytest.raises(AssertionError, match="accumulation bound|RMS"):
        check_against_model(raw[:n_out], bad, cw.w_exp, "swapped offsets 4 / 22")
