"""The f16-range guard of the FP16x3 format (DESIGN 3.0) at every launch that writes planes, and the tf32x3 re-run it
triggers in the detectors.

Kernel level.  Every plane writer -- d3b_split16, the pillar scatter d3b_sparse_to_bev16 (fp32 rows and plane rows),
the fp32-input first sparse layer, the tensor-core sparse kernel at every C_out, and the dense kernel in each shape it
builds (3x3 stride 1 / 2, 1x1, ConvTranspose, k = s deblocks, a two-group launch into a channel slice; the pipelined
schedule in test_bev_conv16_pipelined_gpu) -- is driven across the boundary of the f16 range, with and without ReLU.  The value is placed on one
output channel whose weights are zero, through the bias (scaled by an exact 1/2 in the folded BatchNorm, with a residual
of 1 on the sparse kernel), so it reaches the range check exactly; the other channels carry ordinary O(1) results.  At
every value the flag must be raised exactly when the value written is not below 65504 in magnitude or is NaN; hi / lo
must be the split of the written value (65519.99 keeps a finite hi, 65520 does not), and where the flag stays clear the
fp32 output must equal the value pushed through the epilogue in float64 and hi + lo must hold it to 22 bits.  Under ReLU
a large or infinite negative value must become an exact +0 and leave the flag clear.

Detector level.  One channel of a layer is given BatchNorm weight 0 and bias 7e4, and every consumer of that channel is
given zero weights on it, so the correct detections are those of a finite network.  The FP16x3 forward must raise the
flag, `infer_host` must warn, switch to tf32x3 and re-run, and the re-run's detections must match the configuration's
CPU oracle run on the modified weights.  The same injection with bias 6e4 is the control: no flag, no re-run, and the
FP16x3 detections match the oracle, which shows that each site is live and that its channel really is irrelevant.
"""
import math
import os
import warnings

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_conv_error_model_gpu import _level, dense_layer, split16

pytestmark = pytest.mark.gpu

INF, NAN = float("inf"), float("nan")
# (value, flag raised when it is written without ReLU)
VALUES = [(65503.99, 0), (-65503.99, 0), (65504.0, 1), (-65504.0, 1), (65519.99, 1), (-65519.99, 1), (65520.0, 1),
          (-65520.0, 1), (1.0e6, 1), (-1.0e6, 1), (INF, 1), (-INF, 1), (NAN, 1), (0.75, 0), (-0.75, 0)]


def _f32(v):
    return float(np.float32(v))


def _cases(relu):
    """(value, value written, flag) for one ReLU setting.  A NaN under ReLU is out of the guard's scope: fmaxf turns it
    into 0 (DESIGN 3.0), so it is not a case here."""
    out = []
    for v, flag in VALUES:
        if relu and math.isnan(v):
            continue
        e = max(_f32(v), 0.0) if relu else _f32(v)
        out.append((v, e, 0 if relu and v < 0 else flag))
    return out


def _same(a, b):
    """Equal values, NaN where the other is NaN, and the same sign of every zero."""
    a, b = a.float(), b.float()
    na, nb = torch.isnan(a), torch.isnan(b)
    return (torch.equal(na, nb) and torch.equal(a[~na], b[~nb])
            and torch.equal(torch.signbit(a[~na]), torch.signbit(b[~nb])))


def check_written(what, e, flag, want_flag, hi, lo, f32=None):
    """hi / lo (and the fp32 output, if any) at every position that received the value e."""
    assert flag == want_flag, "%s: flag %d, expected %d" % (what, flag, want_flag)
    want = torch.full(hi.shape, e, dtype=torch.float32, device=hi.device)
    w_hi, w_lo = split16(want)
    assert _same(hi, w_hi) and _same(lo, w_lo), "%s: planes (%r, %r) are not the split of %r" % (
        what, float(hi.flatten()[0]), float(lo.flatten()[0]), e)
    if f32 is not None:
        assert _same(f32, want), "%s: fp32 output %r, expected %r" % (what, float(f32.flatten()[0]), e)
    if not want_flag:
        s = hi.double() + lo.double()
        assert bool(((s - e).abs() <= 2.0 ** -22 * abs(e)).all()), "%s: hi + lo does not hold %r to 22 bits" % (what, e)
        if e == 0.0:
            assert not bool(torch.signbit(hi).any() or torch.signbit(lo).any()), "%s: -0 instead of +0" % what


def _epi(c_out, c, seed, v, res=0.0):
    """Bias / folded BatchNorm with channel c carrying v: bias 2 (v - res), scale 1/2, shift 0 -- exact in fp32."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    bias = torch.randn(c_out, device="cuda", generator=g) * 0.1
    scale = torch.rand(c_out, device="cuda", generator=g) + 0.5
    shift = torch.randn(c_out, device="cuda", generator=g) * 0.1
    bias[c] = 2.0 * (_f32(v) - res)
    scale[c], shift[c] = 0.5, 0.0
    return bias, scale, shift


def _flag(preset=0):
    return torch.full((1,), preset, dtype=torch.int32, device="cuda")


# ---------------------------------------------------------------------------------------------------------------------
# kernel level
# ---------------------------------------------------------------------------------------------------------------------

def test_split16_planes_at_the_boundary():
    from det3d_b200.ops.spconv import conv16
    for v, e, want in _cases(False):
        flag = _flag()
        x = torch.tensor([[0.5, v, -2.0, 3.0]], device="cuda")
        p = conv16.Planes.from_f32(x, flag)
        check_written("split16(%r)" % v, e, int(flag.item()), want, p.hi[:, 1], p.lo[:, 1])
        assert _same(p.hi[:, [0, 2, 3]], x[:, [0, 2, 3]].half())


def _scatter_setup():
    """B = 2, D = 3 level with rows past the live count poisoned (they must not be read)."""
    from det3d_b200.ops.spconv import core
    B, D, H, W, C = 2, 3, 20, 24, 16
    n, cap = 300, 320
    rng = np.random.default_rng(5)
    cells = rng.choice(B * D * H * W, size=cap, replace=False)
    b, rem = np.divmod(cells, D * H * W)
    z, rem = np.divmod(rem, H * W)
    y, x = np.divmod(rem, W)
    coors = torch.from_numpy(np.stack([b, z, y, x], 1).astype(np.int32)).cuda()
    level = core.SparseLevel(coors, torch.tensor([n, n], dtype=torch.int32, device="cuda"), cap, (D, H, W), B)
    feats = torch.randn((cap, C), device="cuda", generator=torch.Generator(device="cuda").manual_seed(5)) * 10.0
    feats[n:] = 1.0e9
    row = int(np.nonzero((b[:n] == 1) & (z[:n] == 2))[0][0])           # a row of sample 1 at z = D - 1
    return (B, D, H, W, C, n), coors, level, feats, row


def _scatter_ref(shape, coors, feats):
    B, D, H, W, C, n = shape
    dense = torch.zeros((B, H, W, C * D), device="cuda")
    q = coors[:n].long()
    ch = torch.arange(C, device="cuda") * D
    dense[q[:, 0:1], q[:, 2:3], q[:, 3:4], ch[None, :] + q[:, 1:2]] = feats[:n]
    return split16(dense)


def test_pillar_scatter_flags_fp32_rows_and_copies_planes_untouched():
    """d3b_sparse_to_bev16: fp32 rows are split and range-checked (channel = c*D + z, B > 1, D > 1); plane rows are
    copied bit for bit and leave the flag as it was (their writer checked them)."""
    from det3d_b200.ops.spconv import conv16
    shape, coors, level, feats, row = _scatter_setup()
    B, D, H, W, C, n = shape
    c = 13
    bq, zq, yq, xq = [int(t) for t in coors[row]]
    for v, e, want in _cases(False):
        f = feats.clone()
        f[row, c] = v
        out = conv16.Planes((B, H, W, C * D), "cuda", zero=True)
        flag = _flag()
        conv16.sparse_to_bev16(f, level, out, overflow=flag)
        what = "scatter fp32 rows, v = %r" % v
        check_written(what, e, int(flag.item()), want, out.hi[bq, yq, xq, c * D + zq:c * D + zq + 1],
                      out.lo[bq, yq, xq, c * D + zq:c * D + zq + 1])
        r_hi, r_lo = _scatter_ref(shape, coors, f)
        assert _same(out.hi, r_hi) and _same(out.lo, r_lo), "%s: BEV planes differ from the scatter of the split" % what
        # plane rows: the same planes, and the flag untouched whatever they hold (preset to 2: an OR of 1 would show)
        planes = conv16.Planes.from_f32(f)
        out2 = conv16.Planes((B, H, W, C * D), "cuda", zero=True)
        flag2 = _flag(2)
        conv16.sparse_to_bev16(planes, level, out2, overflow=flag2)
        assert int(flag2.item()) == 2, "scatter of plane rows touched the flag (v = %r)" % v
        assert _same(out2.hi, out.hi) and _same(out2.lo, out.lo)
    out = conv16.Planes((B, H, W, C * D), "cuda", zero=True)
    flag = _flag()
    conv16.sparse_to_bev16(feats, level, out, overflow=flag)
    assert int(flag.item()) == 0, "rows past the live count were read"


def _sparse_rulebook(n, seed):
    from det3d_b200.ops.spconv import core
    lvl = _level(n, (9, 40, 36), 2, seed)
    return core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, 3))


@pytest.mark.parametrize("c_out", [16, 32, 64])
def test_first_layer_fp32_input_guard(c_out):
    """The fp32-input first sparse layer (spconv_first16_kernel -> epilogue16), C_in = 4."""
    from det3d_b200.ops.spconv import conv16
    n, c = 700, c_out - 3
    rb = _sparse_rulebook(n, c_out)
    g = torch.Generator(device="cuda").manual_seed(c_out)
    x = torch.randn((n, 4), device="cuda", generator=g)
    w = torch.randn((27, 4, c_out), device="cuda", generator=g) * 0.1
    w[..., c] = 0.0
    for relu in (False, True):
        for v, e, want in _cases(relu):
            bias, scale, shift = _epi(c_out, c, c_out, v)
            cw = conv16.ConvWeights16(w, bias=bias, scale=scale, shift=shift, relu=relu)
            assert cw.fp32_input
            out = conv16.Planes((n, c_out), "cuda")
            out32 = torch.empty((n, c_out), device="cuda")
            flag = _flag()
            conv16.sparse_conv16(x, rb, cw, out, out_f32=out32, overflow=flag)
            check_written("first layer C_out %d relu %d v = %r" % (c_out, relu, v), e, int(flag.item()), want,
                          out.hi[:, c], out.lo[:, c], out32[:, c])


@pytest.mark.parametrize("c_out", [16, 32, 64, 128])
def test_sparse_fp16x3_guard_with_residual(c_out):
    """The tensor-core sparse kernel at every C_out, with a residual (1 on the value's channel)."""
    from det3d_b200.ops.spconv import conv16
    n, c_in, c = 900, 32, c_out // 2 + 1
    rb = _sparse_rulebook(n, c_out + 1)
    g = torch.Generator(device="cuda").manual_seed(c_out + 1)
    x = conv16.Planes.from_f32(torch.randn((n, c_in), device="cuda", generator=g))
    w = torch.randn((27, c_in, c_out), device="cuda", generator=g) * 0.05
    w[..., c] = 0.0
    res = torch.randn((n, c_out), device="cuda", generator=g)
    res[:, c] = 1.0
    res_p = conv16.Planes.from_f32(res)
    for relu in (False, True):
        for v, e, want in _cases(relu):
            bias, scale, shift = _epi(c_out, c, c_out, v, res=1.0)
            cw = conv16.ConvWeights16(w, bias=bias, scale=scale, shift=shift, relu=relu)
            assert not cw.fp32_input
            out = conv16.Planes((n, c_out), "cuda")
            out32 = torch.empty((n, c_out), device="cuda")
            flag = _flag()
            conv16.sparse_conv16(x, rb, cw, out, residual=res_p, out_f32=out32, overflow=flag)
            check_written("os16 C_out %d relu %d v = %r" % (c_out, relu, v), e, int(flag.item()), want,
                          out.hi[:, c], out.lo[:, c], out32[:, c])


DENSE = [
    # name, ks, stride, pad, up, c_in, c_out, variant, out_c0, extra channels after the slice, value channel
    ("3x3 s1", 3, 1, 1, 1, 64, 64, 0, 0, 0, 61),
    ("3x3 s2", 3, 2, 1, 1, 64, 128, 0, 0, 0, 77),
    ("1x1", 1, 1, 0, 1, 96, 32, 0, 0, 0, 30),
    ("ConvTranspose up 2", 1, 1, 0, 2, 64, 64, 0, 0, 0, 9),
    ("ConvTranspose up 3", 1, 1, 0, 3, 64, 128, 0, 0, 0, 100),
    ("ConvTranspose up 4", 1, 1, 0, 4, 32, 64, 0, 0, 0, 33),
    ("k = s = 2", 2, 2, 0, 1, 64, 128, 0, 0, 0, 3),
    ("k = s = 3", 3, 3, 0, 1, 64, 64, 0, 0, 0, 40),
    ("k = s = 4", 4, 4, 0, 1, 128, 32, 0, 0, 0, 17),
    ("cgroups 2 into a slice", 3, 1, 1, 1, 64, 256, 0, 64, 64, 128 + 9),
]


@pytest.mark.parametrize("name,ks,stride,pad,up,c_in,c_out,variant,c0,extra,c", DENSE, ids=[d[0] for d in DENSE])
def test_dense_fp16x3_guard(name, ks, stride, pad, up, c_in, c_out, variant, c0, extra, c):
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16
    b, h, w = 2, 19, 23
    g = torch.Generator(device="cuda").manual_seed(ks * 100 + up * 10 + c_out + variant)
    x = conv16.Planes.from_f32(torch.randn((b, h, w, c_in), device="cuda", generator=g))
    wt = torch.randn((up * up, ks * ks, c_in, c_out), device="cuda", generator=g) / math.sqrt(ks * ks * c_in)
    wt[..., c] = 0.0
    total = c0 + c_out + extra
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        _lib.lib().d3b_set_bev_variant(variant)
        for relu in (False, True):
            for v, e, want in _cases(relu):
                bias, scale, shift = _epi(c_out, c, c_out, v)
                layer = dense_layer(wt, ks, stride, pad, up, bias=bias, scale=scale, shift=shift, relu=relu)
                assert layer.cgroups == (2 if c_out == 256 else 1)
                ho, wo = layer.out_hw(h, w)
                out = conv16.Planes((b, ho, wo, total), "cuda", zero=True)
                out32 = torch.zeros((b, ho, wo, total), device="cuda")
                flag = _flag()
                layer(x, out=out, out_f32=out32, out_c0=c0, overflow=flag)
                what = "dense %s relu %d v = %r" % (name, relu, v)
                k = c0 + c
                check_written(what, e, int(flag.item()), want, out.hi[..., k], out.lo[..., k], out32[..., k])
                live = torch.zeros(total, dtype=torch.bool, device="cuda")
                live[c0:c0 + c_out] = True
                live[k] = False
                assert bool(torch.isfinite(out32[..., live]).all()) and float(out32[..., live].abs().max()) < 100.0
                assert float(out32[..., :c0].abs().max() if c0 else 0.0) == 0.0, "%s: wrote below its slice" % what
                assert float(out32[..., c0 + c_out:].abs().max() if extra else 0.0) == 0.0, "%s: wrote past its slice" % what
    finally:
        _lib.lib().d3b_set_bev_variant(prev)


# ---------------------------------------------------------------------------------------------------------------------
# detector level: inject, re-run, compare with the CPU oracle
# ---------------------------------------------------------------------------------------------------------------------

OVERFLOW, CONTROL = 7.0e4, 6.0e4


def _unmatched(want_boxes, got_boxes, tol):
    if want_boxes.shape[0] == 0:
        return 0
    if got_boxes.shape[0] == 0:
        return int(want_boxes.shape[0])
    d = (want_boxes[:, None, :] - got_boxes[None, :, :]).abs().max(-1)[0]
    return int((d.min(1)[0] > tol).sum())


def _config(name):
    from det3d.torchie import Config
    return Config.fromfile(os.path.join(ROOT, "configs", name))


def _pillars_kitti():
    from det3d.models import build_detector
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud, uniform_cloud
    from oracle.pillars_cpu import PillarsCPU
    cfg = _config("pointpillars_kitti_car.py")
    torch.manual_seed(0)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 0)
    rng = cfg.voxel_generator.range
    calibrate_demo_weights_(model, cfg, [uniform_cloud(20000, rng, 4, 70), lidar_like_cloud(20000, rng, 4, 71)], 0,
                            pass_fraction=0.02)
    clouds = [uniform_cloud(20000, rng, 4, 7), lidar_like_cloud(20000, rng, 4, 8)]
    return cfg, model, clouds, PillarsCPU


def _pillars_nusc():
    from test_pillars_nusc import N_POINTS, _demo_model, shipped_config
    from det3d_b200.utils.synthetic import lidar_like_cloud
    from oracle.pillars_nusc_cpu import PillarsNuscCPU
    cfg = shipped_config()
    model = _demo_model(cfg)
    return cfg, model, [lidar_like_cloud(N_POINTS, cfg.voxel_generator.range, 5, 301)], PillarsNuscCPU


def _second():
    from det3d.models import build_detector
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud
    from oracle.second_cpu import SecondCPU
    cfg = _config("second_kitti_car.py")
    torch.manual_seed(0)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 0)
    rng = cfg.voxel_generator.range
    calibrate_demo_weights_(model, cfg, [lidar_like_cloud(20000, rng, 4, 900 + i) for i in range(2)], 0)
    return cfg, model, [lidar_like_cloud(20000, rng, 4, 1)], SecondCPU


def _cbgs():
    from det3d.models import build_detector
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud
    from oracle.cbgs_cpu import CbgsCPU
    cfg = _config("cbgs_nusc.py")
    torch.manual_seed(1)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 1)
    rng = cfg.voxel_generator.range
    calibrate_demo_weights_(model, cfg, [lidar_like_cloud(35000, rng, 5, 50 + i) for i in range(2)], 1,
                            pass_fraction=0.01)
    return cfg, model, [lidar_like_cloud(35000, rng, 5, 2)], CbgsCPU


_BUILDERS = {"pillars_kitti": _pillars_kitti, "pillars_nusc": _pillars_nusc, "second": _second, "cbgs": _cbgs}


@pytest.fixture(scope="module")
def calibrated():
    """One calibrated model per configuration, built on first use: (cfg, CPU state dict, clouds, oracle class)."""
    cache = {}

    def get(name):
        if name not in cache:
            cfg, model, clouds, oracle = _BUILDERS[name]()
            sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
            cache[name] = (cfg, sd, clouds, oracle)
        return cache[name]
    return get


def _bn_site(bn, c, bias):
    bn.weight[c] = 0.0
    bn.bias[c] = bias


def _inject_pillars_reader(model, bias, c=11):
    """Pillar feature channel c = bias for every pillar (BN weight 0 before the ReLU and the max); its only consumer is
    the first (strided) conv of RPN block 0."""
    _bn_site(model.reader.pfn_layers[0].norm, c, bias)
    model.neck.blocks[0][1].weight[:, c] = 0.0


def _inject_rpn_block_conv(model, bias, c=5):
    """The BN after RPN block 0's first conv; its only consumer is the next conv of the block."""
    _bn_site(model.neck.blocks[0][2], c, bias)
    model.neck.blocks[0][4].weight[:, c] = 0.0


def _inject_sparse(layer_bn, consumer):
    def inject(model, bias, c=3):
        mc = model.backbone.middle_conv
        _bn_site(mc[layer_bn], c, bias)
        mc[consumer].weight[..., c, :] = 0.0
    return inject


def _inject_cbgs_residual_chain(model, bias, c=20):
    """The BN after the strided conv 16 -> 32: its output is the identity of the two residual blocks that follow, so
    channel c carries about `bias` through both; every conv that reads it (the blocks' first convs and the next strided
    conv) gets zero weights on it."""
    mc = model.backbone.middle_conv
    _bn_site(mc[6], c, bias)
    for blk in (mc[8], mc[9]):
        blk.conv1.weight[..., c, :] = 0.0
    mc[10].weight[..., c, :] = 0.0


SITES = [
    # config, site, injection, graphed
    ("pillars_kitti", "reader", _inject_pillars_reader, True),
    ("pillars_kitti", "rpn_block0_conv", _inject_rpn_block_conv, False),
    ("pillars_nusc", "reader", _inject_pillars_reader, False),
    ("second", "first_sparse_layer", _inject_sparse(1, 3), True),      # spconv_first16_kernel -> epilogue16
    ("second", "middle_sparse_layer", _inject_sparse(19, 21), False),  # subm2 64 -> 64, tensor-core kernel
    ("second", "rpn_block0_conv", _inject_rpn_block_conv, False),
    ("cbgs", "resnet_encoder", _inject_cbgs_residual_chain, False),
]


def _compare(config, cfg, want, got, stages):
    """-> (ok, report).  PointPillars re-runs on the fp32 torch modules: the detection set must equal the oracle's up to
    counted near-ties.  SECOND / CBGS re-run on the tf32x3 kernels (uncorrected truncating accumulation): at most a
    tenth of the detections may differ by more than 2e-3."""
    thr, pre = cfg.test_cfg.score_threshold, cfg.test_cfg.nms.nms_pre_max_size
    report, ok, total = [], True, 0
    for b in range(len(want)):
        w, g = want[b]["box3d_lidar"], got[b]["box3d_lidar"]
        total += w.shape[0]
        if config.startswith("pillars"):
            heads = stages["heads"] if "heads" in stages else [dict(cls=stages["cls"])]
            fragile = 0
            for h in heads:
                sc = torch.sigmoid(h["cls"][b].reshape(-1))
                top = sc[sc >= thr].sort(descending=True)[0][:pre]
                fragile += int(((top[:-1] - top[1:]) < 2e-6).sum()) + int(((sc - thr).abs() < 2e-6).sum())
            missing, extra = _unmatched(w, g, 1e-3), _unmatched(g, w, 1e-3)
            allowed = fragile
        else:
            missing, extra = _unmatched(w, g, 2e-3), _unmatched(g, w, 2e-3)
            allowed = max(1, w.shape[0] // 10)
        ok &= missing <= allowed and extra <= allowed
        report.append("sample %d: oracle %d, device %d, %d missing, %d extra (allowed %d)"
                      % (b, w.shape[0], g.shape[0], missing, extra, allowed))
    ok &= total >= 5
    return ok, "; ".join(report)


def _run_site(calibrated, config, inject, bias, graphed):
    from det3d.models import build_detector
    from det3d_b200.apis import InferencePipeline
    cfg, sd, clouds, oracle = calibrated(config)
    model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    model.load_state_dict(sd)
    model.eval()
    with torch.no_grad():
        inject(model, bias)
    sd_mod = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    assert pipe.model.fused_bev() is not None and pipe.model.math == "fp16x3"
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        packed = pipe.infer_host([torch.from_numpy(c).pin_memory() for c in clouds], graphed=graphed).clone()
    warned = any("f16 range" in str(w.message) for w in caught)
    got = pipe.unpack(packed)
    cpu = oracle(cfg, sd_mod, [a.cpu().numpy() for a in pipe._anchors])
    stages = {}
    want = cpu.forward(clouds, stages)
    ok, report = _compare(config, cfg, want, got, stages)
    state = dict(warned=warned, math=pipe.model.math, flag=int(pipe.overflow_flag().item()),
                 graphs=[e.graph is not None for e in pipe._graphs.values()], finite=bool(torch.isfinite(packed).all()))
    return ok, "%s | %s" % (state, report), state


@pytest.mark.parametrize("config,site,inject,graphed", SITES, ids=["%s-%s" % s[:2] for s in SITES])
def test_injected_overflow_reruns_and_matches_the_oracle(calibrated, config, site, inject, graphed):
    ok, report, st = _run_site(calibrated, config, inject, OVERFLOW, graphed)
    assert st["warned"], "no f16-range warning: %s" % report
    assert st["math"] == "tf32x3", report
    assert st["flag"] == 0, report
    if graphed:
        assert st["graphs"] == [True], "the re-run's graph only: %s" % report
    assert st["finite"], report
    assert ok, "re-run detections differ from the oracle: %s" % report


@pytest.mark.parametrize("config,site,inject,graphed", SITES, ids=["%s-%s" % s[:2] for s in SITES])
def test_injected_control_stays_on_fp16x3_and_matches_the_oracle(calibrated, config, site, inject, graphed):
    ok, report, st = _run_site(calibrated, config, inject, CONTROL, graphed)
    assert not st["warned"] and st["math"] == "fp16x3" and st["flag"] == 0, report
    if graphed:
        assert st["graphs"] == [True], report
    assert ok, "FP16x3 detections differ from the oracle: %s" % report
