"""Single-pass FP16 (the opt-in math "fp16": one f16 plane per activation, one wgmma(A_hi, W_hi) per k-step) against its
own error model, its f16-range guard, and as a whole forward next to FP16x3.

Error model, per fp32 output of one layer fed fp32 (or float64-derived) activations a, with the quantities of
test_conv_error_model_gpu (float64 on the GPU):
* ``yh1`` = sum a_hi*w_hi, the exact sum of the operands the kernel multiplies (a_hi = f16(a), w_hi = f16(w*2^w_exp)
  scaled back);
* accumulation: a slot chains n = n_ks <= 4 MMAs into a fresh partial (the FP16x3 derivation with n = n_ks), so
      |got - yh1| <= c_acc1 M + u (1 + 2^-20) (sum_s |S_s| + |yh1|),   c_acc1 = (2 n 2^-23 + n eps)(1 + 2^-9);
* representation: rounding both operands to 11 significant bits,
      |yh1 - y| <= (2^-10 + 2^-22) M + 2^-25 sum|w| + 2^-25 2^-w_exp sum|a|,
  the last two terms being the f16-subnormal floors of activations and of scaled weights.  When the input already is an
  f16 plane (a = a_hi) the activation part vanishes: |yh1 - y| <= 2^-11 M + 2^-25 2^-w_exp sum|a|.
This model promises no parity with the reference's fp32 result: 2^-10 relative per product is three orders above the
FP16x3 contract.  The forward tests therefore compare detections with FP16x3's, and the predict with the oracle's predict
run on the device's own head outputs.
"""
import copy
import math
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_conv_error_model_gpu import (BOUNDARY, DENSE_CASES, EPS, SPARSE_CIN, SPARSE_COUT, U, _epi_params, _ksize, _level,
                                       _os16_pack, dense_layer, operands, weight_planes)
from test_encoder_deployed_gpu import LAYERS, RUN_OF, _layer_operands, deployed  # noqa: F401  (module fixture)
from test_f16_guard_gpu import OVERFLOW, SITES, _compare, calibrated  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu


def c_acc1(n_ks):
    return (2 * n_ks * 2.0 ** -23 + n_ks * EPS) * (1 + 2.0 ** -9)


class Ref1:
    """float64 pieces of one single-pass convolution, slot by slot in the kernel's order."""

    def __init__(self, shape, device):
        z = lambda: torch.zeros(shape, dtype=torch.float64, device=device)
        self.y, self.yh, self.M, self.sw, self.sa, self.run_abs, self.var, self.pabs = (z() for _ in range(8))
        self.n_ks = 1

    def slot(self, a, a_hi, w, w_hi, n_ks):
        self.n_ks = max(self.n_ks, n_ks)
        p = a_hi @ w_hi
        m = a.abs() @ w.abs()
        self.y += a @ w
        self.yh += p
        self.M += m
        self.sw += (a != 0).double() @ w.abs()
        self.sa += a.abs().sum(-1, keepdim=True)
        self.run_abs += self.yh.abs()
        self.pabs += p.abs()
        self.var += n_ks * (2 * 2.0 ** -23 * m) ** 2 + (U * self.yh) ** 2

    def elem_tol(self):
        return c_acc1(self.n_ks) * self.M + U * (1 + 2.0 ** -20) * (self.run_abs + self.yh.abs())


def check_model1(got, ref, w_exp, what, f16_input=False):
    got = got.double()
    live = ref.M > 0
    assert bool(live.any()), what
    assert torch.isfinite(got).all(), "%s: non-finite output" % what
    err = (got - ref.yh).abs()
    if bool((~live).any()):
        assert float(err[~live].max()) == 0.0, "%s: output without terms is not 0" % what
    tol = ref.elem_tol()
    worst = float((err[live] / tol[live]).max())
    assert worst <= 1.0, "%s: |got - yh1| reaches %.3g of the accumulation bound" % (what, worst)
    m = ref.M[live]
    rms = float(torch.sqrt((((got - ref.yh)[live] / m) ** 2).mean()))
    rms_tol = float(torch.sqrt(((ref.var[live] + (U * ref.yh[live]) ** 2) / m ** 2).mean())
                    + (4 * EPS * ref.pabs[live] / m).max())
    assert rms <= rms_tol, "%s: RMS relative error %.3g > %.3g" % (what, rms, rms_tol)
    wf = math.ldexp(1.0, -w_exp)
    rep = (2.0 ** -10 + 2.0 ** -22) * ref.M + 2.0 ** -25 * ref.sw + 2.0 ** -25 * wf * ref.sa
    assert bool(((ref.yh - ref.y).abs() <= rep).all()), "%s: |yh1 - y| exceeds its bound" % what
    if f16_input:
        tight = 2.0 ** -11 * ref.M + 2.0 ** -25 * wf * ref.sa
        assert bool(((ref.yh - ref.y).abs() <= tight).all()), "%s: |yh1 - y| exceeds the f16-input bound" % what
    return dict(worst=worst, rms=rms, rel=float(((got - ref.y).abs()[live] / m).max()))


# ---------------------------------------------------------------------------------------------------------------------
# per kernel
# ---------------------------------------------------------------------------------------------------------------------

def sparse_ref1(x, planes, w, w_exp, nbr, n_out):
    k_vol, c_in, c_out = w.shape
    dev = w.device
    a, a_hi = x.double(), planes.hi.double()
    w64 = w.double()
    w_hi, _ = weight_planes(w, w_exp)
    pack = _os16_pack(c_in, k_vol)
    ref = Ref1((n_out, c_out), dev)
    zero = torch.zeros((1, c_in), dtype=torch.float64, device=dev)

    def gather(t, k):
        idx = nbr[k, :n_out].long()
        return torch.cat([t, zero])[torch.where(idx >= 0, idx, t.shape[0])]

    for g in range(0, k_vol, pack):
        ks = list(range(g, min(g + pack, k_vol)))
        if pack > 1:
            ga = [torch.cat([gather(t, k) for k in ks], 1) for t in (a, a_hi)]
            ref.slot(ga[0], ga[1], torch.cat([w64[k] for k in ks]), torch.cat([w_hi[k] for k in ks]), 4)
        else:
            ga = [gather(t, g) for t in (a, a_hi)]
            for kb in range(0, c_in, 64):
                sl = slice(kb, min(kb + 64, c_in))
                ref.slot(ga[0][:, sl], ga[1][:, sl], w64[g][sl], w_hi[g][sl], min(4, (c_in - kb + 15) // 16))
    return ref


def run_sparse1(c_in, c_out, k_vol, n, seed, a_scale=1.0, w_max=None, regime="C", n_dev=None, spatial=(9, 40, 36),
                f16_input=False):
    from det3d_b200.ops.spconv import conv16, core
    gen = torch.Generator(device="cuda").manual_seed(seed)
    lvl = _level(n, spatial, 2, seed)
    if n_dev is not None:
        lvl.n.fill_(n_dev)
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, _ksize(k_vol)))
    n_out = n if n_dev is None else n_dev
    x, w = operands((n, c_in), (k_vol, c_in, c_out), regime, gen, a_scale, w_max)
    if f16_input:
        x = x.half().float()
    cw = conv16.ConvWeights16(w)
    planes = conv16.Planes.from_f32(x, n_planes=1)
    assert planes.lo is None
    out = torch.full((max(n, 1), c_out), float("nan"), device="cuda")
    conv16.sparse_conv16(planes, rb, cw, None, out_f32=out)
    return out, sparse_ref1(x, planes, w, cw.w_exp, rb.nbr, n_out), cw, rb, planes, x, w, n_out


@pytest.mark.parametrize("c_in", SPARSE_CIN)
@pytest.mark.parametrize("c_out", SPARSE_COUT)
def test_sparse_fp16_error_model(c_in, c_out):
    out, ref, cw, *_ = run_sparse1(c_in, c_out, 27, 1500, c_in * 7 + c_out)
    check_model1(out[:1500], ref, cw.w_exp, "sparse fp16 C_in %d C_out %d" % (c_in, c_out))


@pytest.mark.parametrize("k_vol", [3, 1])
@pytest.mark.parametrize("c_in", [16, 32])
@pytest.mark.parametrize("c_out", [16, 64])
def test_sparse_fp16_small_kernels(k_vol, c_in, c_out):
    out, ref, cw, *_ = run_sparse1(c_in, c_out, k_vol, 2000, 31 * k_vol + c_in + c_out)
    check_model1(out[:2000], ref, cw.w_exp, "sparse fp16 k_vol %d C_in %d" % (k_vol, c_in))


@pytest.mark.parametrize("n,n_dev", [(1000, None), (1001, None), (1001, 700), (1001, 0), (1, None), (300 * 128 + 5, None)])
def test_sparse_fp16_row_counts(n, n_dev):
    out, ref, cw, rb, planes, x, w, n_out = run_sparse1(32, 64, 27, n, n + 3, n_dev=n_dev, spatial=(20, 60, 60))
    assert bool(torch.isnan(out[n_out:]).all()), "rows past the live count were written"
    if n_out:
        check_model1(out[:n_out], ref, cw.w_exp, "sparse fp16 rows %d/%d" % (n_out, n))


@pytest.mark.parametrize("c_in", [64, 32])
def test_sparse_fp16_input_already_f16(c_in):
    """Activations that are f16 numbers: the representation bound loses its activation-rounding part."""
    out, ref, cw, *_ = run_sparse1(c_in, 64, 27, 1500, 77 + c_in, f16_input=True)
    check_model1(out[:1500], ref, cw.w_exp, "sparse fp16 f16 input C_in %d" % c_in, f16_input=True)


@pytest.mark.parametrize("c_in", [3, 4, 5, 9, 15])
@pytest.mark.parametrize("c_out", [16, 32, 64])
def test_sparse_first_layer_fp16(c_in, c_out):
    """The FFMA first layer computes the same fp32 sums in both maths; the single-plane launch writes hi = f16(v) of
    them, bit for bit the FP16x3 launch's hi plane."""
    from det3d_b200.ops.spconv import conv16, core
    gen = torch.Generator(device="cuda").manual_seed(c_in * 13 + c_out)
    n = 3000
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(_level(n, (9, 40, 36), 2, c_in + c_out), 3))
    x, w = operands((n, c_in), (27, c_in, c_out), "C", gen)
    cw = conv16.ConvWeights16(w, bias=torch.randn(c_out, device="cuda") * 0.1, relu=True)
    assert cw.fp32_input
    outs = []
    for n_planes in (2, 1):
        o = conv16.Planes((n, c_out), "cuda", n_planes=n_planes)
        f = torch.empty((n, c_out), device="cuda")
        conv16.sparse_conv16(x, rb, cw, o, out_f32=f)
        outs.append((o, f))
    assert torch.equal(outs[0][1], outs[1][1])
    assert torch.equal(outs[0][0].hi, outs[1][0].hi)
    assert torch.equal(outs[1][0].hi, outs[1][1].half())


def test_sparse_fp16_epilogue_and_residual():
    """bias, folded BN, the hi plane of the residual, ReLU; the output plane is f16(v) of the fp32 output."""
    from det3d_b200.ops.spconv import conv16
    out, ref, cw, rb, planes, x, w, n_out = run_sparse1(48, 64, 27, 3000, 5)
    bias, scale, shift = _epi_params(64, 5)
    res = conv16.Planes.from_f32(torch.randn((3000, 64), device="cuda"), n_planes=1)
    e = conv16.ConvWeights16(w, bias=bias, scale=scale, shift=shift, relu=True)
    o = conv16.Planes((3000, 64), "cuda", n_planes=1)
    o32 = torch.empty((3000, 64), device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    conv16.sparse_conv16(planes, rb, e, o, residual=res, out_f32=o32, overflow=flag)
    assert int(flag.item()) == 0
    v = (ref.yh + bias.double()) * scale.double() + shift.double() + res.hi.double()
    tol = ref.elem_tol() * scale.double().abs() + 4 * U * (v.abs() + 1)
    assert bool(((o32.double() - torch.relu(v)).abs() <= tol).all())
    assert torch.equal(o.hi, o32.half())


def dense_ref1(x, planes, wt, w_exp, ks, stride, pad, up):
    b, h, w, c_in = x.shape
    c_out = wt.shape[-1]
    ho, wo = (h + 2 * pad - ks) // stride + 1, (w + 2 * pad - ks) // stride + 1
    padf = lambda t: torch.nn.functional.pad(t.double(), (0, 0, pad, pad, pad, pad))
    xs = [padf(t) for t in (x, planes.hi)]
    w_hi, _ = weight_planes(wt, w_exp)
    w64 = wt.double()
    full = Ref1((b, ho * up, wo * up, c_out), x.device)
    for g in range(up * up):
        ref = Ref1((b, ho, wo, c_out), x.device)
        for kb in range(0, c_in, 64):
            sl = slice(kb, min(kb + 64, c_in))
            for kx in range(ks):
                for ky in range(ks):
                    win = [t[:, ky:ky + stride * (ho - 1) + 1:stride, kx:kx + stride * (wo - 1) + 1:stride, sl] for t in xs]
                    ref.slot(*win, w64[g, ky * ks + kx, sl], w_hi[g, ky * ks + kx, sl], min(4, (c_in - kb + 15) // 16))
        for name in ("y", "yh", "M", "sw", "sa", "run_abs", "var", "pabs"):
            getattr(full, name)[:, g // up::up, g % up::up] = getattr(ref, name)
        full.n_ks = max(full.n_ks, ref.n_ks)
    return full


def run_dense1(b, h, w, c_in, c_out, ks, stride, pad, up, seed, a_scale=1.0, w_max=None, regime="C"):
    from det3d_b200.ops.spconv import conv16
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x, wt = operands((b, h, w, c_in), (up * up, ks * ks, c_in, c_out), regime, gen, a_scale, w_max)
    layer = dense_layer(wt, ks, stride, pad, up)
    planes = conv16.Planes.from_f32(x, n_planes=1)
    ho, wo = layer.out_hw(h, w)
    out = torch.full((b, ho, wo, layer.c_out_padded), float("nan"), device="cuda")
    layer(planes, out_f32=out)
    return out[..., :c_out], dense_ref1(x, planes, wt, layer.w_exp, ks, stride, pad, up), layer, planes, x, wt


@pytest.mark.parametrize("b,h,w,c_in,c_out,ks,stride,pad,up", DENSE_CASES + [
    (1, 21, 35, 128, 128, 3, 1, 1, 1), (2, 17, 23, 64, 64, 2, 2, 0, 1), (1, 31, 29, 64, 128, 3, 3, 0, 1),
    (2, 33, 41, 128, 128, 4, 4, 0, 1)])
def test_dense_fp16_error_model(b, h, w, c_in, c_out, ks, stride, pad, up):
    """Both dense schedules (the pipelined one serves 3x3 s1 with 128-channel blocks and C_in % 64 == 0), strides, 1x1,
    ConvTranspose up 2/3/4, Conv2d(k = s) 2/3/4; then the fused epilogue and the single output plane."""
    from det3d_b200.ops.spconv import conv16
    seed = b * 1000 + h * 31 + c_in + c_out + 7 * up + ks
    got, ref, layer, planes, x, wt = run_dense1(b, h, w, c_in, c_out, ks, stride, pad, up, seed)
    what = "dense fp16 %s" % ((b, h, w, c_in, c_out, ks, stride, pad, up),)
    check_model1(got, ref, layer.w_exp, what)
    bias, scale, shift = _epi_params(c_out, seed)
    epi = dense_layer(wt, ks, stride, pad, up, bias=bias, scale=scale, shift=shift, relu=True)
    ho, wo = epi.out_hw(h, w)
    out = conv16.Planes((b, ho, wo, epi.c_out_padded), "cuda", zero=True, n_planes=1)
    out32 = torch.zeros((b, ho, wo, epi.c_out_padded), device="cuda")
    epi(planes, out=out, out_f32=out32)
    v = torch.relu((ref.yh + bias.double()) * scale.double() + shift.double())
    tol = ref.elem_tol() * scale.double().abs() + 4 * U * (v.abs() + 1)
    assert bool(((out32[..., :c_out].double() - v).abs() <= tol).all()), what
    assert torch.equal(out.hi, out32.half())


@pytest.mark.parametrize("c_in,b,c_out", [(64, 1, 128), (192, 3, 128), (128, 3, 256)])
def test_dense_fp16_pipelined_bit_identical(c_in, b, c_out):
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16
    gen = torch.Generator(device="cuda").manual_seed(c_in + b)
    x, wt = operands((b, 21, 35, c_in), (1, 9, c_in, c_out), "B", gen)
    bias, scale, shift = _epi_params(c_out, c_in)
    layer = dense_layer(wt, 3, 1, 1, 1, bias=bias, scale=scale, shift=shift, relu=True)
    planes = conv16.Planes.from_f32(x, n_planes=1)
    outs = []
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        for variant in (0, 2):
            _lib.lib().d3b_set_bev_variant(variant)
            out = conv16.Planes((b, 21, 35, c_out), "cuda", zero=True, n_planes=1)
            out32 = torch.zeros((b, 21, 35, c_out), device="cuda")
            layer(planes, out=out, out_f32=out32)
            outs.append((out.buf, out32))
    finally:
        _lib.lib().d3b_set_bev_variant(prev)
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("a_exp", [-14, -12, -6, 0, 6, 12])
@pytest.mark.parametrize("w_exp", [-30, -10, 0, 10])
def test_sparse_fp16_magnitude_sweep(a_exp, w_exp):
    """Down to the f16-subnormal end of the activations (2^-14 and below) and up towards 65504."""
    out, ref, cw, *_ = run_sparse1(64, 64, 27, 1500, 5000 + a_exp * 50 + w_exp, a_scale=2.0 ** a_exp, w_max=2.0 ** w_exp)
    check_model1(out[:1500], ref, cw.w_exp, "sparse fp16 2^%d x 2^%d" % (a_exp, w_exp))


@pytest.mark.parametrize("a_exp,w_exp", [(k, 0) for k in (-14, -6, 0, 6, 12)] + [(0, j) for j in (-30, -10, 10)])
def test_dense_fp16_magnitude_sweep(a_exp, w_exp):
    got, ref, layer, *_ = run_dense1(2, 19, 23, 96, 64, 3, 1, 1, 1, 5000 + a_exp * 50 + w_exp, a_scale=2.0 ** a_exp,
                                     w_max=2.0 ** w_exp)
    check_model1(got, ref, layer.w_exp, "dense fp16 2^%d x 2^%d" % (a_exp, w_exp))


def test_fp16_correction_bias():
    """Residual slope of the single-pass kernels against yh1 over large launches (regime B): within the 4 eps of one
    slot's correction, and a kernel with the FP16x3 correction (12 eps) would be rejected."""
    from det3d_b200 import _lib
    from test_conv_error_model_gpu import residual_slope
    out, ref, *_ = run_sparse1(64, 64, 27, 20000, 11, regime="B", spatial=(20, 100, 100))
    cases = [("sparse", out[:20000], ref)]
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        for v in (0, 2):
            _lib.lib().d3b_set_bev_variant(v)
            got, r, *_ = run_dense1(1, 96, 88, 128, 128, 3, 1, 1, 1, 23, regime="B")
            cases.append(("dense_v%d" % v, got, r))
    finally:
        _lib.lib().d3b_set_bev_variant(prev)
    for name, got, r in cases:
        beta, se = residual_slope(got, r.yh)
        print("fp16 %s regime B: beta = %+.3f eps (se %.3f eps)" % (name, beta / EPS, se / EPS))
        assert abs(beta) <= 2 * EPS, name
        assert abs(residual_slope(got.double() * (1 + 8 * EPS), r.yh)[0]) > 2 * EPS


# ---------------------------------------------------------------------------------------------------------------------
# the lo buffer is never touched, and the guard
# ---------------------------------------------------------------------------------------------------------------------

def test_single_plane_launches_never_write_a_lo_buffer():
    """Sentinel-filled lo halves next to single-plane buffers: sparse_to_bev16 (plane-copy and fp32 paths), split16 and the
    convolutions leave them untouched (the single-plane views are the first half of a two-plane allocation)."""
    from det3d_b200.ops.spconv import conv16, core
    sentinel = torch.tensor(12345.0, dtype=torch.float16)

    def single_view(shape):
        two = conv16.Planes(shape, "cuda")
        two.buf[1].fill_(sentinel)
        one = conv16.Planes.__new__(conv16.Planes)
        one.buf, one.shape = two.buf[:1], two.shape
        return two, one

    lvl = _level(900, (2, 30, 40), 2, 3)
    rows = torch.randn((900, 32), device="cuda")
    r2, r1 = single_view((900, 32))
    conv16.Planes.from_f32(rows, out=r1)
    assert torch.equal(r1.hi, rows.half()) and bool((r2.buf[1] == sentinel).all())
    assert torch.equal(r1.to_f32(), rows.half().float())
    b2, b1 = single_view((2, 30, 40, 64))
    b1.zero_()
    conv16.sparse_to_bev16(r1, lvl, b1)
    assert bool((b2.buf[1] == sentinel).all())
    f2, f1 = single_view((2, 30, 40, 64))
    f1.zero_()
    conv16.sparse_to_bev16(rows, lvl, f1)
    assert bool((f2.buf[1] == sentinel).all()) and torch.equal(f1.buf, b1.buf)
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, 3))
    o2, o1 = single_view((900, 64))
    conv16.sparse_conv16(r1, rb, conv16.ConvWeights16(torch.randn((27, 32, 64), device="cuda") * 0.05), o1)
    assert bool((o2.buf[1] == sentinel).all())
    d2, d1 = single_view((2, 30, 40, 128))
    dense_layer(torch.randn((1, 9, 64, 128), device="cuda") * 0.05, 3, 1, 1, 1)(b1, out=d1)
    assert bool((d2.buf[1] == sentinel).all())


def test_single_plane_guard_at_the_boundary():
    """split16, the sparse epilogue (with and without ReLU and residual), the first layer, both dense schedules and the
    fp32-row scatter flag exactly when |v| >= 65504 or v is inf / NaN; an out_f32-only launch never does."""
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16, core
    for v, want in BOUNDARY:
        flag = torch.zeros(1, dtype=torch.int32, device="cuda")
        conv16.Planes.from_f32(torch.tensor([[0.5, v, -2.0, 3.0]], device="cuda"), flag, n_planes=1)
        assert int(flag.item()) == want, "split16(%r)" % v
    lvl = _level(300, (9, 40, 36), 1, 1)
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, 3))
    xin = conv16.Planes.from_f32(torch.randn((300, 32), device="cuda"), n_planes=1)
    x4 = torch.randn((300, 4), device="cuda")
    zero_res = conv16.Planes((300, 128), "cuda", zero=True, n_planes=1)
    zero_res64 = conv16.Planes((300, 64), "cuda", zero=True, n_planes=1)
    grid = conv16.Planes.from_f32(torch.randn((1, 9, 11, 64), device="cuda"), n_planes=1)
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        for v, want in BOUNDARY:
            bias = torch.zeros(128, device="cuda")
            bias[5] = v
            # ReLU keeps a positive v and writes 0 for a negative one or NaN (fmaxf): the flag follows the written value
            for relu in (False, True):
                want_r = want if not relu or v > 0 else 0
                for res in (None, zero_res):
                    cw = conv16.ConvWeights16(torch.zeros((27, 32, 128), device="cuda"), bias=bias, relu=relu)
                    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
                    conv16.sparse_conv16(xin, rb, cw, conv16.Planes((300, 128), "cuda", n_planes=1), residual=res,
                                         overflow=flag)
                    assert int(flag.item()) == want_r, "sparse epilogue v = %r relu %s res %s" % (v, relu, res is not None)
            flag = torch.zeros(1, dtype=torch.int32, device="cuda")
            conv16.sparse_conv16(xin, rb, cw, None, out_f32=torch.empty((300, 128), device="cuda"), overflow=flag)
            assert int(flag.item()) == 0
            for relu in (False, True):
                want_r = want if not relu or v > 0 else 0
                for res in (None, zero_res):
                    cw1 = conv16.ConvWeights16(torch.zeros((27, 4, 64), device="cuda"), bias=bias[:64], relu=relu)
                    flag.zero_()
                    conv16.sparse_conv16(x4, rb, cw1, conv16.Planes((300, 64), "cuda", n_planes=1), overflow=flag,
                                         residual=None if res is None else zero_res64)
                    assert int(flag.item()) == want_r, "first layer v = %r relu %s res %s" % (v, relu, res is not None)
                layer = dense_layer(torch.zeros((1, 9, 64, 128), device="cuda"), 3, 1, 1, 1, bias=bias, relu=relu)
                for variant in (0, 2):
                    _lib.lib().d3b_set_bev_variant(variant)
                    flag.zero_()
                    layer(grid, out=conv16.Planes((1, 9, 11, 128), "cuda", n_planes=1), overflow=flag)
                    assert int(flag.item()) == want_r, "dense (variant %d) v = %r relu %s" % (variant, v, relu)
            flag.zero_()
            rows = torch.full((300, 64), 0.5, device="cuda")
            rows[7, 3] = v
            out = conv16.Planes((1, 40, 36, 64 * 9), "cuda", zero=True, n_planes=1)
            conv16.sparse_to_bev16(rows, lvl, out, overflow=flag)
            assert int(flag.item()) == want, "fp32-row scatter v = %r" % v
    finally:
        _lib.lib().d3b_set_bev_variant(prev)


# an overflow injected into the fp16 forward: the sites of test_f16_guard_gpu on SECOND, PointPillars and CBGS
FP16_SITES = [(c, site, inject, graphed) for c, site, inject, _g in SITES if c in ("second", "pillars_kitti", "cbgs")
              for graphed in (False, True)]


@pytest.mark.parametrize("config,site,inject,graphed", FP16_SITES,
                         ids=["%s-%s-%s" % (s[0], s[1], "graphed" if s[3] else "eager") for s in FP16_SITES])
def test_injected_overflow_in_fp16_reruns_on_tf32x3_and_matches_the_oracle(calibrated, config, site, inject, graphed):  # noqa: F811
    """The pipeline is put in "fp16" and its first attempt runs on one-plane buffers; a feature past 65504 raises the
    flag, the pipeline warns, switches to tf32x3, drops the fp16 graph and returns the oracle's detections."""
    import warnings
    from det3d.models import build_detector
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.ops.spconv import conv16
    cfg, sd, clouds, oracle = calibrated(config)
    model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    model.load_state_dict(sd)
    model.eval()
    with torch.no_grad():
        inject(model, OVERFLOW)
    sd_mod = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    pipe.set_math("fp16")
    bev16 = pipe.model.fused_bev()
    assert pipe.model.math == "fp16" and type(bev16).__name__ == "FusedBevStack"

    def plane_counts():
        """(math, plane counts of the buffers the dense stack, the encoder / scatter wrote) when the flag is read."""
        planes = [p for p in bev16._bufs.values() if isinstance(p, conv16.Planes)]
        fused = getattr(pipe.model.backbone, "fused", None)
        if fused is not None:
            st = fused()._state
            planes += [p for k, pool in st["pools"].items() if k[0] == "p16" for p in pool] + [st["bev_planes"]]
        else:
            planes += list(pipe.model.backbone._planes.values())
        return pipe.model.math, [p.n_planes for p in planes]

    seen, check = [], pipe.check_overflow

    def spy(flag_value):
        seen.append(plane_counts())
        return check(flag_value)

    pipe.check_overflow = spy
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        packed = pipe.infer_host([torch.from_numpy(c).pin_memory() for c in clouds], graphed=graphed).clone()
    # the first attempt ran single-pass, on one-plane buffers only
    math_, counts = seen[0]
    assert math_ == "fp16" and counts and set(counts) == {1}, seen[0]
    assert any("f16 range" in str(w.message) for w in caught), "no f16-range warning"
    assert pipe.model.math == "tf32x3"
    assert int(pipe.overflow_flag().item()) == 0
    if graphed:
        assert [e.graph is not None for e in pipe._graphs.values()] == [True], "the re-run's graph only"
    assert bool(torch.isfinite(packed).all())
    cpu = oracle(cfg, sd_mod, [a.cpu().numpy() for a in pipe._anchors])
    stages = {}
    want = cpu.forward(clouds, stages)
    ok, report = _compare(config, cfg, want, pipe.unpack(packed), stages)
    assert ok, "re-run detections differ from the oracle: %s" % report


# ---------------------------------------------------------------------------------------------------------------------
# deployed encoder layers
# ---------------------------------------------------------------------------------------------------------------------

WORST = {}


@pytest.mark.parametrize("config,layer", LAYERS, ids=["%s-L%02d" % t for t in LAYERS])
def test_deployed_layer_vs_fp16_model(deployed, config, layer):  # noqa: F811
    from det3d_b200.ops.spconv import conv16
    *_, run = deployed(RUN_OF[config])
    L, rb, rec, w, x, n_out = _layer_operands(run, layer)
    cw = conv16.ConvWeights16(w)
    if cw.fp32_input:
        pytest.skip("the FFMA first layer computes the same fp32 sums in both maths (test_sparse_first_layer_fp16)")
    planes = conv16.Planes.from_f32(x, n_planes=1)
    raw = torch.full((rb.out_level.cap, w.shape[2]), float("nan"), device="cuda")
    conv16.sparse_conv16(planes, rb, cw, None, out_f32=raw)
    ref = sparse_ref1(x, planes, w, cw.w_exp, rb.nbr, n_out)
    st = check_model1(raw[:n_out], ref, cw.w_exp, "%s layer %d" % (config, layer))
    print("%s layer %d: worst |got - yh1| / bound %.3f, max |got - y| / M %.3g" % (config, layer, st["worst"], st["rel"]))


# ---------------------------------------------------------------------------------------------------------------------
# whole forward
# ---------------------------------------------------------------------------------------------------------------------

def _config(name):
    from det3d.torchie import Config
    return Config.fromfile(os.path.join(ROOT, "configs", name))


def _build(name):
    """(cfg, calibrated model, clouds of the deployed batch) as the existing end-to-end tests seed and calibrate them."""
    from det3d.models import build_detector
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud
    if name == "second":
        cfg, seed, n, b, nf, kw = _config("second_kitti_car.py"), 0, 20000, 1, 4, {}
    elif name == "pillars":
        cfg, seed, n, b, nf, kw = _config("pointpillars_kitti_car.py"), 0, 20000, 8, 4, dict(pass_fraction=0.02)
    else:
        cfg, seed, n, b, nf, kw = _config("cbgs_nusc.py"), 1, 35000, 4, 5, dict(pass_fraction=0.01)
    r = cfg.voxel_generator.range
    torch.manual_seed(seed)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), seed)
    calib_seed = {"second": 900, "pillars": 70, "cbgs": 50}[name]
    calibrate_demo_weights_(model, cfg, [lidar_like_cloud(n, r, nf, calib_seed + i) for i in range(2)], seed, **kw)
    clouds = [lidar_like_cloud(n - 500 * i, r, nf, 300 + i) for i in range(b)]
    return cfg, model, clouds


FORWARD = {}


def _forward(name):
    """Both maths on the same calibrated weights and clouds (built once per config)."""
    if name in FORWARD:
        return FORWARD[name]
    from det3d_b200.apis import InferencePipeline
    cfg, model, clouds = _build(name)
    out = dict(cfg=cfg, clouds=clouds, sd={k: v.detach().cpu().clone() for k, v in model.state_dict().items()})
    pipes = {}
    for math_ in ("fp16x3", "fp16"):
        pipe = InferencePipeline(cfg, model=copy.deepcopy(model), device="cuda")
        pipe.set_math(math_)
        pts = torch.from_numpy(np.concatenate(clouds)).cuda()
        offsets = np.cumsum([0] + [c.shape[0] for c in clouds]).tolist()
        with torch.no_grad():
            vox = pipe.voxelizer(pts, offsets)
            B = len(clouds)
            heads = _heads(pipe, vox, B)
            det = pipe.pack(pipe.forward_device(pts, offsets)).clone()
        out[math_] = dict(heads=heads, packed=det, counts=vox["counts"].clone(),
                          coors=vox["coors"][:int(vox["counts"][B])].clone(), flag=int(pipe.overflow_flag().item()))
        pipes[math_] = (pipe, pts, offsets)
    out["pipes"] = pipes
    FORWARD[name] = out
    return out


def _heads(pipe, vox, B):
    model = pipe.model
    grid = [int(g) for g in pipe.grid_size]
    n_dev = vox["counts"][B:B + 1]
    if hasattr(model.backbone, "fused"):
        planes = model.backbone.forward_planes(vox["mean"], vox["coors"], B, grid, n_dev=n_dev)
    else:
        feats = model._read(dict(features=vox.get("voxels"), num_voxels=vox["num_points"], coors=vox["coors"], n_dev=n_dev,
                                 point_lists=dict(vox["point_lists"], counts=vox["counts"]) if pipe._reader_takes_lists
                                 else None))
        planes = model.backbone.forward_planes(feats, vox["coors"], B, grid, n_dev=n_dev, n_planes=model.n_planes())
    assert planes.n_planes == model.n_planes()
    return [{k: v.clone() for k, v in d.items()} for d in model.fused_bev().run(planes)]


def _oracle_predict(pipe, cfg, heads, B):
    from oracle.predict_cpu import predict_sample_task
    head = pipe.model.bbox_head
    want = [dict(b=[], s=[], l=[]) for _ in range(B)]
    flag = 0
    for t, p in enumerate(heads):
        anchors = pipe._anchors[t].cpu()
        n_cls = head.num_classes[t]
        code = p["box_preds"][0].numel() // anchors.shape[0]
        for b in range(B):
            bx, sc, lb = predict_sample_task(p["cls_preds"][b].reshape(-1, n_cls).cpu(), p["box_preds"][b].reshape(-1, code).cpu(),
                                             p["dir_cls_preds"][b].reshape(-1, 2).cpu() if "dir_cls_preds" in p else None,
                                             anchors, cfg.test_cfg, bool(head.box_coder.vec_encode),
                                             float(head.direction_offset))
            want[b]["b"].append(bx); want[b]["s"].append(sc); want[b]["l"].append(lb + flag)
        flag += n_cls
    return [{k: torch.cat(v) for k, v in w.items()} for w in want]


CONFIGS = ["second", "pillars", "cbgs"]


def _oracle_class(module, name):
    return lambda: getattr(__import__("oracle." + module, fromlist=[name]), name)


ORACLES = {"second": _oracle_class("second_cpu", "SecondCPU"), "pillars": _oracle_class("pillars_cpu", "PillarsCPU"),
           "cbgs": _oracle_class("cbgs_cpu", "CbgsCPU")}


@pytest.mark.parametrize("name", CONFIGS)
def test_fp16_forward(name):
    """voxel indices and counts bit-exact with the oracle voxelizer's; detections = the oracle predict on the device's own
    fp16 head outputs; two runs and graph replay bit-identical; a cloud's detections independent of its batch mates; no
    cuDNN / cuBLAS kernel."""
    r = _forward(name)
    cfg, clouds = r["cfg"], r["clouds"]
    f = r["fp16"]
    assert f["flag"] == 0
    pipe, pts, offsets = r["pipes"]["fp16"]
    B = len(clouds)
    _v, coors, _n = ORACLES[name]()(cfg, r["sd"], [t.cpu().numpy() for t in pipe._anchors]).voxelize(clouds)
    counts = f["counts"].cpu().numpy()
    assert counts[B] == coors.shape[0] and np.array_equal(counts[:B], np.bincount(coors[:, 0], minlength=B))
    assert np.array_equal(f["coors"].cpu().numpy(), coors)
    got = pipe.unpack(f["packed"].cpu())
    want = _oracle_predict(pipe, cfg, f["heads"], B)
    total = 0
    for b in range(B):
        gb, gs, gl = got[b]["box3d_lidar"], got[b]["scores"], got[b]["label_preds"]
        assert gb.shape == want[b]["b"].shape, "sample %d: %d vs %d" % (b, gb.shape[0], want[b]["b"].shape[0])
        if gb.shape[0]:
            assert float((gb - want[b]["b"]).abs().max()) <= 1e-5 and float((gs - want[b]["s"]).abs().max()) <= 1e-6
            assert torch.equal(gl, want[b]["l"])
        total += gb.shape[0]
    assert total >= 5
    with torch.no_grad():
        again = pipe.pack(pipe.forward_device(pts, offsets)).clone()
    assert torch.equal(again, f["packed"])
    host = [torch.from_numpy(c).pin_memory() for c in clouds]
    graphed = pipe.infer_host(host, graphed=True).clone()
    assert torch.equal(graphed, pipe.infer_host(host).clone())
    assert torch.equal(graphed.cpu(), f["packed"].cpu())
    if B > 1:
        alone = pipe.infer_host([host[1]]).clone()
        assert torch.equal(alone[0], graphed[1])
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pipe.infer_host(host)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    vendor = [n for n in names if any(s in n.lower() for s in ("cudnn", "cublas", "gemm", "implicit_convolve", "winograd"))]
    assert not vendor, vendor
    assert any("f16_kernel" in n for n in names), names


# SECOND KITTI car suppresses at an NMS IoU of 0.01, so every cluster of overlapping candidates keeps exactly one box,
# and which one depends on the order of near-equal scores.  The fp16 heads move the logits by up to 0.07 (measured), which
# re-elects the winner of some clusters; the new winner overlaps the old one by less than the 0.5 this test asks for.
# Measured on an H100 80GB HBM3 at 700 W: 50 of 55 (0.909) -- below 0.95, recorded here rather than loosened.
AGREE = [pytest.param("second", marks=pytest.mark.xfail(strict=True, reason="NMS at IoU 0.01 re-elects cluster winners: "
                                                                           "0.909 measured")), "pillars", "cbgs"]


def _agreement(r):
    """(max abs head difference, confident FP16x3 detections, matched ones, unmatched ones as (box, label, fp16 boxes,
    fp16 labels, rotated BEV IoUs with them)) of one config's forward in both maths."""
    from det3d_b200 import _lib
    from det3d_b200.ops.nms.nms_ops import boxes_iou_bev
    thr = r["cfg"].test_cfg.score_threshold
    diff = max(float((ha[k] - hf[k]).abs().max()) for ha, hf in zip(r["fp16x3"]["heads"], r["fp16"]["heads"]) for k in ha)
    pipe = r["pipes"]["fp16"][0]
    da, df = pipe.unpack(r["fp16x3"]["packed"].cpu()), pipe.unpack(r["fp16"]["packed"].cpu())
    conf = hit = 0
    unmatched = []
    bev = lambda t: t[:, [0, 1, 3, 4, -1]].contiguous().cuda()
    for a, f in zip(da, df):
        keep = a["scores"] >= thr + 0.05
        ba, la = a["box3d_lidar"][keep], a["label_preds"][keep]
        conf += int(keep.sum())
        if ba.shape[0] == 0:
            continue
        fb, fl = f["box3d_lidar"], f["label_preds"]
        if fb.shape[0] == 0:
            unmatched += [(ba[i], la[i], fb, fl, torch.zeros(0)) for i in range(ba.shape[0])]
            continue
        iou = boxes_iou_bev(bev(ba), bev(fb), mode=_lib.IOU_BEV_XYWLR).cpu()      # the overlap rotated NMS thresholds
        ok = ((iou >= 0.5) & (la[:, None] == fl[None, :])).any(1)
        hit += int(ok.sum())
        unmatched += [(ba[i], la[i], fb, fl, iou[i]) for i in range(ba.shape[0]) if not bool(ok[i])]
    return diff, conf, hit, unmatched


@pytest.mark.parametrize("name", AGREE)
def test_fp16_agrees_with_fp16x3(name):
    """Max abs head-output difference, and the share of confident FP16x3 detections (score >= threshold + 0.05) that
    have a same-label fp16 detection with BEV IoU >= 0.5."""
    diff, conf, hit, _ = _agreement(_forward(name))
    frac = hit / max(conf, 1)
    print("%s: max |head fp16 - fp16x3| = %.3g; %d / %d confident FP16x3 detections matched (%.4f)"
          % (name, diff, hit, conf, frac))
    assert conf >= 5
    assert frac >= 0.95


def test_second_shortfall_is_nms_reelection():
    """SECOND's agreement shortfall comes from its NMS at IoU 0.01: every confident FP16x3 detection without an fp16 match
    at IoU >= 0.5 is covered in the fp16 result by a same-label detection overlapping it above the NMS threshold, i.e. one
    that suppressed it -- the cluster kept a different member."""
    r = _forward("second")
    nms_thr = r["cfg"].test_cfg.nms.nms_iou_threshold
    _diff, conf, hit, unmatched = _agreement(r)
    assert len(unmatched) == conf - hit > 0
    for box, label, fb, fl, iou in unmatched:
        same = fl == label
        best = float(iou[same].max()) if bool(same.any()) else 0.0
        print("unmatched FP16x3 box at (%.2f, %.2f): best same-label fp16 overlap %.3f" % (float(box[0]), float(box[1]), best))
        assert nms_thr < best < 0.5, "box at (%.2f, %.2f): best overlap %.3g" % (float(box[0]), float(box[1]), best)
