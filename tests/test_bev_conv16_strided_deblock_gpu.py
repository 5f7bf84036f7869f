"""Conv2d(kernel = stride = s, padding 0), s in {2, 3, 4}, on the pixel-stationary FP16x3 BEV kernel: the deblock
necks/rpn.py builds for an up-sampling stride 1/s (nuScenes PointPillars: Conv2d(64, 128, 2, stride=2)).

Checked against the error model of test_conv_error_model_gpu.py (per-element and RMS accumulation bounds, the
representation bound, and the same tolerances rejecting a float64 result without the A_lo.W_hi or the A_hi.W_lo
term).  Its float64 reference `dense_ref` follows the kernel's slot order (64-channel slice, then kx, then ky), which
this kernel case keeps."""
import pytest
import torch

from test_conv_error_model_gpu import (BOUNDARY, _epi_params, check_against_model, check_epilogue, dense_layer,
                                       operands, run_dense)

pytestmark = pytest.mark.gpu

CASES = [
    # b, h, w, c_in, c_out, s
    (1, 2, 2, 16, 32, 2),            # one output pixel (less than a tile)
    (2, 33, 47, 64, 64, 2),          # odd H and W: the last input row / column is not read
    (4, 64, 64, 128, 128, 2),
    (1, 37, 51, 256, 256, 2),        # C_out 256: two 128-channel groups in one launch
    (4, 256, 256, 64, 128, 2),       # the nuScenes PointPillars deblock at B = 4: 256 tiles, the persistent loop wraps
    (1, 3, 3, 64, 128, 3),
    (3, 49, 50, 16, 256, 3),
    (2, 100, 97, 128, 32, 3),
    (1, 20, 22, 256, 64, 3),
    (1, 4, 7, 128, 64, 4),
    (2, 67, 65, 256, 128, 4),
    (4, 33, 129, 16, 32, 4),
    (1, 130, 66, 64, 256, 4),
]


@pytest.mark.parametrize("b,h,w,c_in,c_out,s", CASES)
def test_kernel_stride_conv_error_model(b, h, w, c_in, c_out, s):
    from det3d_b200.ops.spconv import conv16
    seed = 17 * s + b * 1000 + h * 31 + c_in + c_out
    got, ref, layer, planes, x, wt = run_dense(b, h, w, c_in, c_out, s, s, 0, 1, seed)
    what = "k = s = %d %s" % (s, (b, h, w, c_in, c_out))
    assert tuple(got.shape) == (b, h // s, w // s, c_out)          # floors as torch does
    check_against_model(got, ref, layer.w_exp, what)
    # the float64 gather reference is torch's own strided convolution
    want = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2),
                                      wt[0].double().reshape(s, s, c_in, c_out).permute(3, 2, 0, 1),
                                      stride=s).permute(0, 2, 3, 1)
    assert want.shape == ref.y.shape
    assert float((want - ref.y).abs().max()) <= 1e-12 * float(ref.M.max())
    bias, scale, shift = _epi_params(c_out, seed)
    epi = dense_layer(wt, s, s, 0, 1, bias=bias, scale=scale, shift=shift, relu=True)
    out = conv16.Planes((b, h // s, w // s, epi.c_out_padded), "cuda", zero=True)
    out32 = torch.zeros((b, h // s, w // s, epi.c_out_padded), device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    epi(planes, out=out, out_f32=out32, overflow=flag)
    assert int(flag.item()) == 0
    check_epilogue(out32[..., :c_out], out.to_f32()[..., :c_out], ref, bias, scale, shift, True, what=what)


@pytest.mark.parametrize("s,c_out,c0,total", [(2, 128, 128, 384), (3, 64, 64, 192), (4, 256, 128, 512)])
def test_kernel_stride_conv_writes_only_its_channel_slice(s, c_out, c0, total):
    """Into channels [c0, c0 + C_out) of a wider concat buffer prefilled with a sentinel: the other channels keep it,
    the slice holds the bits of a launch into the layer's own buffer; out_f32 alone gives the same fp32 bits."""
    from det3d_b200.ops.spconv import conv16
    b, h, w = 2, 41, 38
    gen = torch.Generator(device="cuda").manual_seed(s * 100 + c_out)
    x, wt = operands((b, h, w, 64), (1, s * s, 64, c_out), "B", gen)
    bias, scale, shift = _epi_params(c_out, s)
    layer = dense_layer(wt, s, s, 0, 1, bias=bias, scale=scale, shift=shift, relu=True)
    planes = conv16.Planes.from_f32(x)
    ho, wo = h // s, w // s
    sentinel = -3.25
    wide = conv16.Planes((b, ho, wo, total), "cuda")
    wide.buf.fill_(sentinel)
    wide32 = torch.full((b, ho, wo, total), sentinel, device="cuda")
    layer(planes, out=wide, out_f32=wide32, out_c0=c0)
    outside = torch.ones(total, dtype=torch.bool, device="cuda")
    outside[c0:c0 + c_out] = False
    assert bool((wide.buf[..., outside] == sentinel).all()) and bool((wide32[..., outside] == sentinel).all())
    own = conv16.Planes((b, ho, wo, c_out), "cuda")
    own32 = torch.empty((b, ho, wo, c_out), device="cuda")
    layer(planes, out=own, out_f32=own32)
    assert torch.equal(wide.buf[..., c0:c0 + c_out], own.buf) and torch.equal(wide32[..., c0:c0 + c_out], own32)
    only32 = torch.full((b, ho, wo, total), sentinel, device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    layer(planes, out_f32=only32, out_c0=c0, overflow=flag)
    assert torch.equal(only32, wide32) and int(flag.item()) == 0


@pytest.mark.parametrize("s", [2, 3, 4])
def test_kernel_stride_conv_overflow_flag_boundary(s):
    """The epilogue flags exactly when |v| >= 65504 or v is inf / NaN (zero weights, the value through the bias); a
    launch that writes only out_f32 never raises it."""
    from det3d_b200.ops.spconv import conv16
    grid = conv16.Planes.from_f32(torch.randn((1, 9 * s, 11 * s, 64), device="cuda"))
    for v, want in BOUNDARY:
        bias = torch.zeros(128, device="cuda")
        bias[5] = v
        layer = dense_layer(torch.zeros((1, s * s, 64, 128), device="cuda"), s, s, 0, 1, bias=bias)
        flag = torch.zeros(1, dtype=torch.int32, device="cuda")
        layer(grid, out=conv16.Planes((1, 9, 11, 128), "cuda"), overflow=flag)
        assert int(flag.item()) == want, "k = s = %d epilogue, v = %r" % (s, v)
        flag.zero_()
        layer(grid, out_f32=torch.empty((1, 9, 11, 128), device="cuda"), overflow=flag)
        assert int(flag.item()) == 0, "k = s = %d out_f32-only launch raised the flag (v = %r)" % (s, v)


@pytest.mark.parametrize("s", [2, 3, 4])
def test_kernel_stride_conv_sample_independent_of_batch(s):
    """Sample 1 alone and inside a B = 3 batch: the same bits (37 x 29 is not a multiple of s or of the tile)."""
    from det3d_b200.ops.spconv import conv16
    gen = torch.Generator(device="cuda").manual_seed(40 + s)
    x, wt = operands((3, 37, 29, 64), (1, s * s, 64, 128), "B", gen)
    layer = dense_layer(wt, s, s, 0, 1, bias=torch.randn(128, device="cuda") * 0.1, relu=True)
    res = []
    for xin in (x, x[1:2].contiguous()):
        out = conv16.Planes((xin.shape[0], 37 // s, 29 // s, 128), "cuda")
        out32 = torch.empty((xin.shape[0], 37 // s, 29 // s, 128), device="cuda")
        layer(conv16.Planes.from_f32(xin), out=out, out_f32=out32)
        res.append((out.buf, out32))
    assert torch.equal(res[0][0][:, 1], res[1][0][:, 0]) and torch.equal(res[0][1][1], res[1][1][0])


@pytest.mark.parametrize("ks,stride,pad", [(2, 1, 0), (2, 2, 1), (3, 3, 1), (4, 4, 1), (5, 5, 0)])
def test_kernel_stride_conv_rejects_shapes_not_built(ks, stride, pad):
    """kernel 2 stride 1, kernel = stride with padding, and s = 5 are not built: an error, not a wrong result."""
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16
    gen = torch.Generator(device="cuda").manual_seed(ks * 10 + stride + pad)
    x, wt = operands((1, 20, 20, 64), (1, ks * ks, 64, 64), "C", gen)
    layer = dense_layer(wt, ks, stride, pad, 1)
    ho, wo = layer.out_hw(20, 20)
    out = torch.full((1, ho, wo, 64), 7.0, device="cuda")
    with pytest.raises(_lib.D3BError):
        layer(conv16.Planes.from_f32(x), out_f32=out)
    assert bool((out == 7.0).all())
