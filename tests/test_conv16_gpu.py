"""Split-f16 ("FP16x3") wgmma convolutions vs fp32 references (the plain-PyTorch fp32 restatement of the op):
csrc/spconv16_sm90.cu (sparse, output-stationary, deterministic) and csrc/bevconv16_sm90.cu (dense NHWC via TMA)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 1e-4      # north_star: 1e-4 abs on float features (inputs / weights scaled so features are O(1))


def _level(n, spatial, batch, seed):
    from det3d_b200.ops.spconv import core
    rng = np.random.default_rng(seed)
    d, h, w = spatial
    cells = rng.choice(batch * d * h * w, size=n, replace=False)
    b, rem = np.divmod(cells, d * h * w)
    z, rem = np.divmod(rem, h * w)
    y, x = np.divmod(rem, w)
    coors = torch.from_numpy(np.stack([b, z, y, x], 1).astype(np.int32)).cuda()
    return core.level_from_coors(coors, spatial, batch)


def _ref_conv(feat, nbr, w, n_out):
    """fp32 (float64-accumulated) gather-GEMM reference: out[o] = sum_k feat[nbr[k, o]] @ w[k]."""
    out = torch.zeros((n_out, w.shape[2]), dtype=torch.float64, device=feat.device)
    f64, w64 = feat.double(), w.double()
    for k in range(w.shape[0]):
        idx = nbr[k, :n_out].long()
        ok = idx >= 0
        out[ok] += f64[idx[ok]] @ w64[k]
    return out


@pytest.mark.parametrize("c_in,c_out,n,residual", [(16, 16, 3000, False), (16, 32, 777, False), (32, 32, 5000, True),
                                                   (64, 64, 20000, False), (64, 64, 129, True), (128, 128, 4000, True),
                                                   (64, 128, 1500, False), (4, 16, 6000, False), (5, 16, 300, False),
                                                   # C_in 16 / 32 pack 4 / 2 kernel offsets into one pipeline slot: a
                                                   # nearly empty grid leaves whole offset groups out of the tile masks
                                                   (16, 16, 140, True), (32, 64, 129, False), (32, 32, 260, False)])
def test_sparse_conv16_matches_fp32(c_in, c_out, n, residual):
    from det3d_b200.ops.spconv import conv16, core
    torch.manual_seed(c_in * 1000 + c_out)
    lvl = _level(n, (9, 40, 36), 2, n)
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, 3))
    feat = torch.randn((n, c_in), device="cuda")
    w = torch.randn((27, c_in, c_out), device="cuda") * (1.0 / np.sqrt(27 * c_in * 0.3))
    bias = torch.randn(c_out, device="cuda") * 0.1
    scale = torch.rand(c_out, device="cuda") + 0.5
    shift = torch.randn(c_out, device="cuda") * 0.1
    res = torch.randn((n, c_out), device="cuda") if residual else None
    cw = conv16.ConvWeights16(w, bias=bias, scale=scale, shift=shift, relu=True)
    ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
    x = feat if cw.fp32_input else conv16.Planes.from_f32(feat, ovf)
    if not cw.fp32_input:      # the planes carry the input to 22 bits
        assert float((x.to_f32() - feat).abs().max()) <= 2.0 ** -21 * float(feat.abs().max())
    out = conv16.Planes((n, c_out), "cuda")
    out_f32 = torch.empty((n, c_out), device="cuda")
    conv16.sparse_conv16(x, rb, cw, out, residual=None if res is None else conv16.Planes.from_f32(res), out_f32=out_f32,
                         overflow=ovf)
    want = (_ref_conv(feat, rb.nbr, w, n) + bias.double()) * scale.double() + shift.double()
    if res is not None:
        want = want + res.double()
    want = torch.relu(want).float()
    assert int(ovf.item()) == 0
    err = float((out_f32 - want).abs().max())
    assert err <= TOL, "fp32 output error %g" % err
    err_p = float((out.to_f32() - want).abs().max())
    assert err_p <= TOL, "plane output error %g" % err_p
    # deterministic: a second launch gives the same bits
    out2 = conv16.Planes((n, c_out), "cuda")
    conv16.sparse_conv16(x, rb, cw, out2, residual=None if res is None else conv16.Planes.from_f32(res))
    assert torch.equal(out.buf, out2.buf)


def test_sparse_conv16_strided_rulebook_and_overflow_flag():
    from det3d_b200.ops.spconv import conv16, core
    torch.manual_seed(3)
    n = 4000
    lvl = _level(n, (11, 50, 44), 1, 5)
    rb = core.build_conv_rulebook(core.alloc_conv_rulebook(lvl, 3, 2, 1))
    n_out = rb.out_level.count()
    feat = torch.randn((n, 32), device="cuda")
    w = torch.randn((27, 32, 64), device="cuda") * 0.05
    cw = conv16.ConvWeights16(w)
    ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
    out_f32 = torch.zeros((rb.out_level.cap, 64), device="cuda")
    conv16.sparse_conv16(conv16.Planes.from_f32(feat), rb, cw, None, out_f32=out_f32, overflow=ovf)
    want = _ref_conv(feat, rb.nbr, w, n_out).float()
    assert float((out_f32[:n_out] - want).abs().max()) <= TOL and int(ovf.item()) == 0
    # a result beyond the f16 range is reported, not saturated silently
    big = conv16.ConvWeights16(w * 1e5)
    out = conv16.Planes((rb.out_level.cap, 64), "cuda")
    conv16.sparse_conv16(conv16.Planes.from_f32(feat * 100), rb, big, out, overflow=ovf)
    assert int(ovf.item()) == 1


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("b,h,w,c_in,c_out,ks,stride", [
    (1, 200, 176, 128, 128, 3, 1),       # SECOND RPN layer
    (2, 37, 29, 64, 64, 3, 1),           # ragged grid, two samples
    (1, 200, 176, 128, 128, 1, 1),       # deblock 1x1
    (1, 50, 40, 128, 20, 1, 1),          # fused heads, padded to 32
    (1, 64, 48, 384, 276, 1, 1),         # wide head: C_in 384, C_out 276 -> 3 blocks of 128
    (1, 124, 108, 64, 128, 3, 2),        # RPN down-sampling block
    (2, 31, 45, 128, 256, 3, 2),         # stride 2, odd grid, C_out 256
    (1, 40, 40, 256, 256, 3, 1),
])
def test_bev_conv16_matches_conv2d(b, h, w, c_in, c_out, ks, stride):
    from det3d_b200.ops.spconv import conv16
    torch.manual_seed(h * 7 + c_out)
    x = torch.randn((b, c_in, h, w), device="cuda")
    wt = torch.randn((c_out, c_in, ks, ks), device="cuda") * (1.0 / np.sqrt(ks * ks * c_in * 0.3))
    scale = torch.rand(c_out, device="cuda") + 0.5
    shift = torch.randn(c_out, device="cuda") * 0.1
    pad = ks // 2
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        want = F.conv2d(x.double(), wt.double(), stride=stride, padding=pad)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    want = torch.relu(want * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)).float()
    layer = conv16.BevConv16(wt.permute(2, 3, 1, 0).reshape(ks * ks, c_in, c_out), ks, stride=stride, pad=pad,
                             scale=scale, shift=shift, relu=True, device="cuda")
    xin = conv16.Planes.from_f32(_nhwc(x))
    ho, wo = layer.out_hw(h, w)
    assert (ho, wo) == tuple(want.shape[2:])
    out = conv16.Planes((b, ho, wo, layer.c_out_padded), "cuda", zero=True)
    out_f32 = torch.zeros((b, ho, wo, layer.c_out_padded), device="cuda")
    ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
    layer(xin, out=out, out_f32=out_f32, overflow=ovf)
    got = out_f32[..., :c_out]
    err = float((got - _nhwc(want)).abs().max())
    assert err <= TOL, "fp32 output error %g" % err
    assert float((out.to_f32()[..., :c_out] - _nhwc(want)).abs().max()) <= TOL
    assert int(ovf.item()) == 0
    out2 = conv16.Planes((b, ho, wo, layer.c_out_padded), "cuda", zero=True)
    layer(xin, out=out2)
    assert torch.equal(out.buf, out2.buf)


@pytest.mark.parametrize("up,c_in,c_out,h,w", [(2, 128, 128, 62, 54), (4, 256, 128, 31, 27), (2, 256, 256, 64, 64)])
def test_bev_conv16_transpose_into_concat_slice(up, c_in, c_out, h, w):
    """ConvTranspose2d(k = s, stride = s) + BN + ReLU written into a channel slice of a wider concat buffer
    (necks/rpn.py:108-122,153-157)."""
    from det3d_b200.ops.spconv import conv16
    torch.manual_seed(up)
    x = torch.randn((1, c_in, h, w), device="cuda")
    wt = torch.randn((c_in, c_out, up, up), device="cuda") * (1.0 / np.sqrt(c_in * 0.3))
    scale = torch.rand(c_out, device="cuda") + 0.5
    shift = torch.randn(c_out, device="cuda") * 0.1
    want = F.conv_transpose2d(x.double(), wt.double(), stride=up)
    want = torch.relu(want * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)).float()
    # [up*up, 1, C_in, C_out], sub-pixel index = dy*up + dx
    wk = wt.permute(2, 3, 0, 1).reshape(up * up, 1, c_in, c_out)
    layer = conv16.BevConv16(wk, 1, up=up, scale=scale, shift=shift, relu=True, device="cuda")
    total = c_out + 64
    out = conv16.Planes((1, h * up, w * up, total), "cuda", zero=True)
    layer(conv16.Planes.from_f32(_nhwc(x)), out=out, out_c0=64)
    got = out.to_f32()
    assert float(got[..., :64].abs().max()) == 0.0                       # the neighbouring slice is untouched
    assert float((got[..., 64:] - _nhwc(want)).abs().max()) <= TOL


@pytest.mark.parametrize("b,h,w,c_in,c_out", [
    (1, 200, 176, 128, 128),      # SECOND RPN layer: 143 tiles, one per CTA
    (2, 37, 29, 64, 128),         # ragged grid, two samples, one 64-channel slice
    (1, 40, 40, 256, 256),        # two output blocks of 128, four input slices
    (5, 64, 48, 128, 128),        # more tiles than SMs: CTAs walk several tiles (buffer / stage parities carry over)
])
def test_bev_conv16_channel_stationary_variant(b, h, w, c_in, c_out):
    """d3b_set_bev_variant(1): the transposed schedule (C_out as the wgmma M dimension, the tile's pixels as N)
    against float64 conv2d and against the pixel-stationary schedule (same products, same order, same chains)."""
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16
    torch.manual_seed(h * 11 + c_out)
    x = torch.randn((b, c_in, h, w), device="cuda")
    wt = torch.randn((c_out, c_in, 3, 3), device="cuda") * (1.0 / np.sqrt(9 * c_in * 0.3))
    bias = torch.randn(c_out, device="cuda") * 0.1
    scale = torch.rand(c_out, device="cuda") + 0.5
    shift = torch.randn(c_out, device="cuda") * 0.1
    want = F.conv2d(x.double(), wt.double(), bias=bias.double(), padding=1)
    want = torch.relu(want * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)).float()
    layer = conv16.BevConv16(wt.permute(2, 3, 1, 0).reshape(9, c_in, c_out), 3, stride=1, pad=1, bias=bias, scale=scale,
                             shift=shift, relu=True, device="cuda")
    xin = conv16.Planes.from_f32(_nhwc(x))
    total = c_out + 32                      # written into a channel slice of a wider buffer
    outs = {}
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        for variant in (0, 1):
            _lib.lib().d3b_set_bev_variant(variant)
            out = conv16.Planes((b, h, w, total), "cuda", zero=True)
            out_f32 = torch.zeros((b, h, w, total), device="cuda")
            ovf = torch.zeros(1, dtype=torch.int32, device="cuda")
            layer(xin, out=out, out_f32=out_f32, out_c0=32, overflow=ovf)
            assert int(ovf.item()) == 0
            outs[variant] = (out, out_f32)
    finally:
        _lib.lib().d3b_set_bev_variant(prev)
    out, out_f32 = outs[1]
    assert float(out_f32[..., :32].abs().max()) == 0.0 and float(out.to_f32()[..., :32].abs().max()) == 0.0
    assert float((out_f32[..., 32:] - _nhwc(want)).abs().max()) <= TOL
    assert float((out.to_f32()[..., 32:] - _nhwc(want)).abs().max()) <= TOL
    assert torch.equal(out_f32, outs[0][1]) and torch.equal(out.buf, outs[0][0].buf)
