"""The pipelined 3x3 stride-1 dense kernel (bev_conv16_pl_kernel), which the automatic variant runs for every layer with
128-channel output blocks and C_in a multiple of 64.

It is the pixel-stationary kernel's arithmetic in another schedule (16 x 8 pixel tiles, one m64n128k16 chain per slot,
two partials in flight), so its planes and fp32 rows must equal variant 0's bit for bit: at SECOND's RPN shape, on a
ragged grid of two samples, with an odd tile count, with two output blocks and four input slices, with more tiles than
SMs (ring parities carried across tiles), with one 64-channel input slice, and into a channel slice with the fp32
output only.  torch.profiler shows which kernel ran.  The f16-range guard of its epilogue is driven across the boundary
as test_f16_guard_gpu does for the other dense schedules.
"""
import math

import pytest
import torch

from test_conv_error_model_gpu import dense_layer
from test_f16_guard_gpu import _cases, _epi, _flag, check_written

pytestmark = pytest.mark.gpu

PL = "bev_conv16_pl_kernel"
PS = "bev_conv16_kernel"                 # the pixel-stationary template (not a substring of PL)


def _kernels(fn):
    """Names of the CUDA kernels fn launches."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "bev_conv16" in e.name]


def _with_variant(variant, fn):
    from det3d_b200 import _lib
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        _lib.lib().d3b_set_bev_variant(variant)
        return fn()
    finally:
        _lib.lib().d3b_set_bev_variant(prev)


CASES = [
    # name, b, h, w, c_in, c_out, out_c0, extra channels after the slice, planes written
    ("SECOND RPN 200x176", 1, 200, 176, 128, 128, 0, 0, True),
    ("ragged, two samples", 2, 37, 29, 128, 128, 0, 0, True),
    ("odd tile count", 1, 37, 21, 128, 128, 0, 0, True),
    ("two output blocks, four input slices", 1, 40, 40, 256, 256, 0, 0, True),
    ("several tiles per CTA", 5, 64, 48, 128, 128, 0, 0, True),
    ("CBGS RPN 128x128, B = 4", 4, 128, 128, 128, 128, 0, 0, True),
    ("C_in 64", 2, 37, 29, 64, 128, 0, 0, True),
    ("fp32 rows only, into a channel slice", 1, 40, 40, 128, 256, 64, 32, False),
]


@pytest.mark.parametrize("name,b,h,w,c_in,c_out,c0,extra,planes", CASES, ids=[c[0] for c in CASES])
def test_pipelined_bit_identical_to_pixel_stationary(name, b, h, w, c_in, c_out, c0, extra, planes):
    from det3d_b200.ops.spconv import conv16
    g = torch.Generator(device="cuda").manual_seed(h * 7 + w + c_in)
    x = torch.randn((b, h, w, c_in), device="cuda", generator=g)
    wt = torch.randn((9, c_in, c_out), device="cuda", generator=g) / math.sqrt(9 * c_in * 0.3)
    bias = torch.randn(c_out, device="cuda", generator=g) * 0.1
    scale = torch.rand(c_out, device="cuda", generator=g) + 0.5
    shift = torch.randn(c_out, device="cuda", generator=g) * 0.1
    layer = conv16.BevConv16(wt, 3, stride=1, pad=1, bias=bias, scale=scale, shift=shift, relu=True, device="cuda")
    xin = conv16.Planes.from_f32(x)
    total = c0 + c_out + extra
    outs = {}
    for variant in (0, 2):
        out = conv16.Planes((b, h, w, total), "cuda", zero=True) if planes else None
        out32 = torch.zeros((b, h, w, total), device="cuda")
        ovf = _flag()
        ran = _with_variant(variant, lambda: _kernels(lambda: layer(xin, out=out, out_f32=out32, out_c0=c0, overflow=ovf)))
        want = PL if variant == 2 else PS
        assert ran and all(want in n for n in ran), "%s: variant %d ran %s" % (name, variant, ran)
        assert int(ovf.item()) == 0
        outs[variant] = (out, out32)
    (p0, f0), (p2, f2) = outs[0], outs[2]
    assert float(f0[..., c0:c0 + c_out].abs().max()) > 0.1
    assert torch.equal(f2, f0), "%s: fp32 rows differ from the pixel-stationary kernel's" % name
    if planes:
        assert torch.equal(p2.buf, p0.buf), "%s: planes differ from the pixel-stationary kernel's" % name


GUARD = [
    # name, c_in, c_out, out_c0, extra channels after the slice, value channel
    ("3x3 s1 128", 128, 128, 0, 0, 90),
    ("cgroups 2 into a slice", 64, 256, 64, 64, 128 + 9),
]


@pytest.mark.parametrize("name,c_in,c_out,c0,extra,c", GUARD, ids=[d[0] for d in GUARD])
def test_pipelined_fp16x3_guard(name, c_in, c_out, c0, extra, c):
    """The value on one zero-weight channel through the bias: flag raised exactly when |v| is not below 65504 or v is
    NaN, hi / lo the split of the value written, +0 under ReLU for negative values (test_f16_guard_gpu's cases)."""
    from det3d_b200.ops.spconv import conv16
    b, h, w = 2, 19, 23
    g = torch.Generator(device="cuda").manual_seed(300 + c_out)
    x = conv16.Planes.from_f32(torch.randn((b, h, w, c_in), device="cuda", generator=g))
    wt = torch.randn((1, 9, c_in, c_out), device="cuda", generator=g) / math.sqrt(9 * c_in)
    wt[..., c] = 0.0
    total = c0 + c_out + extra
    checked_kernel = False

    def run():
        nonlocal checked_kernel
        for relu in (False, True):
            for v, e, want in _cases(relu):
                bias, scale, shift = _epi(c_out, c, c_out, v)
                layer = dense_layer(wt, 3, 1, 1, 1, bias=bias, scale=scale, shift=shift, relu=relu)
                out = conv16.Planes((b, h, w, total), "cuda", zero=True)
                out32 = torch.zeros((b, h, w, total), device="cuda")
                flag = _flag()
                call = lambda: layer(x, out=out, out_f32=out32, out_c0=c0, overflow=flag)
                if not checked_kernel:
                    ran = _kernels(call)
                    assert ran and all(PL in n for n in ran), "%s ran %s" % (name, ran)
                    checked_kernel = True
                else:
                    call()
                what = "pipelined %s relu %d v = %r" % (name, relu, v)
                k = c0 + c
                check_written(what, e, int(flag.item()), want, out.hi[..., k], out.lo[..., k], out32[..., k])
                live = torch.zeros(total, dtype=torch.bool, device="cuda")
                live[c0:c0 + c_out] = True
                live[k] = False
                assert bool(torch.isfinite(out32[..., live]).all()) and float(out32[..., live].abs().max()) < 100.0
                assert float(out32[..., :c0].abs().max() if c0 else 0.0) == 0.0, "%s: wrote below its slice" % what
                assert float(out32[..., c0 + c_out:].abs().max() if extra else 0.0) == 0.0, "%s: wrote past its slice" % what

    _with_variant(2, run)
