"""Chains of 3x3 stride-1 layers as one persistent launch (d3b_bev_conv16_chain, bev_conv16_pl_kernel with a work
list): a tile of layer k waits only for the <= 9 tiles of layer k - 1 it reads, so the layers overlap.

Each tile keeps the pipelined kernel's arithmetic, so a chain's planes must equal the layers run one by one on the
pixel-stationary kernel (variant 0) bit for bit: at SECOND's, SECOND three-class's, PointPillars block 3's and CBGS
block 2's shapes, on a ragged grid whose second layer overwrites the chain's input, with fewer tiles than SMs (every
tile of a later layer waits), and in single-pass FP16.  A captured chain replays on changing inputs (its counters reset
themselves), each RPN stack launches one kernel per chain, and the f16-range guard reports a value produced by a middle
layer.  The argument checks run without a GPU.
"""
import math

import pytest
import torch
from torch import nn

from test_bev_conv16_pipelined_gpu import PL, PS, _kernels, _with_variant

D3B_ERR_INVALID_ARG = 1


def _layers(n, c, seed, device="cuda", relu=True):
    from det3d_b200.ops.spconv import conv16
    g = torch.Generator(device=device).manual_seed(seed)
    out = []
    for _ in range(n):
        wt = torch.randn((9, c, c), device=device, generator=g) / math.sqrt(9 * c * 0.3)
        out.append(conv16.BevConv16(wt, 3, stride=1, pad=1, bias=torch.randn(c, device=device, generator=g) * 0.1,
                                    scale=torch.rand(c, device=device, generator=g) + 0.5,
                                    shift=torch.randn(c, device=device, generator=g) * 0.1, relu=relu, device=device))
    return out


def _run_chain(layers, x, outs, ws, flag):
    from det3d_b200.ops.spconv import conv16
    return conv16.bev_chain(layers, x, outs, ws, overflow=flag)


CASES = [
    # name, batch, h, w, channels, layers, planes, input overwritten by layer 1
    ("SECOND 1x200x176, six layers", 1, 200, 176, 128, 6, 2, False),
    ("SECOND three-class 2x200x176", 2, 200, 176, 128, 6, 2, False),
    ("PointPillars block 3 8x62x54x256", 8, 62, 54, 256, 5, 2, False),
    ("CBGS block 2 4x64x64x256", 4, 64, 64, 256, 5, 2, False),
    ("ragged 2x37x29, chain of 2 over its input", 2, 37, 29, 128, 2, 2, True),
    ("fewer tiles than SMs, four layers", 1, 32, 40, 128, 4, 2, False),
    ("single-pass FP16, SECOND", 1, 200, 176, 128, 6, 1, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,b,h,w,c,n,planes,over_input", CASES, ids=[c[0] for c in CASES])
def test_chain_bit_identical_to_layer_by_layer(name, b, h, w, c, n, planes, over_input):
    from det3d_b200.ops.spconv import conv16
    layers = _layers(n, c, seed=h + w + c + n)
    x32 = torch.randn((b, h, w, c), device="cuda", generator=torch.Generator(device="cuda").manual_seed(b * h))
    res = {}
    for variant in (0, 2):
        x = conv16.Planes.from_f32(x32, n_planes=planes)
        bufs = [x if over_input else conv16.Planes((b, h, w, c), "cuda", zero=True, n_planes=planes),
                conv16.Planes((b, h, w, c), "cuda", zero=True, n_planes=planes)]
        outs = [bufs[(k + 1) % 2] for k in range(n)]          # ping-pong, as the RPN stack does
        ws = conv16.chain_workspace(b, h, w, n, "cuda")
        flag = torch.zeros(1, dtype=torch.int32, device="cuda")
        ran = _with_variant(variant, lambda: _kernels(lambda: _run_chain(layers, x, outs, ws, flag)))
        pl, ps = (PL, PS) if planes == 2 else ("bev_conv16_pl_f16_kernel", "bev_conv16_f16_kernel")
        if variant == 2:
            assert ran and len(ran) == 1 and pl in ran[0], "%s: the chain ran %s" % (name, ran)
            assert int(ws.abs().sum()) == 0, "%s: the chain left its counters set" % name
        else:
            assert len(ran) == n and all(ps in k for k in ran), "%s: variant 0 ran %s" % (name, ran)
        assert int(flag.item()) == 0
        res[variant] = [o.buf.clone() for o in outs[-2:]]
    assert float(res[0][-1].float().abs().max()) > 0.01
    for a, r in zip(res[2], res[0]):
        assert torch.equal(a, r), "%s: the chain's planes differ from the layers run one by one" % name


@pytest.mark.gpu
def test_chain_graph_replays_on_changing_inputs():
    """One SECOND chain captured once and replayed 20 times on new inputs gives the eager chain's bits every time: the
    last CTA of each launch sets the workspace back to zero."""
    from det3d_b200.ops.spconv import conv16
    b, h, w, c, n = 1, 200, 176, 128, 6
    layers = _layers(n, c, seed=5)
    x = conv16.Planes((b, h, w, c), "cuda", zero=True)
    bufs = [conv16.Planes((b, h, w, c), "cuda"), conv16.Planes((b, h, w, c), "cuda")]
    outs = [bufs[k % 2] for k in range(n)]
    ws = conv16.chain_workspace(b, h, w, n, "cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(9)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _with_variant(2, lambda: _run_chain(layers, x, outs, ws, flag))      # warm-up (smem opt-in) off the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _with_variant(2, lambda: _run_chain(layers, x, outs, ws, flag))
    for i in range(20):
        conv16.Planes.from_f32(torch.randn((b, h, w, c), device="cuda", generator=g), out=x)
        graph.replay()
        got = outs[-1].buf.clone()
        _with_variant(2, lambda: _run_chain(layers, x, outs, ws, flag))
        assert torch.equal(got, outs[-1].buf), "replay %d differs from the eager chain" % i
        assert int(ws.abs().sum()) == 0
    assert int(flag.item()) == 0


@pytest.mark.gpu
def test_chain_flags_a_value_out_of_f16_range_in_a_middle_layer():
    """A bias of 2e5 on one channel of the third layer of four: the flag is raised."""
    from det3d_b200.ops.spconv import conv16
    b, h, w, c = 1, 40, 48, 128
    layers = _layers(4, c, seed=3, relu=False)
    bad = layers[2]
    bad.bias = bad.bias.clone()
    bad.bias[17] = 2e5
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    x = conv16.Planes.from_f32(torch.randn((b, h, w, c), device="cuda"))
    bufs = [conv16.Planes((b, h, w, c), "cuda"), conv16.Planes((b, h, w, c), "cuda")]
    outs = [bufs[k % 2] for k in range(4)]
    _with_variant(2, lambda: _run_chain(layers, x, outs, conv16.chain_workspace(b, h, w, 4, "cuda"), flag))
    assert int(flag.item()) == 1


class _Task(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv_box, self.conv_cls, self.use_dir = nn.Conv2d(c, 14, 1), nn.Conv2d(c, 2, 1), False


class _Head(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.tasks = nn.ModuleList([_Task(c)])


STACKS = [
    # config, neck arguments, input [B, H, W, C], chains
    ("second", dict(layer_nums=[5], ds_layer_strides=[1], ds_num_filters=[128], us_layer_strides=[1],
                    us_num_filters=[128], num_input_features=128), (1, 64, 48, 128), 1),
    ("pillars", dict(layer_nums=[3, 5, 5], ds_layer_strides=[2, 2, 2], ds_num_filters=[64, 128, 256],
                     us_layer_strides=[1, 2, 4], us_num_filters=[128, 128, 128], num_input_features=64),
     (2, 64, 64, 64), 2),
    ("cbgs", dict(layer_nums=[5, 5], ds_layer_strides=[1, 2], ds_num_filters=[128, 256], us_layer_strides=[1, 2],
                  us_num_filters=[256, 256], num_input_features=256), (1, 64, 64, 256), 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,neck,shape,chains", STACKS, ids=[s[0] for s in STACKS])
def test_stack_launches_one_kernel_per_chain(name, neck, shape, chains):
    """Each block's run of 3x3 stride-1 layers is one bev_conv16_pl_kernel launch, and the stack's result equals
    variant 0's, layer by layer on the pixel-stationary kernel, bit for bit."""
    from det3d_b200.models.necks.rpn import RPN
    from det3d_b200.ops.spconv import bev, conv16
    torch.manual_seed(0)
    rpn = RPN(**neck).eval().cuda()
    for m in rpn.modules():
        if isinstance(m, nn.modules.batchnorm._BatchNorm):
            m.running_mean.uniform_(-0.1, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    head = _Head(sum(neck["us_num_filters"])).cuda()
    stack = bev.FusedBevStack(rpn, head)
    x = conv16.Planes.from_f32(torch.randn(shape, device="cuda"))
    ran = _with_variant(2, lambda: _kernels(lambda: stack.run(x)))
    assert sum(PL in k for k in ran) == chains, "%s: %s" % (name, ran)
    res = {v: _with_variant(v, lambda: stack.run(x))[0]["box_preds"].clone() for v in (0, 2)}
    assert torch.equal(res[2], res[0]), "%s: the chained stack differs from variant 0" % name


# ---- argument checks (no GPU: every rejection happens before any CUDA call) ------------------------------------------
A, B, W, WS = 0x10000, 0x20000, 0x30000, 0x40000


def _chain_params(n, edits=None):
    from det3d_b200 import _lib
    arr = (_lib.Bev16Params * n)()
    for k in range(n):
        p = arr[k]
        p.batch, p.h_in, p.w_in, p.c_in, p.c_out = 1, 32, 40, 128, 128
        p.ksize, p.stride, p.pad, p.groups, p.cgroups, p.up = 3, 1, 1, 1, 1, 1
        p.out_channels, p.out_c0, p.acc_scale, p.weight_packed = 128, 0, 1.0, W
        src, dst = (A, B) if k % 2 == 0 else (B, A)
        p.in_hi, p.in_lo, p.out_hi, p.out_lo = src, src + 0x100, dst, dst + 0x100
    for (k, field), v in (edits or {}).items():
        setattr(arr[k], field, v)
    return arr


def _chain_rejected(arr, n, ws_bytes=None, what=""):
    from det3d_b200 import _lib
    lib = _lib.lib()
    if ws_bytes is None:
        ws_bytes = lib.d3b_bev_conv16_chain_workspace_bytes(1, 32, 40, max(1, min(n, 8)))
    st = lib.d3b_bev_conv16_chain(arr, n, WS, ws_bytes, None)
    msg = (lib.d3b_last_error() or b"").decode()
    assert st == D3B_ERR_INVALID_ARG, "%s: status %d (%s)" % (what, st, msg)
    assert "d3b_bev_conv16_chain" in msg and what in msg, msg


def test_chain_workspace_bytes():
    from det3d_b200 import _lib
    lib = _lib.lib()
    assert lib.d3b_bev_conv16_chain_workspace_bytes(1, 200, 176, 6) == 4 * (2 + 5 * 13 * 22)
    assert lib.d3b_bev_conv16_chain_workspace_bytes(1, 200, 176, 9) == 0
    assert lib.d3b_bev_conv16_chain_workspace_bytes(0, 200, 176, 2) == 0


@pytest.mark.parametrize("n", [0, 9])
def test_chain_rejects_layer_count(n):
    _chain_rejected(_chain_params(max(n, 1)), n, what="n_layers")


@pytest.mark.parametrize("field,value", [("stride", 2), ("c_out", 64), ("pad", 0), ("out_c0", 8), ("out_hi", None)])
def test_chain_rejects_a_layer_it_does_not_take(field, value):
    _chain_rejected(_chain_params(3, {(1, field): value}), 3, what="layer 1")


def test_chain_rejects_a_layer_not_reading_the_previous_output():
    _chain_rejected(_chain_params(3, {(2, "in_hi"): 0x50000}), 3, what="layer 2's input is not layer 1's output")


def test_chain_rejects_an_input_aliasing_its_own_output():
    _chain_rejected(_chain_params(1, {(0, "out_hi"): A, (0, "out_lo"): A + 0x100}), 1, what="aliases its own output")


def test_chain_rejects_a_short_workspace():
    from det3d_b200 import _lib
    need = _lib.lib().d3b_bev_conv16_chain_workspace_bytes(1, 32, 40, 4)
    _chain_rejected(_chain_params(4), 4, ws_bytes=need - 4, what="workspace")
