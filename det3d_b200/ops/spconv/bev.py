"""Fused RPN + heads executors on the BEV map: the reference's RPN (det3d/models/necks/rpn.py:82-159) and the
MultiGroupHead convs (det3d/models/bbox_heads/mg_head.py:198-230) with BN / ReLU folded into each conv's epilogue.

`FusedBevStack` (fp16x3 / fp16) takes every RPN the reference builds, on NHWC f16 planes through TMA tensor maps
(csrc/bevconv16_sm90.cu).  `FusedBevStackTF32` (tf32x3: the re-run after an f16-range overflow) takes the stride-1 /
1x1-deblock RPN shape (the SECOND configs) through the 3xTF32 sparse-conv kernel: in channels-last layout a dense
stride-1 conv IS the gather-GEMM that kernel performs, with a static rulebook (d3b_rulebook_dense2d: neighbour = row
+- 1, +- W, -1 at the border = zero padding); any other RPN stays on the module's regular torch forward under tf32x3.
In both, the heads of all tasks are ONE 1x1 conv whose fp32 output rows are already the NHWC-permuted layout
`Head.forward` produces with `.permute(0, 2, 3, 1)`.
"""
import ctypes as C

import torch
from torch import nn

from ... import _lib
from . import conv16, core
from .fused import _bn_fold


class _DenseLevel:
    """Stand-in for SparseLevel: n rows on the device, capacity = n."""

    def __init__(self, n_rows, device):
        self.cap = int(n_rows)
        self.n = torch.zeros(2, dtype=torch.int32, device=device)


class BevGrid:
    def __init__(self, batch, height, width, device):
        self.batch, self.h, self.w, self.device = int(batch), int(height), int(width), device
        self.n_rows = self.batch * self.h * self.w
        self.level = _DenseLevel(self.n_rows, device)
        self._rb = {}

    def rulebook(self, kh, kw, ph, pw):
        key = (kh, kw, ph, pw)
        rb = self._rb.get(key)
        if rb is None:
            k_vol = kh * kw
            nbr = torch.empty((k_vol, self.n_rows), dtype=torch.int32, device=self.device)
            tile_mask = torch.empty((self.n_rows + core.TILE_M - 1) // core.TILE_M, dtype=torch.int32, device=self.device)
            st = _lib.lib().d3b_rulebook_dense2d(
                self.batch, self.h, self.w, (C.c_int32 * 2)(kh, kw), (C.c_int32 * 2)(ph, pw), nbr.data_ptr(),
                tile_mask.data_ptr(), self.level.n.data_ptr(), _lib.current_stream())
            _lib.check(st, "d3b_rulebook_dense2d")
            rb = core.Rulebook(nbr, tile_mask, (1, kh, kw), self.level, self.level, "dense2d")
            self._rb[key] = rb
        return rb


def _conv2d_weight(conv):
    """nn.Conv2d weight [Cout, Cin, kh, kw] -> [kh*kw, Cin, Cout] (k = ky*kw + kx)."""
    w = conv.weight.detach().float()
    co, ci, kh, kw = w.shape
    return w.permute(2, 3, 1, 0).reshape(kh * kw, ci, co).contiguous()


def rpn_is_fusable(rpn):
    """stride-1 blocks and 1x1 stride-1 conv deblocks only (kitti_car...rpn1 shape)."""
    try:
        if any(int(s) != 1 for s in rpn._layer_strides):
            return False
        if len(rpn.blocks) != 1 or len(rpn.deblocks) != 1:
            return False
        for m in rpn.deblocks[0]:
            if isinstance(m, nn.ConvTranspose2d):
                return False
            if isinstance(m, nn.Conv2d) and (m.kernel_size != (1, 1) or m.stride != (1, 1)):
                return False
        chans = [m for blk in rpn.blocks for m in blk if isinstance(m, nn.Conv2d)]
        return all(core.tc_supported(m.in_channels, m.out_channels) and m.bias is None for m in chans)
    except AttributeError:
        return False


def _conv_bn_relu(seq, i):
    """(conv, bn | None, relu, next index) for the conv module at seq[i]."""
    conv = seq[i]
    j = i + 1
    bn = None
    if j < len(seq) and isinstance(seq[j], nn.modules.batchnorm._BatchNorm):
        bn = seq[j]
        j += 1
    relu = j < len(seq) and isinstance(seq[j], nn.ReLU)
    if relu:
        j += 1
    return conv, bn, relu, j


def _convs(seq):
    """(conv, bn | None, relu, extra padding) of each Conv2d in `seq`; a ZeroPad2d pads the conv after it."""
    out, i, pad = [], 0, 0
    while i < len(seq):
        if isinstance(seq[i], nn.ZeroPad2d):
            pad = int(seq[i].padding[0])
            i += 1
        elif isinstance(seq[i], nn.Conv2d):
            conv, bn, relu, i = _conv_bn_relu(seq, i)
            out.append((conv, bn, relu, pad))
            pad = 0
        else:
            i += 1
    return out


def _folded_bn(bn):
    """(scale, shift) of a BatchNorm in eval mode, or (None, None) without one."""
    if bn is None:
        return None, None
    if bn.training:
        raise RuntimeError("fused BEV stack is inference-only: call .eval()")
    return _bn_fold(bn)


class _BevStack:
    """What both stacks share: the parameter signature their device weights were made from, the heads of every task as
    one 1x1 conv, and the split of its output columns into one dict per task."""

    def __init__(self, rpn, head):
        self.rpn, self.head = rpn, head
        self._sig = None
        self._plan = None
        self._bufs = {}

    def _signature(self):
        ts = [p for p in self.rpn.parameters()] + [b for b in self.rpn.buffers()] + [p for p in self.head.tasks.parameters()]
        return tuple((t._version, t.data_ptr()) for t in ts)

    def _compiled(self, device):
        """The stack's device weights (its _compile), made again whenever a parameter has changed."""
        sig = self._signature()
        if self._plan is None or sig != self._sig:
            self._plan = self._compile(device)
            self._sig = sig
        return self._plan

    def _heads(self):
        """(weight [1, C_in, C_total], bias [C_total]) of every task's box / cls / dir convs as one 1x1 conv."""
        ws, bs, self._splits = [], [], []
        for task in self.head.tasks:
            parts = [("box_preds", task.conv_box), ("cls_preds", task.conv_cls)]
            if task.use_dir:
                parts.append(("dir_cls_preds", task.conv_dir))
            names = []
            for name, conv in parts:
                ws.append(_conv2d_weight(conv))
                bs.append(conv.bias.detach().float())
                names.append((name, conv.out_channels))
            self._splits.append(names)
        return torch.cat(ws, dim=2), torch.cat(bs)

    def _split(self, out):
        """Head output [B, H, W, >= C_total] -> list (per task) of dicts like Head.forward: box_preds [B,H,W,a*code],
        cls_preds [B,H,W,a*cls], dir_cls_preds [B,H,W,a*2] (views of `out`)."""
        preds, c0 = [], 0
        for names in self._splits:
            d = {}
            for name, c in names:
                d[name] = out[..., c0:c0 + c]
                c0 += c
            preds.append(d)
        return preds


class FusedBevStackTF32(_BevStack):
    """tf32x3: the stride-1 RPN and the heads through the 3xTF32 gather kernel over dense rulebooks; also an in-library
    cross-check of `FusedBevStack`."""
    _grid = None

    def _compile(self, device):
        to = lambda t: None if t is None else t.to(device)
        layers = []  # (ConvWeights, (kh, kw, ph, pw))
        for conv, bn, relu, pad in _convs(list(self.rpn.blocks[0]) + list(self.rpn.deblocks[0])):
            scale, shift = _folded_bn(bn)
            cw = core.ConvWeights(_conv2d_weight(conv).to(device), bias=to(conv.bias), scale=to(scale), shift=to(shift),
                                  relu=relu, algo=_lib.ALGO_TC)
            kh, kw = conv.kernel_size
            layers.append((cw, (kh, kw, int(conv.padding[0]) + pad, int(conv.padding[1]) + pad)))
        # the heads, padded with zero columns to a width the tensor-core kernel takes
        w, b = self._heads()
        total = w.shape[2]
        width = next(c for c in (16, 32, 64, 128) if c >= total)
        w = torch.cat([w, w.new_zeros((1, w.shape[1], width - total))], dim=2)
        b = torch.cat([b, b.new_zeros(width - total)])
        layers.append((core.ConvWeights(w.to(device), bias=b.to(device), relu=False, algo=_lib.ALGO_TC), (1, 1, 0, 0)))
        return layers

    def _buf(self, n, c, busy, device):
        pool = self._bufs.setdefault((n, c), [])
        for t in pool:
            if t is not busy:
                return t
        t = torch.empty((n, c), dtype=torch.float32, device=device)
        pool.append(t)
        return t

    def run(self, x, overflow=None):
        """x: [B, H, W, C] fp32 channels-last BEV features -> list (per task) of dicts like Head.forward (views of one
        fp32 output buffer).  `overflow` is unused: fp32 activations have no f16 range to leave."""
        device = x.device
        b, h, w, c = x.shape
        with _lib.on_device_of(x):
            if self._grid is None or (self._grid.batch, self._grid.h, self._grid.w) != (b, h, w):
                self._grid = BevGrid(b, h, w, device)
            layers = self._compiled(device)
            x = x.reshape(b * h * w, c)
            for cw, geom in layers:
                rb = self._grid.rulebook(*geom)
                out = self._buf(self._grid.n_rows, cw.c_out, x, device)
                core.sparse_conv(x, rb, cw, out)
                x = out
        return self._split(x.view(b, h, w, x.shape[1]))


def _layer16(conv, bn, relu, extra_pad, device):
    scale, shift = _folded_bn(bn)
    bias = None if conv.bias is None else conv.bias.detach().float()
    if isinstance(conv, nn.ConvTranspose2d):
        s = int(conv.stride[0])
        assert tuple(conv.kernel_size) == (s, s) and tuple(conv.stride) == (s, s) and tuple(conv.padding) == (0, 0)
        w = conv.weight.detach().float()                     # [C_in, C_out, s, s]
        wk = w.permute(2, 3, 0, 1).reshape(s * s, 1, w.shape[0], w.shape[1])
        return conv16.BevConv16(wk, 1, up=s, bias=bias, scale=scale, shift=shift, relu=relu, device=device)
    kh, kw = conv.kernel_size
    st = int(conv.stride[0])
    pad = int(conv.padding[0]) + extra_pad
    assert kh == kw and tuple(conv.stride) == (st, st) and int(conv.padding[1]) + extra_pad == pad
    return conv16.BevConv16(_conv2d_weight(conv), kh, stride=st, pad=pad, bias=bias, scale=scale, shift=shift, relu=relu,
                            device=device)


def rpn_is_fusable16(rpn):
    """Every RPN the reference builds (necks/rpn.py:82-143): 3x3 blocks with stride 1 or 2; deblocks that are 1x1 convs,
    ConvTranspose2d(kernel = stride <= 4), or Conv2d(kernel = stride = s, s in {2, 3, 4}, no padding / dilation /
    groups: an up-sampling stride of 1/s, as in nuScenes PointPillars); channel counts multiples of 16."""
    try:
        for blk in rpn.blocks:
            for m in blk:
                if isinstance(m, nn.Conv2d):
                    if m.kernel_size != (3, 3) or m.stride not in ((1, 1), (2, 2)) or m.in_channels % 16 or m.groups != 1:
                        return False
                elif not isinstance(m, (nn.ZeroPad2d, nn.ReLU, nn.modules.batchnorm._BatchNorm)):
                    return False
        for blk in rpn.deblocks:
            for m in blk:
                if isinstance(m, nn.ConvTranspose2d):
                    if m.kernel_size != m.stride or m.stride[0] != m.stride[1] or m.stride[0] > 4 or m.in_channels % 16:
                        return False
                elif isinstance(m, nn.Conv2d):
                    s = m.stride[0]
                    k_is_s = (m.kernel_size == m.stride == (s, s) and s in (2, 3, 4) and m.padding == (0, 0)
                              and m.dilation == (1, 1) and m.groups == 1)
                    if not (m.kernel_size == (1, 1) and m.stride == (1, 1) or k_is_s) or m.in_channels % 16:
                        return False
                elif not isinstance(m, (nn.ReLU, nn.modules.batchnorm._BatchNorm)):
                    return False
        ok_width = all(int(c) in (32, 64, 128) or int(c) % 128 == 0 for c in rpn._num_upsample_filters)
        return len(rpn.deblocks) >= 1 and ok_width       # a deblock fills whole channel blocks of its concat slice
    except AttributeError:
        return False


class FusedBevStack(_BevStack):
    """fp16x3 / fp16: RPN + all task heads on NHWC f16 planes (single-pass FP16 when the input carries one plane: every
    layer then runs on one plane, with the same packed weights): one launch per conv layer, except that each block's run
    of 3x3 stride-1 layers is one chained launch (conv16.bev_chain), and the deblocks write straight into their channel
    slice of the concat buffer."""

    def _compile(self, device):
        rpn = self.rpn
        blocks = [[_layer16(conv, bn, relu, pad, device) for conv, bn, relu, pad in _convs(list(blk))]
                  for blk in rpn.blocks]
        deblocks = []
        for blk in rpn.deblocks:
            conv, bn, relu, _ = _conv_bn_relu(list(blk), 0)
            deblocks.append(_layer16(conv, bn, relu, 0, device))
        w, b = self._heads()
        heads = conv16.BevConv16(w, 1, bias=b, relu=False, device=device)
        return dict(blocks=blocks, deblocks=deblocks, heads=heads, start=rpn._upsample_start_idx,
                    concat=sum(d.c_out_total for d in deblocks))

    def _planes(self, key, shape, device, n_planes):
        p = self._bufs.get(key)
        if p is None or p.shape != tuple(shape) or p.n_planes != n_planes:
            p = self._bufs[key] = conv16.Planes(shape, device, n_planes=n_planes)
        return p

    def _chain_workspace(self, b, h, w, n, device):
        # owned by the stack and keyed by shape, so a captured graph bakes in a pointer that stays valid
        key = ("chain", b, h, w, n)
        ws = self._bufs.get(key)
        if ws is None:
            ws = self._bufs[key] = conv16.chain_workspace(b, h, w, n, device)
        return ws

    def layers(self):
        """Flat (tag, layer) list in execution order (bench / accounting)."""
        out = []
        for i, blk in enumerate(self._plan["blocks"]):
            out += [("block%d.%d" % (i, j), l) for j, l in enumerate(blk)]
            if i - self._plan["start"] >= 0:
                out.append(("deblock%d" % (i - self._plan["start"]), self._plan["deblocks"][i - self._plan["start"]]))
        out.append(("heads", self._plan["heads"]))
        return out

    def run(self, x, overflow=None):
        """x: Planes [B, H, W, C] -> list (per task) of dicts like Head.forward (fp32 views of one output buffer, on the
        grid of the deblocks' outputs).  A value that leaves the f16 range ORs 1 into `overflow` (int32[1] device flag,
        or None)."""
        device = x.device
        with _lib.on_device_of(x.buf):
            pl = self._compiled(device)
            b, n_planes = x.shape[0], x.n_planes
            concat = None
            col = 0
            for i, blk in enumerate(pl["blocks"]):
                j = 0
                while j < len(blk):
                    # a run of consecutive 3x3 stride-1 layers is one chained launch (at most 8 layers each)
                    n = 1
                    while blk[j].chainable and n < 8 and j + n < len(blk) and blk[j + n].chainable:
                        n += 1
                    ho, wo = blk[j].out_hw(x.shape[1], x.shape[2])
                    outs = [self._planes(("blk", i, (j + k) % 2), (b, ho, wo, blk[j + k].c_out_padded), device, n_planes)
                            for k in range(n)]
                    if n == 1:
                        layer = blk[j]
                        layer(x, out=outs[0], overflow=overflow, tag="bev3x3" if layer.ksize == 3 else "bev1x1")
                    else:
                        conv16.bev_chain(blk[j:j + n], x, outs, self._chain_workspace(b, ho, wo, n, device),
                                         overflow=overflow)
                    x = outs[-1]
                    j += n
                k = i - pl["start"]
                if k >= 0:
                    de = pl["deblocks"][k]
                    ho, wo = de.out_hw(x.shape[1], x.shape[2])
                    if concat is None:
                        concat = self._planes(("concat",), (b, ho, wo, pl["concat"]), device, n_planes)
                    assert tuple(concat.shape[1:3]) == (ho, wo), "deblock outputs must share one grid"
                    de(x, out=concat, out_c0=col, overflow=overflow, tag="deblock")
                    col += de.c_out_total
            heads = pl["heads"]
            hc, wc = concat.shape[1], concat.shape[2]
            key = ("heads", b, hc, wc)
            out32 = self._bufs.get(key)
            if out32 is None:
                out32 = self._bufs[key] = torch.empty((b, hc, wc, heads.c_out_padded), dtype=torch.float32, device=device)
            heads(concat, out_f32=out32, tag="heads")
        return self._split(out32)
