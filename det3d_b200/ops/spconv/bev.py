"""Channels-last dense BEV convolutions through the sparse-conv tensor-core kernel.

The reference's RPN (det3d/models/necks/rpn.py:124-159: ZeroPad+conv3x3, N x conv3x3, each
followed by BN2d + ReLU, then a 1x1 "deblock") and the MultiGroupHead 1x1 convs
(det3d/models/bbox_heads/mg_head.py:198-230) are dense stride-1 convolutions over the
[B, 200, 176] BEV grid.  In channels-last layout a dense conv IS the gather-GEMM the sparse
kernel already performs, with a static rulebook (d3b_rulebook_dense2d: neighbour = row +- 1,
+- W, -1 at the border = zero padding).  So the same tensor-core 3xTF32 kernel -- fp32-equivalent
accuracy, BN/ReLU folded into its epilogue -- replaces fp32 cuDNN here, and the head's three
1x1 convs become ONE conv whose [B*H*W, 32] output rows are already the NHWC-permuted layout
`Head.forward` produces with `.permute(0, 2, 3, 1)`.

Only the stride-1 / 1x1-deblock RPN shape (the SECOND configs) is taken; anything else
(strided blocks, ConvTranspose deblocks) stays on the module's regular torch forward.
"""
import ctypes as C

import torch
from torch import nn

from ... import _lib
from . import core
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


class FusedBevStackTF32:
    """Round-1 path (3xTF32 through the sparse gather kernel, stride-1 RPN only); kept as the fallback when a
    feature leaves the f16 range and as an in-library cross-check of `FusedBevStack`."""

    def __init__(self, rpn, head):
        self.rpn, self.head = rpn, head
        self._grid = None
        self._layers = None
        self._sig = None
        self._bufs = {}

    def _signature(self):
        ts = [p for p in self.rpn.parameters()] + [b for b in self.rpn.buffers()] + [p for p in self.head.tasks.parameters()]
        return tuple((t._version, t.data_ptr()) for t in ts)

    def _compile(self, device):
        layers = []  # (ConvWeights, (kh, kw, ph, pw))
        seq = list(self.rpn.blocks[0]) + list(self.rpn.deblocks[0])
        i = 0
        pending_pad = 0
        while i < len(seq):
            m = seq[i]
            if isinstance(m, nn.ZeroPad2d):
                pending_pad = int(m.padding[0])
                i += 1
                continue
            if isinstance(m, nn.Conv2d):
                bn = seq[i + 1] if i + 1 < len(seq) and isinstance(seq[i + 1], nn.modules.batchnorm._BatchNorm) else None
                relu = any(isinstance(x, nn.ReLU) for x in seq[i + 1:i + 3])
                if bn is not None and bn.training:
                    raise RuntimeError("fused BEV stack is inference-only: call .eval()")
                scale = shift = None
                if bn is not None:
                    scale, shift = _bn_fold(bn)
                    scale, shift = scale.to(device), shift.to(device)
                kh, kw = m.kernel_size
                ph, pw = int(m.padding[0]) + pending_pad, int(m.padding[1]) + pending_pad
                pending_pad = 0
                cw = core.ConvWeights(_conv2d_weight(m).to(device), bias=None if m.bias is None else m.bias.to(device),
                                      scale=scale, shift=shift, relu=relu, algo=_lib.ALGO_TC)
                layers.append((cw, (kh, kw, ph, pw)))
                i += 1 + (1 if bn is not None else 0) + (1 if relu else 0)
                continue
            i += 1
        # heads: one conv over the concatenated output channels, padded to a supported width
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
        w = torch.cat(ws, dim=2)
        b = torch.cat(bs)
        total = w.shape[2]
        width = next(c for c in (16, 32, 64, 128) if c >= total)
        w = torch.cat([w, w.new_zeros((1, w.shape[1], width - total))], dim=2)
        b = torch.cat([b, b.new_zeros(width - total)])
        layers.append((core.ConvWeights(w.to(device), bias=b.to(device), relu=False, algo=_lib.ALGO_TC), (1, 1, 0, 0)))
        self._layers = layers

    def _buf(self, n, c, busy, device):
        pool = self._bufs.setdefault((n, c), [])
        for t in pool:
            if t is not busy:
                return t
        t = torch.empty((n, c), dtype=torch.float32, device=device)
        pool.append(t)
        return t

    def run(self, rows, batch, height, width):
        with _lib.on_device_of(rows):
            return self._run(rows, batch, height, width)

    def _run(self, rows, batch, height, width):
        """rows [B*H*W, C] channels-last BEV features -> list (per task) of dicts like Head.forward:
        box_preds [B,H,W,a*code], cls_preds [B,H,W,a*cls], dir_cls_preds [B,H,W,a*2]."""
        device = rows.device
        if self._grid is None or (self._grid.batch, self._grid.h, self._grid.w) != (batch, height, width):
            self._grid = BevGrid(batch, height, width, device)
        sig = self._signature()
        if self._layers is None or sig != self._sig:
            self._compile(device)
            self._sig = sig
        x = rows
        for cw, geom in self._layers:
            rb = self._grid.rulebook(*geom)
            out = self._buf(self._grid.n_rows, cw.c_out, x, device)
            core.sparse_conv(x, rb, cw, out)
            x = out
        preds, col = [], 0
        flat = x.view(batch, height, width, x.shape[1])
        for names in self._splits:
            d = {}
            for name, c in names:
                d[name] = flat[..., col:col + c]
                col += c
            preds.append(d)
        return preds


# ======================================================================================================
# FP16x3 path: the whole RPN (any block strides / ConvTranspose deblocks / concat) + all task heads on
# NHWC f16 planes through TMA tensor maps (csrc/bevconv16_sm90.cu).
# ======================================================================================================
from . import conv16  # noqa: E402


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


def _layer16(conv, bn, relu, extra_pad, device):
    if bn is not None and bn.training:
        raise RuntimeError("fused BEV stack is inference-only: call .eval()")
    scale = shift = None
    if bn is not None:
        scale, shift = _bn_fold(bn)
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
    """Every RPN the reference builds (necks/rpn.py:82-143): 3x3 blocks with stride 1 or 2, deblocks that are 1x1 convs
    or ConvTranspose2d(kernel = stride); channel counts multiples of 16."""
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
                    if m.kernel_size != (1, 1) or m.stride != (1, 1) or m.in_channels % 16:
                        return False
                elif not isinstance(m, (nn.ReLU, nn.modules.batchnorm._BatchNorm)):
                    return False
        ok_width = all(int(c) in (32, 64, 128) or int(c) % 128 == 0 for c in rpn._num_upsample_filters)
        return len(rpn.deblocks) >= 1 and ok_width       # a deblock fills whole channel blocks of its concat slice
    except AttributeError:
        return False


class FusedBevStack:
    """RPN + all task heads on NHWC f16 planes (FP16x3): one launch per conv layer, the deblocks write straight into
    their channel slice of the concat buffer, and the heads of all tasks are ONE 1x1 conv whose fp32 output rows are
    already the NHWC-permuted layout `Head.forward` produces (mg_head.py:214-230)."""

    def __init__(self, rpn, head):
        self.rpn, self.head = rpn, head
        self._sig = None
        self._plan = None
        self._bufs = {}

    def _signature(self):
        ts = [p for p in self.rpn.parameters()] + [b for b in self.rpn.buffers()] + [p for p in self.head.tasks.parameters()]
        return tuple((t._version, t.data_ptr()) for t in ts)

    def _compile(self, device):
        rpn = self.rpn
        start = rpn._upsample_start_idx
        blocks = []
        for blk in rpn.blocks:
            seq, layers, i, pad = list(blk), [], 0, 0
            while i < len(seq):
                m = seq[i]
                if isinstance(m, nn.ZeroPad2d):
                    pad = int(m.padding[0])
                    i += 1
                elif isinstance(m, nn.Conv2d):
                    conv, bn, relu, i = _conv_bn_relu(seq, i)
                    layers.append(_layer16(conv, bn, relu, pad, device))
                    pad = 0
                else:
                    i += 1
            blocks.append(layers)
        deblocks = []
        for blk in rpn.deblocks:
            seq = list(blk)
            conv, bn, relu, _ = _conv_bn_relu(seq, 0)
            deblocks.append(_layer16(conv, bn, relu, 0, device))
        # heads: one 1x1 conv over the concatenated output channels of every task
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
        heads = conv16.BevConv16(torch.cat(ws, dim=2), 1, bias=torch.cat(bs), relu=False, device=device)
        self._plan = dict(blocks=blocks, deblocks=deblocks, heads=heads, start=start,
                          concat=sum(d.c_out_total for d in deblocks))

    def _planes(self, key, shape, device):
        p = self._bufs.get(key)
        if p is None or p.shape != tuple(shape):
            p = self._bufs[key] = conv16.Planes(shape, device)
        return p

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
        """x: Planes [B, H, W, C] -> list (per task) of dicts like Head.forward: box_preds [B,H',W',a*code],
        cls_preds [B,H',W',a*cls], dir_cls_preds [B,H',W',a*2] (fp32 views of one output buffer)."""
        device = x.device
        with _lib.on_device_of(x.buf):
            sig = self._signature()
            if self._plan is None or sig != self._sig:
                self._compile(device)
                self._sig = sig
            pl = self._plan
            b = x.shape[0]
            concat = None
            col = 0
            for i, blk in enumerate(pl["blocks"]):
                for j, layer in enumerate(blk):
                    ho, wo = layer.out_hw(x.shape[1], x.shape[2])
                    out = self._planes(("blk", i, j % 2), (b, ho, wo, layer.c_out_padded), device)
                    layer(x, out=out, overflow=overflow, tag="bev3x3" if layer.ksize == 3 else "bev1x1")
                    x = out
                k = i - pl["start"]
                if k >= 0:
                    de = pl["deblocks"][k]
                    ho, wo = de.out_hw(x.shape[1], x.shape[2])
                    if concat is None:
                        concat = self._planes(("concat",), (b, ho, wo, pl["concat"]), device)
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
        preds, c0 = [], 0
        for names in self._splits:
            d = {}
            for name, c in names:
                d[name] = out32[..., c0:c0 + c]
                c0 += c
            preds.append(d)
        return preds
