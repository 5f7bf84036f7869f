"""Split-f16 ("FP16x3") convolution primitives over the det3d_b200 C ABI (include/det3d_b200.h section 3b).

An activation is carried as two f16 planes, hi = f16(x) and lo = f16(x - hi) (`Planes`); weights are split the same
way after an exact power-of-two scaling.  `sparse_conv16` is the output-stationary sparse convolution
(csrc/spconv16_sm90.cu: deterministic, fused bias/BN/residual/ReLU epilogue), `BevConv16` a dense NHWC 3x3 / 1x1 /
ConvTranspose layer through TMA tensor maps (csrc/bevconv16_sm90.cu).

Reference call sites: det3d/models/backbones/scn.py:106-157,323-355 (sparse levels),
det3d/models/necks/rpn.py:82-159 and det3d/models/bbox_heads/mg_head.py:198-230 (dense BEV).
"""
import ctypes as C
import math

import torch

from ... import _lib
from ..._lib import Bev16Params, Conv16Params



class Planes:
    """hi / lo f16 planes of a [rows, C] (or [B, H, W, C]) activation: x = hi + lo to 22 significant bits."""

    __slots__ = ("buf", "shape")

    def __init__(self, shape, device, zero=False):
        self.shape = tuple(int(s) for s in shape)
        alloc = torch.zeros if zero else torch.empty
        self.buf = alloc((2,) + self.shape, dtype=torch.float16, device=device)

    hi = property(lambda self: self.buf[0])
    lo = property(lambda self: self.buf[1])
    device = property(lambda self: self.buf.device)

    def view(self, *shape):
        p = Planes.__new__(Planes)
        p.buf = self.buf.view((2,) + tuple(shape))
        p.shape = tuple(p.buf.shape[1:])
        return p

    def zero_(self):
        self.buf.zero_()
        return self

    @staticmethod
    def from_f32(x, overflow=None, out=None):
        x = x.contiguous().float()
        p = out if out is not None else Planes(x.shape, x.device)
        with _lib.on_device_of(x):
            st = _lib.lib().d3b_split16(x.data_ptr(), x.numel(), p.hi.data_ptr(), p.lo.data_ptr(), _lib.ptr(overflow),
                                        _lib.current_stream())
        _lib.check(st, "d3b_split16")
        return p

    def to_f32(self, out=None):
        x = out if out is not None else torch.empty(self.shape, dtype=torch.float32, device=self.device)
        with _lib.on_device_of(self.buf):
            st = _lib.lib().d3b_merge16(self.hi.data_ptr(), self.lo.data_ptr(), x.numel(), x.data_ptr(),
                                        _lib.current_stream())
        _lib.check(st, "d3b_merge16")
        return x


def supported(c_in, c_out):
    """Shapes the wgmma FP16x3 sparse kernel takes (first layers with a handful of fp32 channels run on the
    fp32-input variant instead)."""
    return c_in % 8 == 0 and 8 <= c_in <= 512 and c_out in (16, 32, 64, 128)


def _weight_exponent(w):
    """Exact power-of-two scaling that puts max|w| near 2^13: the weights' lo parts stay f16-normal down to
    weights 2^-16 of the largest, and hi stays far below 65504."""
    m = float(w.abs().max())
    if not math.isfinite(m) or m <= 0.0:
        return 0
    return max(-40, min(40, 13 - int(math.floor(math.log2(m)))))


def pack_weight16(w, w_exp=None):
    """w [K, C_in, C_out] f32 (device) -> (packed f16 image, w_exp)."""
    w = w.detach().float().contiguous()
    k_vol, c_in, c_out = w.shape
    n = _lib.lib().d3b_conv16_packed_weight_halves(c_in, c_out, k_vol)
    if n == 0:
        raise _lib.D3BError("FP16x3 conv: unsupported C_in=%d C_out=%d k_vol=%d" % (c_in, c_out, k_vol))
    if w_exp is None:
        w_exp = _weight_exponent(w)
    packed = torch.empty(n, dtype=torch.float16, device=w.device)
    with _lib.on_device_of(w):
        st = _lib.lib().d3b_conv16_pack_weight(w.data_ptr(), c_in, c_out, k_vol, int(w_exp), packed.data_ptr(),
                                               _lib.current_stream())
    _lib.check(st, "d3b_conv16_pack_weight")
    return packed, int(w_exp)


class ConvWeights16:
    """Device-side parameters of one sparse conv (FP16x3) with its fused epilogue."""

    def __init__(self, weight, bias=None, scale=None, shift=None, relu=False):
        w = weight.detach().to(torch.float32)
        if w.dim() == 5:                                  # spconv v1 layout [kD, kH, kW, Cin, Cout]
            w = w.reshape(-1, w.shape[3], w.shape[4])
        self.k_vol, self.c_in, self.c_out = w.shape
        self.fp32_input = self.c_in <= 16 and self.c_in % 8 != 0     # the voxel-feature layer (4 / 5 channels)
        f = lambda t: None if t is None else t.detach().to(torch.float32).contiguous()
        self.bias, self.scale, self.shift = f(bias), f(scale), f(shift)
        self.relu = bool(relu)
        if self.fp32_input:
            self.weight = w.contiguous()
            self.packed, self.w_exp = None, 0
        else:
            if not supported(self.c_in, self.c_out):
                raise _lib.D3BError("FP16x3 sparse conv does not take C_in=%d C_out=%d" % (self.c_in, self.c_out))
            self.weight = None
            self.packed, self.w_exp = pack_weight16(w)
        self.acc_scale = math.ldexp(1.0, -self.w_exp)


def sparse_conv16(x, rb, cw, out, residual=None, out_f32=None, overflow=None, tag="sparse"):
    """out[:n_out] = epilogue(sum_k x[nbr[k]] @ W[k]).  x: Planes (or an fp32 [rows, C] tensor for the first layer);
    out: Planes [cap, C_out] (or None when only `out_f32` is wanted)."""
    p = Conv16Params()
    p.c_in, p.c_out, p.k_vol = cw.c_in, cw.c_out, cw.k_vol
    assert rb.k_vol == cw.k_vol, "kernel volume mismatch"
    if cw.fp32_input:
        assert torch.is_tensor(x) and x.dtype == torch.float32 and x.is_contiguous() and x.shape[1] == cw.c_in
        p.in_f32, p.weight = x.data_ptr(), cw.weight.data_ptr()
        dev_t = x
    else:
        assert isinstance(x, Planes) and x.shape[-1] == cw.c_in
        p.in_hi, p.in_lo, p.weight_packed = x.hi.data_ptr(), x.lo.data_ptr(), cw.packed.data_ptr()
        dev_t = x.buf
    p.acc_scale = cw.acc_scale
    p.bias, p.scale, p.shift = _lib.ptr(cw.bias), _lib.ptr(cw.scale), _lib.ptr(cw.shift)
    if residual is not None:
        assert residual.shape[-1] == cw.c_out
        p.residual_hi, p.residual_lo = residual.hi.data_ptr(), residual.lo.data_ptr()
    p.relu = 1 if cw.relu else 0
    if out is not None:
        assert out.shape[-1] == cw.c_out and out.shape[0] >= rb.out_level.cap
        p.out_hi, p.out_lo = out.hi.data_ptr(), out.lo.data_ptr()
    if out_f32 is not None:
        assert out_f32.dtype == torch.float32 and out_f32.is_contiguous() and out_f32.shape[1] == cw.c_out
        p.out_f32 = out_f32.data_ptr()
    p.overflow = _lib.ptr(overflow)
    with _lib.on_device_of(dev_t), _lib.timed(tag, c_in=cw.c_in, c_out=cw.c_out, k_vol=cw.k_vol, math="fp16x3"):
        st = _lib.lib().d3b_sparse_conv16(rb.nbr.data_ptr(), rb.tile_mask.data_ptr(), rb.out_level.n.data_ptr(),
                                          rb.out_level.cap, C.byref(p), _lib.current_stream())
    _lib.check(st, "d3b_sparse_conv16")
    return out


def sparse_to_bev16(x, level, out):
    """Sparse rows (Planes [cap, C] or fp32 [cap, C]) -> zero-filled NHWC planes `out` [B, H, W, C*D], channel = c*D+z."""
    c = x.shape[-1]
    hi = lo = f32 = None
    if isinstance(x, Planes):
        hi, lo, dev_t = x.hi.data_ptr(), x.lo.data_ptr(), x.buf
    else:
        assert x.dtype == torch.float32 and x.is_contiguous()
        f32, dev_t = x.data_ptr(), x
    sp = (C.c_int32 * 3)(*[int(v) for v in level.spatial])
    with _lib.on_device_of(dev_t):
        st = _lib.lib().d3b_sparse_to_bev16(hi, lo, f32, level.coors.data_ptr(), level.n.data_ptr(), level.cap, c, sp,
                                            level.batch, out.hi.data_ptr(), out.lo.data_ptr(), _lib.current_stream())
    _lib.check(st, "d3b_sparse_to_bev16")
    return out


class BevConv16:
    """One dense NHWC layer: Conv2d 3x3 (stride 1 / 2) or 1x1, or ConvTranspose2d(kernel = stride = up), with folded
    BatchNorm / bias / ReLU.  Output channels wider than 128 run as `cgroups` blocks of one launch; the result can land in
    a channel slice [out_c0, out_c0 + C_out) of a wider (concat) buffer."""

    def __init__(self, weight, ksize, stride=1, pad=0, up=1, bias=None, scale=None, shift=None, relu=False, device=None):
        # weight: [up*up, K*K, C_in, C_out] f32 (up*up = 1 for plain convs)
        w = weight.detach().float().to(device)
        if w.dim() == 3:
            w = w.unsqueeze(0)
        ugroups, k_vol, c_in, c_out = w.shape
        assert ugroups == up * up and k_vol == ksize * ksize
        self.ksize, self.stride, self.pad, self.up = int(ksize), int(stride), int(pad), int(up)
        self.c_in, self.c_out_total = c_in, c_out
        # split / pad the output channels into blocks the kernel takes
        if c_out > 128:
            self.c_blk = 128
        else:
            self.c_blk = next(c for c in (32, 64, 128) if c >= c_out)
        self.cgroups = (c_out + self.c_blk - 1) // self.c_blk
        c_pad = self.cgroups * self.c_blk
        self.c_out_padded = c_pad

        def padc(t, fill=0.0):
            if t is None:
                return None
            t = t.detach().float().to(device)
            return torch.cat([t, t.new_full((c_pad - c_out,), fill)]) if c_pad > c_out else t

        if c_pad > c_out:
            w = torch.cat([w, w.new_zeros((ugroups, k_vol, c_in, c_pad - c_out))], dim=3)
        w_exp = _weight_exponent(w)
        images = []
        for ug in range(ugroups):
            for cg in range(self.cgroups):
                blk = w[ug, :, :, cg * self.c_blk:(cg + 1) * self.c_blk].contiguous()
                images.append(pack_weight16(blk, w_exp)[0])
        self.packed = torch.cat(images)
        self.w_exp = w_exp
        self.acc_scale = math.ldexp(1.0, -w_exp)
        self.groups = ugroups * self.cgroups
        rep = lambda t: None if t is None else t.repeat(ugroups).contiguous()      # group-major: (ug, cg, c)
        self.bias, self.scale, self.shift = rep(padc(bias)), rep(padc(scale, 1.0)), rep(padc(shift))
        self.relu = bool(relu)

    def out_hw(self, h, w):
        ho = (h + 2 * self.pad - self.ksize) // self.stride + 1
        wo = (w + 2 * self.pad - self.ksize) // self.stride + 1
        return ho * self.up, wo * self.up

    def __call__(self, x, out=None, out_f32=None, out_c0=0, overflow=None, tag="bev"):
        """x: Planes [B, H, W, C_in]; out: Planes [B, H', W', C_total] and/or out_f32 [B, H', W', C_total] fp32."""
        b, h, w, c = x.shape
        assert c == self.c_in
        p = Bev16Params()
        p.batch, p.h_in, p.w_in, p.c_in = b, h, w, c
        p.c_out, p.ksize, p.stride, p.pad = self.c_blk, self.ksize, self.stride, self.pad
        p.groups, p.cgroups, p.up = self.groups, self.cgroups, self.up
        p.in_hi, p.in_lo, p.weight_packed = x.hi.data_ptr(), x.lo.data_ptr(), self.packed.data_ptr()
        p.acc_scale = self.acc_scale
        p.bias, p.scale, p.shift = _lib.ptr(self.bias), _lib.ptr(self.scale), _lib.ptr(self.shift)
        p.relu = 1 if self.relu else 0
        ho, wo = self.out_hw(h, w)
        ref = out if out is not None else out_f32
        shape = ref.shape
        assert tuple(shape[:3]) == (b, ho, wo), "output grid %s != %s" % (tuple(shape[:3]), (b, ho, wo))
        p.out_channels, p.out_c0 = int(shape[3]), int(out_c0)
        if out is not None:
            p.out_hi, p.out_lo = out.hi.data_ptr(), out.lo.data_ptr()
        if out_f32 is not None:
            assert out_f32.dtype == torch.float32 and out_f32.is_contiguous()
            if out is not None:
                assert tuple(out_f32.shape) == tuple(out.shape)
            p.out_f32 = out_f32.data_ptr()
        p.overflow = _lib.ptr(overflow)
        with _lib.on_device_of(x.buf), _lib.timed(tag, flops=self.flops(b, h, w), c_in=self.c_in, c_out=self.c_out_total,
                                                  ksize=self.ksize, stride=self.stride, up=self.up, math="fp16x3",
                                                  pixels_in=b * h * w, pixels_out=b * ho * wo,
                                                  tiles=b * (-(-(ho // self.up) // 16)) * (-(-(wo // self.up) // 16)) * self.groups):
            st = _lib.lib().d3b_bev_conv16(C.byref(p), _lib.current_stream())
        _lib.check(st, "d3b_bev_conv16")
        return out if out is not None else out_f32

    def flops(self, b, h, w):
        """fp32-equivalent flops of one call on a [b, h, w] input grid."""
        ho = (h + 2 * self.pad - self.ksize) // self.stride + 1
        wo = (w + 2 * self.pad - self.ksize) // self.stride + 1
        return 2 * b * ho * wo * self.ksize * self.ksize * self.c_in * self.c_out_total * self.up * self.up
