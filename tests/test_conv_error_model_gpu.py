"""FP16x3 convolutions against their own error model (csrc/spconv16_sm90.cu, csrc/bevconv16_sm90.cu), and the tf32x3
fallback kernels at the magnitudes where they actually run.

Every check compares a kernel with float64 quantities computed on the GPU with plain torch, per output:

* ``y``  = sum a*w, the exact result of the fp32 operands;
* ``yh`` = sum (a_hi*w_hi + a_hi*w_lo + a_lo*w_hi), the split-exact result built from the operands the kernel sees
  (activation planes as stored, weights w*2^w_exp split with round-to-nearest-even like __float2half_rn, scaled back).
  A product of two f16 values is exact in float64, so ``yh`` is what an exactly rounded accumulator would give;
* ``M``  = sum |a|*|w|, the magnitude every bound below is relative to (scale-free: the same constant holds for
  activations of 2^-12 and of 2^12).

Units: u = 2^-24 (fp32 round-to-nearest), eps = 2^-26 (``kTruncLossPerMma``).

Accumulation error (``c_acc``, per element).  One slot = one kernel offset (or a packed group of offsets) x one 64-channel
slice: n = 3 * n_ks <= 12 MMAs chained into a fresh register partial P_s, added into the running fp32 sum S with
round-to-nearest; the epilogue scales the sum by 1 + c, c = the layer's mean n eps, as fmaf(v, c, v) (one more rounding).  Hardware model of one wgmma k16 step: the 16
products are exact, they are aligned with the running value and summed, and the result is truncated to fp32; the
alignment and the final truncation each lose less than one ulp of the largest magnitude involved, which is at most the
slot's magnitude M_s (sum of |a_hi w_hi| + |a_hi w_lo| + |a_lo w_hi| over the slot, <= (1 + 2^-9) M_s(exact)).  So
    |P_s - yh_s| <= 2 n 2^-23 M_s,     |RN add of slot s| <= u |S_s|,     |c yh| <= n eps M,   |RN of fmaf| <= u |yh|
with S_s the running sum after slot s.  Summed over the slots (sum M_s = M):
    |got - yh| <= c_acc M + u (1 + 2^-20) (sum_s |S_s| + |yh|),       c_acc = (2 n 2^-23 + n eps) (1 + 2^-9),
and the kernel's epilogue scale 2^-w_exp is exact.  sum_s |S_s| is computed from the float64 slot partials in the
kernel's slot order.  For n = 12, c_acc ~ 208 eps ~ 3.1e-6.  This is a worst-case bound, not a fit.  (A full slot's
correction is not applied as one factor 1 + 12 eps: that is not an fp32 number and would round to 1 + 16 eps.)

Aggregate (RMS over all outputs of (got - yh) / M).  If the roundings are independent, each bounded as above, and their
mean is removed by the correction up to a residual rho per partial, the expected square of the error of one output is at
most  sum_s [n (2 2^-23 M_s)^2 + (u S_s)^2] + (u yh)^2  plus the bias  rho sum_s |P_s|  (Minkowski: the RMS of a sum is at most
the sum of the RMSs).  rho = 12 eps is the bias test's outer bound (a correction that is never worse than none).

Representation error (what ``yh`` removes).  With hi = rn16(x), r = x - hi, lo = rn16(r): |x - hi - lo| < 2^-23 2^e(x)
for normal lo (a tie, the only case with |r| = 2^-11 2^e(x), is exact) and <= 2^-25 when lo is f16-subnormal.  Then
y - yh = a_lo w_lo + (a_hi + a_lo) e_w + e_a w gives
    |yh - y| <= 2^-21 M + 2^-25 sum|w| + 2^-25 2^-w_exp sum|a|
the last two terms being the f16-subnormal floors of the activation and of the (scaled) weight lo planes: activations
are not rescaled, so below about |x| = 2^-3 they carry fewer than 22 significant bits (DESIGN 3.0).

Mutation checks.  At every case the same tolerances are applied on the host to the float64 outputs of plausible wrong
kernels -- yh without the A_lo.W_hi term, yh without the A_hi.W_lo term -- and must reject them; the bias bound must reject
got * (1 +- 12 eps), a missing or doubled correction.  A tolerance that cannot tell those apart from the kernel fails the
test.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
EPS = 2.0 ** -26
F16_MAX = 65504.0


def c_acc(n_ks):
    n = 3 * n_ks
    return (2 * n * 2.0 ** -23 + n * EPS) * (1 + 2.0 ** -9)


def split16(x):
    """fp32 tensor -> (hi, lo) f16 exactly as split_f16 does it."""
    x = x.float()
    hi = x.half()
    return hi, (x - hi.float()).half()


def weight_planes(w, w_exp):
    """(w_hi, w_lo) in float64 as the kernel multiplies them, scaled back by 2^-w_exp."""
    hi, lo = split16(w.float() * math.ldexp(1.0, w_exp))      # exact power-of-two scaling in fp32
    s = math.ldexp(1.0, -w_exp)
    return hi.double() * s, lo.double() * s


class Ref:
    """float64 pieces of one convolution, accumulated slot by slot in the kernel's slot order."""

    def __init__(self, shape, device):
        z = lambda: torch.zeros(shape, dtype=torch.float64, device=device)
        self.y, self.hh, self.hl, self.lh, self.M = z(), z(), z(), z(), z()
        self.sw, self.sa = z(), z()                # sum |w|, sum |a| over the present terms
        self.run_abs, self.var, self.pabs = z(), z(), z()     # sum_s |S_s|, sum_s variance bounds, sum_s |P_s|
        self.n_ks = 1

    def slot(self, a, a_hi, a_lo, w, w_hi, w_lo, n_ks):
        """a*: [..., K] operands of one slot (zeros where absent), w*: [K, C_out]."""
        self.n_ks = max(self.n_ks, n_ks)
        hh, hl, lh = a_hi @ w_hi, a_hi @ w_lo, a_lo @ w_hi
        m = a.abs() @ w.abs()
        self.y += a @ w
        self.hh += hh
        self.hl += hl
        self.lh += lh
        self.M += m
        self.sw += (a != 0).double() @ w.abs()
        self.sa += a.abs().sum(-1, keepdim=True)
        p = hh + hl + lh
        s = self.hh + self.hl + self.lh
        self.run_abs += s.abs()
        self.pabs += p.abs()
        self.var += 3 * n_ks * (2 * 2.0 ** -23 * m) ** 2 + (U * s) ** 2

    @property
    def yh(self):
        return self.hh + self.hl + self.lh

    def elem_tol(self):
        return c_acc(self.n_ks) * self.M + U * (1 + 2.0 ** -20) * (self.run_abs + self.yh.abs())

    def rms_tol(self, live):
        """Bound on the RMS over `live` outputs of (got - yh) / M (see the module docstring)."""
        m = self.M[live]
        noise = torch.sqrt(((self.var[live] + (U * self.yh[live]) ** 2) / m ** 2).mean())
        bias = (12 * EPS * self.pabs[live] / m).max()
        return float(noise + bias)


def _rms(x):
    return float(torch.sqrt((x * x).mean()))


def check_against_model(got, ref, w_exp, what):
    """Per-element accumulation bound, aggregate RMS bound, representation bound, and the mutation checks."""
    got = got.double()
    live = ref.M > 0
    assert bool(live.any()), "%s: no output has a nonzero term" % what
    yh, M = ref.yh, ref.M
    assert torch.isfinite(got).all(), "%s: non-finite output" % what
    err = (got - yh).abs()
    tol = ref.elem_tol()
    # zero-magnitude outputs (no neighbour / all-zero operands) must be exact zeros
    assert float(err[~live].max()) == 0.0 if bool((~live).any()) else True, "%s: output without terms is not 0" % what
    worst = float((err[live] / tol[live]).max())
    assert worst <= 1.0, "%s: |got - yh| reaches %.3g of the accumulation bound" % (what, worst)
    rms = _rms((got - yh)[live] / M[live])
    rms_tol = ref.rms_tol(live)
    assert rms <= rms_tol, "%s: RMS relative error %.3g > %.3g" % (what, rms, rms_tol)
    # representation error: yh vs the exact result of the fp32 operands
    rep_tol = 2.0 ** -21 * M + 2.0 ** -25 * ref.sw + 2.0 ** -25 * math.ldexp(1.0, -w_exp) * ref.sa
    rep = float(((yh - ref.y).abs() - rep_tol).max())
    assert rep <= 0.0, "%s: |yh - y| exceeds its bound by %.3g" % (what, rep)
    # the same tolerances must reject kernels that drop a split term
    for name, dropped in (("A_lo.W_hi", ref.lh), ("A_hi.W_lo", ref.hl)):
        elem_ok = bool((dropped.abs() <= tol).all())
        rms_ok = _rms(dropped[live] / M[live]) <= rms_tol
        assert not (elem_ok and rms_ok), "%s: a kernel without the %s term would pass the tolerances" % (what, name)
    return dict(worst=worst, rms=rms, rms_tol=rms_tol)


# ---------------------------------------------------------------------------------------------------------------------
# sparse (output-stationary FP16x3)
# ---------------------------------------------------------------------------------------------------------------------

def _level(n, spatial, batch, seed):
    from det3d_b200.ops.spconv import core
    rng = np.random.default_rng(seed)
    d, h, w = spatial
    cells = rng.choice(batch * d * h * w, size=n, replace=False)
    b, rem = np.divmod(cells, d * h * w)
    z, rem = np.divmod(rem, h * w)
    yy, x = np.divmod(rem, w)
    coors = torch.from_numpy(np.stack([b, z, yy, x], 1).astype(np.int32)).cuda()
    return core.level_from_coors(coors, spatial, batch)


def _ksize(k_vol):
    return {27: (3, 3, 3), 3: (3, 1, 1), 1: (1, 1, 1)}[k_vol]


def _os16_pack(c_in, k_vol):
    """os16_pack of spconv16_sm90.cu: C_in 16 / 32 layers put 4 / 2 kernel offsets into one slot."""
    return 64 // c_in if k_vol > 1 and c_in in (16, 32) else 1


def sparse_ref(x, planes, w, w_exp, nbr, n_out):
    """Ref of out[o] = sum_k x[nbr[k, o]] @ w[k] with the kernel's slots: (offset group of `pack`, 64-channel slice kb),
    offsets ascending, kb inner."""
    k_vol, c_in, c_out = w.shape
    dev = w.device
    a = x.double()
    a_hi, a_lo = planes.hi.double(), planes.lo.double()
    w64 = w.double()
    w_hi, w_lo = weight_planes(w, w_exp)
    pack = _os16_pack(c_in, k_vol)
    ref = Ref((n_out, c_out), dev)
    zero = torch.zeros((1, c_in), dtype=torch.float64, device=dev)

    def gather(t, k):
        idx = nbr[k, :n_out].long()
        tz = torch.cat([t, zero])
        return tz[torch.where(idx >= 0, idx, t.shape[0])]

    for g in range(0, k_vol, pack):
        ks = list(range(g, min(g + pack, k_vol)))
        if pack > 1:              # one slot: the offsets side by side along K
            ga = [torch.cat([gather(t, k) for k in ks], 1) for t in (a, a_hi, a_lo)]
            gw = [torch.cat([t[k] for k in ks], 0) for t in (w64, w_hi, w_lo)]
            ref.slot(*ga[:1], *ga[1:], *gw, n_ks=4)
        else:
            ga = [gather(t, g) for t in (a, a_hi, a_lo)]
            for kb in range(0, c_in, 64):
                sl = slice(kb, min(kb + 64, c_in))
                ref.slot(ga[0][:, sl], ga[1][:, sl], ga[2][:, sl], w64[g][sl], w_hi[g][sl], w_lo[g][sl],
                         n_ks=min(4, (c_in - kb + 15) // 16))
    return ref


def run_sparse(c_in, c_out, k_vol, n, seed, a_scale=1.0, w_max=None, regime="C", cap=None, n_dev=None, spatial=(9, 40, 36),
               batch=2):
    """One FP16x3 sparse launch on seeded data -> (got [n_out, C_out] fp32, ref, w_exp, rulebook)."""
    from det3d_b200.ops.spconv import conv16, core
    gen = torch.Generator(device="cuda").manual_seed(seed)
    lvl = _level(n, spatial, batch, seed)
    if n_dev is not None:                        # fewer live rows than the capacity
        lvl.n.fill_(n_dev)
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, _ksize(k_vol)))
    n_out = n if n_dev is None else n_dev
    x, w = operands((n, c_in), (k_vol, c_in, c_out), regime, gen, a_scale, w_max)
    cw = conv16.ConvWeights16(w)
    planes = conv16.Planes.from_f32(x)
    out_f32 = torch.full((max(n, 1), c_out), float("nan"), device="cuda")
    conv16.sparse_conv16(planes, rb, cw, None, out_f32=out_f32)
    ref = sparse_ref(x, planes, w, cw.w_exp, rb.nbr, n_out)
    return out_f32[:n_out], ref, cw, rb, planes, x, w


def operands(a_shape, w_shape, regime, gen, a_scale=1.0, w_max=None):
    """Seeded operands. A: all positive; B: ReLU-like activations (half zeros) with zero-mean weights; C: zero-mean both.
    Weights are scaled so that outputs are O(a_scale) (or to max|w| = w_max)."""
    fan_in = float(np.prod(w_shape[:-1]))
    if regime == "A":
        x = torch.rand(a_shape, device="cuda", generator=gen) + 0.05
        w = torch.rand(w_shape, device="cuda", generator=gen) / fan_in
    elif regime == "B":
        x = torch.relu(torch.randn(a_shape, device="cuda", generator=gen))
        w = torch.randn(w_shape, device="cuda", generator=gen) / math.sqrt(fan_in * 0.5)
    else:
        x = torch.randn(a_shape, device="cuda", generator=gen)
        w = torch.randn(w_shape, device="cuda", generator=gen) / math.sqrt(fan_in)
    x = x * a_scale
    if w_max is not None:
        w = w * (w_max / float(w.abs().max()))
    return x.contiguous(), w.contiguous()


# ---------------------------------------------------------------------------------------------------------------------
# dense (pixel-stationary and pipelined FP16x3)
# ---------------------------------------------------------------------------------------------------------------------

def dense_ref(x, planes, wt, w_exp, ks, stride, pad, up):
    """Ref of the BevConv16 layer on NHWC x [B, H, W, C_in] with weights wt [up*up, ks*ks, C_in, C_out]: a gather-GEMM per
    tap in the kernel's slot order (64-channel slice kb, then kx, then ky); sub-pixel group g writes pixel
    (y*up + g // up, x*up + g % up)."""
    b, h, w, c_in = x.shape
    c_out = wt.shape[-1]
    ho, wo = (h + 2 * pad - ks) // stride + 1, (w + 2 * pad - ks) // stride + 1
    padf = lambda t: torch.nn.functional.pad(t.double(), (0, 0, pad, pad, pad, pad))
    xs = [padf(t) for t in (x, planes.hi, planes.lo)]
    w_hi, w_lo = weight_planes(wt, w_exp)
    w64 = wt.double()
    full = Ref((b, ho * up, wo * up, c_out), x.device)
    for g in range(up * up):
        ref = Ref((b, ho, wo, c_out), x.device)
        for kb in range(0, c_in, 64):
            sl = slice(kb, min(kb + 64, c_in))
            n_ks = min(4, (c_in - kb + 15) // 16)
            for kx in range(ks):
                for ky in range(ks):
                    win = [t[:, ky:ky + stride * (ho - 1) + 1:stride, kx:kx + stride * (wo - 1) + 1:stride, sl] for t in xs]
                    tap = ky * ks + kx
                    ref.slot(*win, w64[g, tap, sl], w_hi[g, tap, sl], w_lo[g, tap, sl], n_ks=n_ks)
        dy, dx = g // up, g % up
        for name in ("y", "hh", "hl", "lh", "M", "sw", "sa", "run_abs", "var", "pabs"):
            getattr(full, name)[:, dy::up, dx::up] = getattr(ref, name)
        full.n_ks = max(full.n_ks, ref.n_ks)
    return full


def dense_layer(wt, ks, stride, pad, up, **epi):
    from det3d_b200.ops.spconv import conv16
    return conv16.BevConv16(wt, ks, stride=stride, pad=pad, up=up, device="cuda", **epi)


def run_dense(b, h, w, c_in, c_out, ks, stride, pad, up, seed, a_scale=1.0, w_max=None, regime="C"):
    from det3d_b200.ops.spconv import conv16
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x, wt = operands((b, h, w, c_in), (up * up, ks * ks, c_in, c_out), regime, gen, a_scale, w_max)
    layer = dense_layer(wt, ks, stride, pad, up)
    planes = conv16.Planes.from_f32(x)
    ho, wo = layer.out_hw(h, w)
    out = torch.full((b, ho, wo, layer.c_out_padded), float("nan"), device="cuda")
    layer(planes, out_f32=out)
    ref = dense_ref(x, planes, wt, layer.w_exp, ks, stride, pad, up)
    return out[..., :c_out], ref, layer, planes, x, wt


def check_epilogue(got_f32, got_planes, ref, bias, scale, shift, relu, res=None, what=""):
    """Epilogue (bias, folded BN, residual, ReLU) and the f16 plane outputs against yh pushed through it in float64:
    the raw error bound carried through |scale|, plus one fp32 rounding per epilogue operation, plus the planes' 22 bits."""
    yh, tol = ref.yh, ref.elem_tol()
    v = yh + bias.double()
    t_v = tol + U * v.abs()
    v = v * scale.double() + shift.double()
    t_v = t_v * scale.double().abs() + U * v.abs()
    if res is not None:
        v = v + res.double()
        t_v = t_v + U * v.abs()
    if relu:
        v = torch.relu(v)
    err = (got_f32.double() - v).abs()
    assert bool((err <= t_v).all()), "%s: epilogue error %.3g over its bound" % (what, float((err - t_v).max()))
    p = got_planes.double()
    assert bool(((p - got_f32.double()).abs() <= 2.0 ** -22 * got_f32.double().abs() + 2.0 ** -25).all()), \
        "%s: planes do not hold the fp32 output to 22 bits" % what


def _epi_params(c_out, seed):
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    return (torch.randn(c_out, device="cuda", generator=g) * 0.1, torch.rand(c_out, device="cuda", generator=g) + 0.5,
            torch.randn(c_out, device="cuda", generator=g) * 0.1)


# ---------------------------------------------------------------------------------------------------------------------
# section 4: shape and edge sweep
# ---------------------------------------------------------------------------------------------------------------------

SPARSE_CIN = (8, 16, 24, 32, 48, 64, 96, 192, 256, 512)
SPARSE_COUT = (16, 32, 64, 128)


@pytest.mark.parametrize("c_in", SPARSE_CIN)
@pytest.mark.parametrize("c_out", SPARSE_COUT)
def test_sparse_fp16x3_error_model(c_in, c_out):
    """Every C_in the sparse FP16x3 kernel takes (ragged last 64-channel slice for 8 / 24 / 48 / 96, offset packing for
    16 / 32) x every C_out, 3x3x3 submanifold."""
    seed = c_in * 7 + c_out
    got, ref, cw, rb, planes, x, w = run_sparse(c_in, c_out, 27, 1500, seed)
    check_against_model(got, ref, cw.w_exp, "sparse C_in %d C_out %d" % (c_in, c_out))


@pytest.mark.parametrize("k_vol", [3, 1])
@pytest.mark.parametrize("c_in", [16, 32])
@pytest.mark.parametrize("c_out", [16, 64])
def test_sparse_fp16x3_small_kernels(k_vol, c_in, c_out):
    """(3,1,1) kernels: the only packed slot has phantom members; k_vol = 1 turns packing off (n_ks = 1 / 2)."""
    got, ref, cw, rb, planes, x, w = run_sparse(c_in, c_out, k_vol, 2000, 31 * k_vol + c_in + c_out)
    check_against_model(got, ref, cw.w_exp, "sparse k_vol %d C_in %d" % (k_vol, c_in))


@pytest.mark.parametrize("n,n_dev", [(1000, None),      # out_cap % 4 == 0: neighbour rows by cp.async.bulk
                                     (1001, None),      # out_cap % 4 != 0: per-thread neighbour loads
                                     (1001, 700),       # device row count below the capacity
                                     (1001, 0),         # zero rows
                                     (1, None),         # one row
                                     (300 * 128 + 5, None)])   # > 2 x 132 tiles: the persistent loop wraps
def test_sparse_fp16x3_row_counts(n, n_dev):
    got, ref, cw, rb, planes, x, w = run_sparse(32, 64, 27, n, n + 3, n_dev=n_dev, spatial=(20, 60, 60))
    from det3d_b200.ops.spconv import conv16
    out = torch.full((n, 64), float("nan"), device="cuda")
    conv16.sparse_conv16(planes, rb, cw, None, out_f32=out)
    n_out = n if n_dev is None else n_dev
    assert bool(torch.isnan(out[n_out:]).all()), "rows past the live count were written"
    if n_out:
        check_against_model(out[:n_out], ref, cw.w_exp, "sparse rows %d/%d" % (n_out, n))


@pytest.mark.parametrize("c_in", [1, 3, 4, 5, 7, 9, 12, 15])
@pytest.mark.parametrize("c_out", [16, 32, 64])
def test_sparse_first_layer_fp32_input(c_in, c_out):
    """The fp32-input first layer (C_in <= 16, not a multiple of 8): FFMA chains, so the reference is the exact y.
    A lane chains ceil(27 / 4) offsets x C_in FMAs, then two shuffle adds: L = 7 C_in + 2 roundings of at most u
    relative to the running magnitude <= M, |got - y| <= L u (1 + L u) M."""
    from det3d_b200.ops.spconv import conv16, core
    gen = torch.Generator(device="cuda").manual_seed(c_in * 13 + c_out)
    n = 3000
    lvl = _level(n, (9, 40, 36), 2, c_in + c_out)
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, 3))
    x, w = operands((n, c_in), (27, c_in, c_out), "C", gen)
    cw = conv16.ConvWeights16(w)
    assert cw.fp32_input
    out = torch.full((n, c_out), float("nan"), device="cuda")
    conv16.sparse_conv16(x, rb, cw, None, out_f32=out)
    idx = rb.nbr[:, :n].long()
    y = torch.zeros((n, c_out), dtype=torch.float64, device="cuda")
    m = torch.zeros_like(y)
    for k in range(27):
        ok = idx[k] >= 0
        y[ok] += x.double()[idx[k][ok]] @ w.double()[k]
        m[ok] += x.double().abs()[idx[k][ok]] @ w.double().abs()[k]
    L = 7 * c_in + 2
    err = (out.double() - y).abs()
    assert bool((err <= L * U * (1 + L * U) * m).all()), "first layer C_in %d: error %.3g of M" % (
        c_in, float((err / m.clamp_min(1e-300)).max()))


DENSE_CASES = [
    # b, h, w, c_in, c_out, ks, stride, pad, up
    (1, 1, 1, 16, 16, 3, 1, 1, 1),           # output grid of one pixel (less than a tile)
    (3, 7, 9, 32, 20, 3, 1, 1, 1),
    (2, 16, 16, 48, 64, 3, 1, 0, 1),         # pad 0
    (1, 17, 17, 80, 96, 3, 1, 2, 1),         # pad 2: output larger than the input
    (8, 7, 9, 96, 129, 3, 2, 1, 1),          # B = 8, two output blocks with a padded tail
    (1, 31, 45, 64, 256, 3, 2, 0, 1),
    (2, 17, 17, 192, 64, 3, 2, 2, 1),
    (2, 31, 45, 16, 256, 3, 1, 1, 1),
    (1, 31, 45, 80, 16, 1, 1, 0, 1),         # 1x1
    (1, 7, 9, 32, 32, 1, 1, 1, 1),           # 1x1 with pad 1: a zero border
    (4, 16, 16, 192, 129, 1, 1, 0, 1),
    (1, 7, 9, 48, 96, 1, 1, 0, 2),           # ConvTranspose2d(k = s = 2)
    (2, 17, 17, 32, 64, 1, 1, 0, 3),         # up 3
    (1, 16, 16, 96, 20, 1, 1, 0, 4),         # up 4
    (1, 1, 1, 64, 256, 1, 1, 0, 2),
]


@pytest.mark.parametrize("b,h,w,c_in,c_out,ks,stride,pad,up", DENSE_CASES)
def test_dense_fp16x3_error_model(b, h, w, c_in, c_out, ks, stride, pad, up):
    """Pixel-stationary BEV kernel: C_in multiples of 16 that are not multiples of 64 (ragged last slice), strides,
    pads, 1x1, ConvTranspose, padded C_out, grids below / at / above a 16 x 16 tile.  Raw sums through the error model,
    then the fused epilogue and the plane outputs."""
    from det3d_b200.ops.spconv import conv16
    seed = b * 1000 + h * 31 + c_in + c_out + 7 * up
    got, ref, layer, planes, x, wt = run_dense(b, h, w, c_in, c_out, ks, stride, pad, up, seed)
    what = "dense %s" % ((b, h, w, c_in, c_out, ks, stride, pad, up),)
    check_against_model(got, ref, layer.w_exp, what)
    if up == 1 and ks == 3 and pad == 1 and stride == 1:      # the float64 gather reference is conv2d itself
        want = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), wt[0].double().reshape(3, 3, c_in, c_out)
                                          .permute(3, 2, 0, 1), padding=1).permute(0, 2, 3, 1)
        assert float((want - ref.y).abs().max()) <= 1e-12 * float(ref.M.max())
    bias, scale, shift = _epi_params(c_out, seed)
    epi = dense_layer(wt, ks, stride, pad, up, bias=bias, scale=scale, shift=shift, relu=True)
    ho, wo = epi.out_hw(h, w)
    out = conv16.Planes((b, ho, wo, epi.c_out_padded), "cuda", zero=True)
    out32 = torch.zeros((b, ho, wo, epi.c_out_padded), device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    epi(planes, out=out, out_f32=out32, overflow=flag)
    assert int(flag.item()) == 0
    check_epilogue(out32[..., :c_out], out.to_f32()[..., :c_out], ref, bias, scale, shift, True, what=what)


def test_sparse_fp16x3_epilogue_and_planes():
    from det3d_b200.ops.spconv import conv16
    got, ref, cw, rb, planes, x, w = run_sparse(48, 64, 27, 3000, 5)
    check_against_model(got, ref, cw.w_exp, "sparse 48 -> 64")
    bias, scale, shift = _epi_params(64, 5)
    res = torch.randn((3000, 64), device="cuda")
    res_p = conv16.Planes.from_f32(res)
    cwe = conv16.ConvWeights16(w, bias=bias, scale=scale, shift=shift, relu=True)
    out = conv16.Planes((3000, 64), "cuda")
    out32 = torch.empty((3000, 64), device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    conv16.sparse_conv16(planes, rb, cwe, out, residual=res_p, out_f32=out32, overflow=flag)
    assert int(flag.item()) == 0
    check_epilogue(out32, out.to_f32(), ref, bias, scale, shift, True, res=res_p.to_f32(), what="sparse epilogue")


@pytest.mark.parametrize("c_in,b,c_out", [(64, 1, 128), (192, 3, 128), (256, 8, 256), (128, 3, 256)])
def test_pipelined_bit_identical(c_in, b, c_out):
    """The pipelined schedule (the automatic choice for 3x3 / stride 1 / 128-channel blocks / C_in % 64 == 0) gives the
    bits of the pixel-stationary one, on more C_in multiples of 64 and batch sizes, with a ragged grid."""
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16
    gen = torch.Generator(device="cuda").manual_seed(c_in + b)
    x, wt = operands((b, 21, 35, c_in), (1, 9, c_in, c_out), "B", gen)
    bias, scale, shift = _epi_params(c_out, c_in)
    layer = dense_layer(wt, 3, 1, 1, 1, bias=bias, scale=scale, shift=shift, relu=True)
    planes = conv16.Planes.from_f32(x)
    outs = []
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        for variant in (0, 2):
            _lib.lib().d3b_set_bev_variant(variant)
            out = conv16.Planes((b, 21, 35, c_out), "cuda", zero=True)
            out32 = torch.zeros((b, 21, 35, c_out), device="cuda")
            layer(planes, out=out, out_f32=out32)
            outs.append((out.buf, out32))
    finally:
        _lib.lib().d3b_set_bev_variant(prev)
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("a_exp", [-12, -6, 0, 6, 12])
@pytest.mark.parametrize("w_exp", [-30, -10, 0, 10])
def test_sparse_magnitude_sweep(a_exp, w_exp):
    """Activations x 2^k and weights with max|w| = 2^j: the bounds are scale-free, w_exp (clamped to +-40) moves the
    weights into the f16 range, and small activations hit the lo plane's subnormal floor."""
    got, ref, cw, rb, planes, x, w = run_sparse(64, 64, 27, 1500, 5000 + a_exp * 50 + w_exp,
                                                a_scale=2.0 ** a_exp, w_max=2.0 ** w_exp)
    assert float(x.abs().max()) < F16_MAX
    check_against_model(got, ref, cw.w_exp, "sparse 2^%d x 2^%d" % (a_exp, w_exp))


@pytest.mark.parametrize("a_exp,w_exp", [(k, 0) for k in (-12, -6, 0, 6, 12)] + [(0, j) for j in (-30, -10, 10)])
def test_dense_magnitude_sweep(a_exp, w_exp):
    got, ref, layer, planes, x, wt = run_dense(2, 19, 23, 96, 64, 3, 1, 1, 1, 5000 + a_exp * 50 + w_exp,
                                               a_scale=2.0 ** a_exp, w_max=2.0 ** w_exp)
    check_against_model(got, ref, layer.w_exp, "dense 2^%d x 2^%d" % (a_exp, w_exp))


# 65519.99 still rounds to a finite hi (65504), 65520 is the first value whose hi is inf: both must be flagged
BOUNDARY = [(65503.99, 0), (-65503.99, 0), (65504.0, 1), (-65504.0, 1), (65519.99, 1), (-65519.99, 1), (65520.0, 1),
            (-65520.0, 1), (1.0e5, 1), (float("inf"), 1), (float("-inf"), 1), (float("nan"), 1), (1.0, 0)]


def test_overflow_flag_boundary():
    """d3b_split16 and every FP16x3 epilogue flag exactly when |v| >= 65504 or v is inf / NaN (65503.99 is not);
    a launch that writes only out_f32 (the fused heads) never raises it."""
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16, core
    for v, want in BOUNDARY:
        flag = torch.zeros(1, dtype=torch.int32, device="cuda")
        conv16.Planes.from_f32(torch.tensor([[0.5, v, -2.0, 3.0]], device="cuda"), flag)
        assert int(flag.item()) == want, "split16(%r)" % v
    # epilogues: zero weights, the value through the bias (0 + b is exact)
    lvl = _level(300, (9, 40, 36), 1, 1)
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, 3))
    xin = conv16.Planes.from_f32(torch.randn((300, 32), device="cuda"))
    grid = conv16.Planes.from_f32(torch.randn((1, 9, 11, 64), device="cuda"))
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        for v, want in BOUNDARY:
            bias = torch.zeros(128, device="cuda")
            bias[5] = v
            cw = conv16.ConvWeights16(torch.zeros((27, 32, 128), device="cuda"), bias=bias)
            flag = torch.zeros(1, dtype=torch.int32, device="cuda")
            conv16.sparse_conv16(xin, rb, cw, conv16.Planes((300, 128), "cuda"), overflow=flag)
            assert int(flag.item()) == want, "sparse epilogue, v = %r" % v
            flag.zero_()
            conv16.sparse_conv16(xin, rb, cw, None, out_f32=torch.empty((300, 128), device="cuda"), overflow=flag)
            assert int(flag.item()) == 0, "sparse out_f32-only launch raised the flag (v = %r)" % v
            layer = dense_layer(torch.zeros((1, 9, 64, 128), device="cuda"), 3, 1, 1, 1, bias=bias)
            for variant in (0, 2):
                _lib.lib().d3b_set_bev_variant(variant)
                flag.zero_()
                layer(grid, out=conv16.Planes((1, 9, 11, 128), "cuda"), overflow=flag)
                assert int(flag.item()) == want, "dense epilogue (variant %d), v = %r" % (variant, v)
                flag.zero_()
                layer(grid, out_f32=torch.empty((1, 9, 11, 128), device="cuda"), overflow=flag)
                assert int(flag.item()) == 0, "dense out_f32-only launch raised the flag (v = %r)" % v
    finally:
        _lib.lib().d3b_set_bev_variant(prev)


# ---------------------------------------------------------------------------------------------------------------------
# section 5: bit-level invariants
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("c_in", [64, 32, 16])          # pack 1, 2, 4
@pytest.mark.parametrize("c_out", SPARSE_COUT)
def test_sparse_rows_independent_of_row_order(c_in, c_out):
    """Permuting the input rows (hence the level, the rulebook and the output rows) gives the same bits per row: a row's
    sum depends on its own neighbourhood, not on which rows share its 128-row tile (DESIGN 3.3)."""
    from det3d_b200.ops.spconv import conv16, core
    n = 2500
    rng = np.random.default_rng(c_in + c_out)
    d, h, w = 9, 40, 36
    cells = rng.choice(2 * d * h * w, size=n, replace=False)
    b, rem = np.divmod(cells, d * h * w)
    z, rem = np.divmod(rem, h * w)
    yy, xx = np.divmod(rem, w)
    coors = torch.from_numpy(np.stack([b, z, yy, xx], 1).astype(np.int32)).cuda()
    gen = torch.Generator(device="cuda").manual_seed(c_in * c_out)
    x, wt = operands((n, c_in), (27, c_in, c_out), "B", gen)
    cw = conv16.ConvWeights16(wt, bias=torch.randn(c_out, device="cuda") * 0.1, relu=True)
    perm = torch.from_numpy(rng.permutation(n)).cuda()
    outs = []
    for p in (torch.arange(n, device="cuda"), perm):
        lvl = core.level_from_coors(coors[p].contiguous(), (d, h, w), 2)
        rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, 3))
        out = conv16.Planes((n, c_out), "cuda")
        out32 = torch.empty((n, c_out), device="cuda")
        conv16.sparse_conv16(conv16.Planes.from_f32(x[p].contiguous()), rb, cw, out, out_f32=out32)
        back = torch.empty_like(p)
        back[p] = torch.arange(n, device="cuda")
        outs.append((out.buf[:, back], out32[back]))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("ks,stride,up,variant", [(3, 1, 1, 0), (3, 1, 1, 2), (3, 2, 1, 0), (1, 1, 2, 0)])
def test_dense_sample_independent_of_batch(ks, stride, up, variant):
    """Sample s alone (B = 1) and at position 1 of a B = 3 batch: the same bits (H = 37, W = 29 are not multiples of 16,
    so tiles reach past the sample border, where the TMA fill must be zeros, not the next sample)."""
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16
    gen = torch.Generator(device="cuda").manual_seed(ks * 10 + stride + up + variant)
    x, wt = operands((3, 37, 29, 64), (up * up, ks * ks, 64, 128), "B", gen)
    layer = dense_layer(wt, ks, stride, ks // 2, up, bias=torch.randn(128, device="cuda") * 0.1, relu=True)
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        _lib.lib().d3b_set_bev_variant(variant)
        res = []
        for xin in (x, x[1:2].contiguous()):
            ho, wo = layer.out_hw(37, 29)
            out = conv16.Planes((xin.shape[0], ho, wo, 128), "cuda")
            layer(conv16.Planes.from_f32(xin), out=out)
            res.append(out.buf)
    finally:
        _lib.lib().d3b_set_bev_variant(prev)
    assert torch.equal(res[0][:, 1], res[1][:, 0])


# ---------------------------------------------------------------------------------------------------------------------
# section 3: bias of the truncation correction
# ---------------------------------------------------------------------------------------------------------------------

def residual_slope(got, yh):
    """beta = sum (got - yh) yh / sum yh^2 and its standard error (outputs treated as independent)."""
    g, y = got.double().flatten(), yh.flatten()
    syy = float((y * y).sum())
    beta = float(((g - y) * y).sum()) / syy
    r = g - y - beta * y
    se = math.sqrt(float((r * r).sum()) / max(g.numel() - 1, 1) / syy)
    return beta, se


def bias_case(kernel, regime, seed=0):
    """One large seeded launch (>= 10^5 outputs) of `kernel` in operand `regime` -> (got, Ref, full slots' n)."""
    from det3d_b200 import _lib
    if kernel == "sparse":
        got, ref, *_ = run_sparse(64, 64, 27, 20000, 11 + seed, regime=regime, spatial=(20, 100, 100))
        return got, ref
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        _lib.lib().d3b_set_bev_variant(2 if kernel == "dense_pl" else 0)
        got, ref, *_ = run_dense(1, 96, 88, 128, 128, 3, 1, 1, 1, 23 + seed, regime=regime)
    finally:
        _lib.lib().d3b_set_bev_variant(prev)
    return got, ref


BIAS_B = 3 * EPS          # regime B (what the network feeds): a quarter of the 12-MMA correction
BIAS_ALL = 12 * EPS       # every regime: never worse than no correction at all


@pytest.mark.parametrize("kernel", ["sparse", "dense_ps", "dense_pl"])
@pytest.mark.parametrize("regime", ["A", "B", "C"])
def test_truncation_correction_bias(kernel, regime):
    """Residual slope of the kernel against yh over a large launch.  The FP16x3 kernels are deterministic, so on seeded
    inputs beta is reproducible.  A kernel without the correction (or with it twice) shifts beta by the 12 eps of a full
    slot; the regime-B bound must reject got * (1 -+ 12 eps)."""
    got, ref = bias_case(kernel, regime)
    assert got.numel() >= 10 ** 5
    beta, se = residual_slope(got, ref.yh)
    bound = BIAS_B if regime == "B" else BIAS_ALL
    print("%s regime %s: beta = %+.3f eps (se %.3f eps)" % (kernel, regime, beta / EPS, se / EPS))
    assert se < bound / 4, "standard error %.3g eps too large for a %.3g eps bound" % (se / EPS, bound / EPS)
    assert abs(beta) <= BIAS_ALL
    assert abs(beta) <= bound, "%s regime %s: beta = %.3f eps" % (kernel, regime, beta / EPS)
    if regime == "B":
        for m in (1 - 12 * EPS, 1 + 12 * EPS):
            assert abs(residual_slope(got.double() * m, ref.yh)[0]) > BIAS_B


# ---------------------------------------------------------------------------------------------------------------------
# section 6: the tf32x3 fallback where it runs (features beyond the f16 range)
# ---------------------------------------------------------------------------------------------------------------------

def tf32x3_bound(algo, c_in, k_vol):
    """|got - y| <= c M for the tf32x3 kernels.  Representation: hi = x with the low 13 mantissa bits cleared, lo = x - hi
    (|lo| < 2^-10 |x|) read by the tensor core as tf32 (error < 2^-10 |lo|), lo.lo dropped: 3 2^-20 M.  Accumulation:
    the output-stationary kernel chains every MMA of the layer (3 per k8 step, C_in / 8 steps per offset, k_vol offsets)
    into one uncorrected accumulator, each truncation < 2 ulp of the running magnitude <= M: 2 n 2^-23 M.  SIMT: one
    fp32 FMA chain of k_vol C_in terms."""
    c4 = (c_in + 3) // 4 * 4
    if algo == "simt":
        L = k_vol * c_in + 2
        return L * U * (1 + L * U)
    n = 3 * ((c4 + 7) // 8) * k_vol
    return 3 * 2.0 ** -20 + 2 * n * 2.0 ** -23


@pytest.mark.parametrize("algo", ["simt", "tc"])
@pytest.mark.parametrize("c_in,c_out", [(16, 32), (64, 64), (128, 128), (32, 32), (64, 128)])
def test_tf32x3_output_stationary_beyond_f16_range(algo, c_in, c_out):
    """Features around 3e5 (they trip the FP16x3 flag): simt and tc against the exact y, at the encoders' layer shapes."""
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16, core
    gen = torch.Generator(device="cuda").manual_seed(c_in + c_out)
    n = 4000
    lvl = _level(n, (9, 40, 36), 2, c_in)
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, 3))
    x, w = operands((n, c_in), (27, c_in, c_out), "C", gen, a_scale=3.0e5)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    conv16.Planes.from_f32(x, flag)
    assert int(flag.item()) == 1, "these features must be beyond the FP16x3 range"
    cw = core.ConvWeights(w, algo=_lib.ALGO_SIMT if algo == "simt" else _lib.ALGO_TC)
    out = torch.full((n, c_out), float("nan"), device="cuda")
    core.sparse_conv(x, rb, cw, out)
    idx = rb.nbr[:, :n].long()
    y = torch.zeros((n, c_out), dtype=torch.float64, device="cuda")
    m = torch.zeros_like(y)
    for k in range(27):
        ok = idx[k] >= 0
        y[ok] += x.double()[idx[k][ok]] @ w.double()[k]
        m[ok] += x.double().abs()[idx[k][ok]] @ w.double().abs()[k]
    c = tf32x3_bound(algo, c_in, 27)
    rel = float(((out.double() - y).abs() / m.clamp_min(1e-300)).max())
    print("tf32x3 %s C_in %d: max |got - y| / M = %.3g (bound %.3g)" % (algo, c_in, rel, c))
    assert rel <= c


@pytest.mark.parametrize("b,h,w,c_in,c_out", [(1, 61, 53, 64, 64), (2, 37, 29, 128, 128)])
def test_tf32x3_dense_beyond_f16_range(b, h, w, c_in, c_out):
    """The tf32x3 dense path (the gather kernel over a dense 3x3 rulebook, FusedBevStackTF32) at features ~3e5."""
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import bev, core
    gen = torch.Generator(device="cuda").manual_seed(h)
    x, wt = operands((b, h, w, c_in), (9, c_in, c_out), "B", gen, a_scale=3.0e5)
    grid = bev.BevGrid(b, h, w, "cuda")
    cw = core.ConvWeights(wt, algo=_lib.ALGO_TC)
    out = torch.full((b * h * w, c_out), float("nan"), device="cuda")
    core.sparse_conv(x.reshape(-1, c_in), grid.rulebook(3, 3, 1, 1), cw, out)
    w4 = wt.double().reshape(3, 3, c_in, c_out).permute(3, 2, 0, 1)
    xn = x.double().permute(0, 3, 1, 2)
    y = torch.nn.functional.conv2d(xn, w4, padding=1).permute(0, 2, 3, 1).reshape(-1, c_out)
    m = torch.nn.functional.conv2d(xn.abs(), w4.abs(), padding=1).permute(0, 2, 3, 1).reshape(-1, c_out)
    c = tf32x3_bound("tc", c_in, 9)
    rel = float(((out.double() - y).abs() / m.clamp_min(1e-300)).max())
    print("tf32x3 dense C_in %d: max |got - y| / M = %.3g (bound %.3g)" % (c_in, rel, c))
    assert rel <= c


# ---------------------------------------------------------------------------------------------------------------------
# BevConv16 channel slices with a padded C_out
# ---------------------------------------------------------------------------------------------------------------------

def test_bev_conv16_padded_cout_keeps_to_its_slice():
    """A C_out that is not a whole block (96 -> 128) computes padded columns: writing into a channel slice of a wider
    buffer would overwrite the neighbouring slice, so BevConv16 refuses it; its own padded buffer is fine."""
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16
    gen = torch.Generator(device="cuda").manual_seed(96)
    x, wt = operands((1, 20, 18, 64), (1, 9, 64, 96), "C", gen)
    layer = dense_layer(wt, 3, 1, 1, 1, bias=torch.randn(96, device="cuda"))
    assert layer.c_out_padded == 128
    planes = conv16.Planes.from_f32(x)
    wide = conv16.Planes((1, 20, 18, 32 + 96 + 64), "cuda", zero=True)
    with pytest.raises(_lib.D3BError):
        layer(planes, out=wide, out_c0=32)
    with pytest.raises(_lib.D3BError):
        layer(planes, out=wide, out_c0=0)
    with pytest.raises(_lib.D3BError):
        layer(planes, out_f32=torch.zeros((1, 20, 18, 192), device="cuda"))
    assert float(wide.buf.abs().max()) == 0.0
    own = torch.zeros((1, 20, 18, 128), device="cuda")
    layer(planes, out_f32=own)
    full = dense_layer(torch.cat([wt, wt.new_zeros((1, 9, 64, 32))], 3), 3, 1, 1, 1,
                       bias=torch.cat([layer.bias[:96], layer.bias.new_zeros(32)]))
    want = torch.zeros_like(own)
    full(planes, out_f32=want)
    assert torch.equal(own, want)
