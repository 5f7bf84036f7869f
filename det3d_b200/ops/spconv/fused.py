"""Fused, sync-free executor for a Det3D sparse middle encoder.

Walks the `middle_conv` SparseSequential of SpMiddleFHD / SpMiddleResNetFHD
(det3d/models/backbones/scn.py:106-157, 323-355), folds every
`conv -> BatchNorm1d(eval) -> ReLU` triple (and every SparseBasicBlock,
scn.py:46-89, including its residual add) into one kernel launch per conv, and
runs rulebooks + convs + `.dense()` back to back on the current stream with
all row counts kept on the device.  Buffers are sized once per
(row capacity, batch) and reused, so the sequence is CUDA-graph capturable.
"""
import torch
from torch import nn

from ... import _lib
from . import conv16, core
from .modules import SparseConvolution


class _Layer:
    __slots__ = ("conv", "bn", "relu", "residual", "save_identity", "cw", "cw16", "sig")

    def __init__(self, conv, bn, relu, residual=False, save_identity=False):
        self.conv, self.bn, self.relu = conv, bn, relu
        self.residual = residual            # add the saved block input before the ReLU
        self.save_identity = save_identity  # this layer's INPUT is a block input
        self.cw = None      # tf32x3 device weights (core.ConvWeights)
        self.cw16 = None    # fp16x3 / fp16 device weights (conv16.ConvWeights16)
        self.sig = {}       # slot name -> the _signature its weights were made from


def _bn_fold(bn):
    """BatchNorm1d(eval) -> per-channel (scale, shift), computed in fp64."""
    var = bn.running_var.detach().double()
    mean = bn.running_mean.detach().double()
    gamma = bn.weight.detach().double() if bn.weight is not None else torch.ones_like(var)
    beta = bn.bias.detach().double() if bn.bias is not None else torch.zeros_like(var)
    scale = gamma / torch.sqrt(var + bn.eps)
    shift = beta - mean * scale
    return scale.float(), shift.float()


def _signature(L):
    """Identity of the parameters a layer's device weights were made from (version + storage of each tensor)."""
    tensors = [L.conv.weight, L.conv.bias]
    if L.bn is not None:
        tensors += [L.bn.weight, L.bn.bias, L.bn.running_mean, L.bn.running_var]
    return tuple((None if t is None else (t._version, t.data_ptr())) for t in tensors)


def _folded_bn(L, device):
    """(scale, shift) of the layer's BatchNorm on `device`, or (None, None) without one."""
    if L.bn is None:
        return None, None
    if L.bn.training:
        raise RuntimeError("det3d_b200 sparse encoders are inference-only: call .eval() first")
    scale, shift = _bn_fold(L.bn)
    return scale.to(device), shift.to(device)


def _conv_bias(L, device):
    return None if L.conv.bias is None else L.conv.bias.to(device)


def _is_basic_block(m):
    return all(hasattr(m, a) for a in ("conv1", "bn1", "conv2", "bn2", "relu")) and isinstance(
        getattr(m, "conv1"), SparseConvolution
    )


def compile_plan(middle_conv):
    """middle_conv (SparseSequential) -> list[_Layer]."""
    mods = list(middle_conv._modules.values())
    plan = []
    i = 0
    while i < len(mods):
        m = mods[i]
        if isinstance(m, SparseConvolution):
            bn = relu = None
            j = i + 1
            if j < len(mods) and isinstance(mods[j], nn.modules.batchnorm._BatchNorm):
                bn = mods[j]
                j += 1
            if j < len(mods) and isinstance(mods[j], nn.ReLU):
                relu = True
                j += 1
            plan.append(_Layer(m, bn, bool(relu)))
            i = j
        elif _is_basic_block(m):
            if getattr(m, "downsample", None) is not None:
                raise NotImplementedError("SparseBasicBlock.downsample is unused by the Det3D configs")
            plan.append(_Layer(m.conv1, m.bn1, True, save_identity=True))
            plan.append(_Layer(m.conv2, m.bn2, True, residual=True))
            i += 1
        else:
            raise NotImplementedError("cannot fuse module %r inside a sparse middle encoder" % type(m).__name__)
    return plan


class FusedSparseEncoder:
    def __init__(self, middle_conv):
        self.plan = compile_plan(middle_conv)
        self._state = None
        # "fp16x3" (default): output-stationary wgmma kernels on split-f16 planes (csrc/spconv16_sm90.cu).  "fp16": the
        # same kernels on the hi plane alone, one MMA per product (opt-in, not fp32-equivalent: DESIGN 3.0).  "tf32x3":
        # the output-stationary 3xTF32 kernels (csrc/sparse_conv_sm90.cu, SIMT where the shape is not built), the
        # fallback when a feature leaves the f16 range.  All are deterministic: fused epilogues, no atomics.
        self.math = "fp16x3"
        self.external_overflow = None   # int32[1] device flag shared with the rest of the model (else a private one)
        self.algo_override = None  # testing hook (tf32x3 path): force SIMT / TC for every layer
        self.overlap_rulebooks = True   # build the rulebook chain on a side stream (see _fork_rulebooks)

    # ---- parameters ------------------------------------------------------------
    def _refresh_weights(self, slot, device):
        """Makes each layer's device weights in `slot` ("cw": tf32x3, "cw16": the f16 maths) again where its parameters
        have changed."""
        for L in self.plan:
            sig = _signature(L) + ((self.algo_override,) if slot == "cw" else ())
            if L.sig.get(slot) == sig:
                continue
            scale, shift = _folded_bn(L, device)
            w = L.conv.weight.to(device)
            kw = dict(bias=_conv_bias(L, device), scale=scale, shift=shift, relu=L.relu)
            if slot == "cw":
                L.cw = core.ConvWeights(w, algo=self.algo_override, **kw)
            else:
                L.cw16 = conv16.ConvWeights16(w, **kw)
            L.sig[slot] = sig

    # ---- buffers -----------------------------------------------------------------
    def _build_state(self, cap0, spatial, batch, device):
        st = {"cap0": cap0, "spatial": tuple(spatial), "batch": batch, "device": device}
        n0 = torch.zeros(2, dtype=torch.int32, device=device)
        coors0 = torch.zeros((max(cap0, 1), 4), dtype=torch.int32, device=device)
        level = core.SparseLevel(coors0, n0, cap0, spatial, batch).build_hash_index()
        st["level0"] = level
        steps = []       # (layer, rulebook, build_fn or None)
        keyed = {}       # (indice_key) -> rulebook
        cur = level
        for L in self.plan:
            conv = L.conv
            build = None
            if conv.subm:
                key = (conv.indice_key, id(cur), tuple(conv.kernel_size)) if conv.indice_key is not None else None
                rb = keyed.get(key) if key is not None else None
                if rb is None:
                    rb = core.alloc_subm_rulebook(cur, conv.kernel_size)
                    build = core.build_subm_rulebook
                    if key is not None:
                        keyed[key] = rb
            else:
                rb = core.alloc_conv_rulebook(cur, conv.kernel_size, conv.stride, conv.padding)
                build = core.build_conv_rulebook
                cur = rb.out_level
            steps.append((L, rb, build))
        st["steps"] = steps
        st["pools"] = {}
        st["final_level"] = cur
        c_last = self.plan[-1].conv.out_channels
        d, h, w = cur.spatial
        st["dense"] = torch.empty((batch, c_last, d, h, w), dtype=torch.float32, device=device)
        return st

    @staticmethod
    def _take(pools, key, busy, make):
        """A buffer of pool `key` that is none of `busy`; make() adds one when all are busy."""
        pool = pools.setdefault(key, [])
        for t in pool:
            if all(t is not b for b in busy):
                return t
        t = make()
        pool.append(t)
        return t

    @staticmethod
    def _adopt_level0(st, features, coors, n_dev):
        """Take the caller's coordinate rows (and live-row count) as level 0 and index them; returns the fp32 features,
        which keep their row stride when their columns are contiguous (the FP16x3 first layer reads strided rows)."""
        device = features.device
        m = features.shape[0]
        lvl0 = st["level0"]
        coors = coors.to(torch.int32).contiguous()
        feats = features.to(torch.float32)
        if feats.stride(-1) != 1:
            feats = feats.contiguous()
        if m == 0:  # keep pointers valid; the device row count (0) makes every kernel a no-op
            feats = torch.zeros((1, features.shape[1]), dtype=torch.float32, device=device)
        else:
            lvl0.coors[:m].copy_(coors)
        if n_dev is None:
            lvl0.n.fill_(m)
        else:
            lvl0.n[:1].copy_(n_dev.reshape(-1)[:1].to(torch.int32))
            lvl0.n[1:2].copy_(lvl0.n[:1])
        lvl0.rebuild_index()
        return feats

    def _fork_rulebooks(self, st, device):
        """Rulebooks depend on coordinates only: build the whole chain (level 0 .. 3) on a side stream while the main
        stream runs the convolutions of the levels already indexed.  Fork / join through events, so the overlap is
        preserved as parallel branches when the forward is captured into a CUDA graph.

        Returns (side, before_conv): `side` is the side stream, or None when the chain is built in line on the main
        stream; before_conv(rb, build) is called before each step's convolution."""
        main = torch.cuda.current_stream(device)
        builds = [(rb, build) for _L, rb, build in st["steps"] if build is not None]
        if not (self.overlap_rulebooks and len(builds) > 1):
            def build_in_line(rb, build):
                if build is not None:
                    build(rb)
            return None, build_in_line
        side = st.get("side_stream")
        if side is None:
            side = st["side_stream"] = torch.cuda.Stream(device=device)
        side.wait_stream(main)
        ready = {}
        with torch.cuda.stream(side):
            for rb, build in builds:
                build(rb)
                ev = torch.cuda.Event()
                ev.record(side)
                ready[id(rb)] = ev

        def wait_once(rb, _build):
            ev = ready.pop(id(rb), None)
            if ev is not None:
                main.wait_event(ev)
        return side, wait_once

    # ---- run ------------------------------------------------------------------------
    def run(self, features, coors, batch_size, spatial, n_dev=None, row_cap=None, bev_rows=False):
        with _lib.on_device_of(features, coors, n_dev):
            return self._run(features, coors, batch_size, spatial, n_dev, row_cap, bev_rows)

    def _run(self, features, coors, batch_size, spatial, n_dev=None, row_cap=None, bev_rows=False):
        """features [M, C] f32, coors [M, 4] int (b,z,y,x) -> dense [B, C_out, D, H, W]; with `bev_rows` fp32 BEV rows
        [B*H*W, C*D] (channel = c*D + z: the values of dense.view(B, C*D, H, W), channels last), with
        bev_rows="planes" (f16 maths only) NHWC planes [B, H, W, C*D].

        With `n_dev` (int32[>=1] device tensor) only the first n_dev[0] rows are
        live and M is a capacity; otherwise all M rows are live.
        """
        device = features.device
        m = features.shape[0]
        cap_needed = m if row_cap is None else max(row_cap, m)
        st = self._state
        if (st is None or st["cap0"] < cap_needed or st["batch"] != batch_size
                or st["spatial"] != tuple(spatial) or st["device"] != device):
            st = self._state = self._build_state(cap_needed, spatial, batch_size, device)
        f16 = self.math in ("fp16x3", "fp16") and self.algo_override is None
        if bev_rows == "planes" and not f16:
            raise ValueError("BEV planes are produced by the fp16x3 / fp16 paths only")
        slot = "cw16" if f16 else "cw"
        self._refresh_weights(slot, device)
        feats = self._adopt_level0(st, features, coors, n_dev)
        if f16:
            ovf = self.external_overflow
            if ovf is None:
                ovf = st.get("overflow")
                if ovf is None:
                    ovf = st["overflow"] = torch.zeros(1, dtype=torch.int32, device=device)
            n_planes = self.n_planes
            pool = ("p16", n_planes)
            make = lambda cap, c: conv16.Planes((max(cap, 1), c), device, n_planes=n_planes)
            conv = lambda x, rb, cw, out, residual: conv16.sparse_conv16(x, rb, cw, out, residual=residual,
                                                                         overflow=ovf)
        else:
            pool = ("f32",)
            make = lambda cap, c: torch.empty((max(cap, 1), c), dtype=torch.float32, device=device)
            conv = core.sparse_conv
        side, before_conv = self._fork_rulebooks(st, device)
        planes_cleared = None
        if f16 and bev_rows and side is not None:
            # the BEV planes are cleared behind the rulebook chain, off the critical path (18 MB for SECOND)
            with torch.cuda.stream(side):
                self._bev_planes(st, batch_size, device).zero_()
                planes_cleared = torch.cuda.Event()
                planes_cleared.record(side)

        if not f16:
            x = feats.contiguous()
        elif self.plan[0].cw16.fp32_input:
            x = feats
        else:
            x = conv16.Planes.from_f32(feats, ovf, n_planes=n_planes)
        identity = None
        for L, rb, build in st["steps"]:
            before_conv(rb, build)
            if L.save_identity:
                identity = x
            cap, c = rb.out_level.cap, L.conv.out_channels
            out = self._take(st["pools"], pool + (cap, c), (x, identity), lambda: make(cap, c))
            conv(x, rb, getattr(L, slot), out, residual=identity if L.residual else None)
            if L.residual:
                identity = None
            x = out

        final = st["final_level"]
        d, h, w = final.spatial
        c = x.shape[-1]
        rows_shape = (batch_size * h * w, c * d)
        if bev_rows and not f16:
            rows = self._f32_buffer(st, "bev_rows", rows_shape, device)
            rows.zero_()
            return core.sparse_to_bev_rows(x, final, rows)
        if bev_rows:
            planes = self._bev_planes(st, batch_size, device)
            assert tuple(planes.shape) == (batch_size, h, w, c * d)
            if planes_cleared is not None:
                torch.cuda.current_stream(device).wait_event(planes_cleared)
            else:
                planes.zero_()
            conv16.sparse_to_bev16(x, final, planes)
            if bev_rows == "planes":
                return planes
            return planes.view(*rows_shape).to_f32(out=self._f32_buffer(st, "bev_rows", rows_shape, device))
        if f16:
            x = x.to_f32(out=self._f32_buffer(st, "final_f32", (max(final.cap, 1), c), device))
        dense = st["dense"]
        dense.zero_()
        return core.sparse_to_dense(x, final, out=dense)

    @staticmethod
    def _f32_buffer(st, key, shape, device):
        """The state's fp32 buffer `key`, allocated on first use."""
        t = st.get(key)
        if t is None:
            t = st[key] = torch.empty(shape, dtype=torch.float32, device=device)
        return t

    @property
    def n_planes(self):
        return 1 if self.math == "fp16" else 2

    def _bev_planes(self, st, batch_size, device):
        """NHWC f16 planes [B, H, W, C * D] of the encoder output (scn.py:192-195: dense.view(N, C * D, H, W))."""
        planes = st.get("bev_planes")
        if planes is None or planes.shape[0] != batch_size or planes.n_planes != self.n_planes:
            d, h, w = st["final_level"].spatial
            c = self.plan[-1].conv.out_channels
            planes = st["bev_planes"] = conv16.Planes((batch_size, h, w, c * d), device, n_planes=self.n_planes)
        return planes

    def overflowed(self):
        """True if a feature left the f16 range since the last call (synchronises; the flag is then cleared).
        The caller must re-run with math='tf32x3' -- nothing was saturated silently."""
        st = self._state
        flag = self.external_overflow if self.external_overflow is not None else (st or {}).get("overflow")
        if flag is None:
            return False
        hit = bool(int(flag.item()))
        if hit:
            flag.zero_()
        return hit

    def accounting(self):
        """Algorithmic bytes / flops of the most recent run (SURVEY 8d formulas; synchronises).

        per layer: bytes = N_in*Cin*4 + N_out*Cout*4 + P*8 + K*Cin*Cout*4, flops = 2*P*Cin*Cout,
        P = rulebook pairs.  Plus the dense write B*C*D*H*W*4 reported separately."""
        layers, tot_b, tot_f = [], 0, 0
        pair_cache = {}
        for L, rb, _b in self._state["steps"]:
            n_out = int(rb.out_level.n[0].item())
            n_in = int(rb.in_level.n[0].item())
            key = id(rb)
            if key not in pair_cache:
                pair_cache[key] = int((rb.nbr[:, :n_out] >= 0).sum().item()) if n_out else 0
            pairs = pair_cache[key]
            cin, cout, k = L.conv.in_channels, L.conv.out_channels, rb.k_vol
            b = n_in * cin * 4 + n_out * cout * 4 + pairs * 8 + k * cin * cout * 4
            f = 2 * pairs * cin * cout
            layers.append(dict(n_in=n_in, n_out=n_out, pairs=pairs, c_in=cin, c_out=cout, k_vol=k, bytes=b, flops=f,
                               algo=self.math if L.cw is None else L.cw.algo))
            tot_b += b
            tot_f += f
        return dict(layers=layers, bytes=tot_b, flops=tot_f, dense_bytes=int(self._state["dense"].numel() * 4))

    def last_levels(self):
        """(level, rulebook) pairs of the most recent run, for tests / roofline accounting."""
        return [(rb.out_level, rb, L) for (L, rb, _b) in self._state["steps"]]
