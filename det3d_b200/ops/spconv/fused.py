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
    __slots__ = ("conv", "bn", "relu", "residual", "save_identity", "cw", "sig", "cw16", "sig16")

    def __init__(self, conv, bn, relu, residual=False, save_identity=False):
        self.conv, self.bn, self.relu = conv, bn, relu
        self.residual = residual            # add the saved block input before the ReLU
        self.save_identity = save_identity  # this layer's INPUT is a block input
        self.cw = None
        self.sig = None
        self.cw16 = None
        self.sig16 = None


def _bn_fold(bn):
    """BatchNorm1d(eval) -> per-channel (scale, shift), computed in fp64."""
    var = bn.running_var.detach().double()
    mean = bn.running_mean.detach().double()
    gamma = bn.weight.detach().double() if bn.weight is not None else torch.ones_like(var)
    beta = bn.bias.detach().double() if bn.bias is not None else torch.zeros_like(var)
    scale = gamma / torch.sqrt(var + bn.eps)
    shift = beta - mean * scale
    return scale.float(), shift.float()


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
        # "fp16x3" (default): output-stationary wgmma kernels on split-f16 planes (csrc/spconv16_sm90.cu) --
        # deterministic, fused epilogues, no atomics.  "tf32x3": the round-1 kernels (pair-based + fp32 atomics, or
        # output-stationary with deterministic=True); also the fallback when a feature leaves the f16 range.
        self.math = "fp16x3"
        self.external_overflow = None   # int32[1] device flag shared with the rest of the model (else a private one)
        self.algo_override = None  # testing hook (tf32x3 path): force SIMT / TC for every layer
        # deterministic=True runs every layer output-stationary (D3B_ALGO_TC: one CTA owns an output tile, fixed
        # summation order, no atomics) -> bit-identical results run to run; the default pair-based kernel sums the
        # offsets' partial products with fp32 atomics, whose order varies
        self.deterministic = False
        self.overlap_rulebooks = True   # build the rulebook chain on a side stream (see run)

    # ---- parameters ------------------------------------------------------------
    def _refresh_weights(self, device):
        for L in self.plan:
            tensors = [L.conv.weight, L.conv.bias]
            if L.bn is not None:
                tensors += [L.bn.weight, L.bn.bias, L.bn.running_mean, L.bn.running_var]
            sig = tuple((None if t is None else (t._version, t.data_ptr())) for t in tensors) + (self.algo_override, self.deterministic)
            if L.cw is not None and L.sig == sig:
                continue
            if L.bn is not None and L.bn.training:
                raise RuntimeError("det3d_b200 sparse encoders are inference-only: call .eval() first")
            scale = shift = None
            if L.bn is not None:
                scale, shift = _bn_fold(L.bn)
                scale, shift = scale.to(device), shift.to(device)
            algo = self.algo_override
            if algo is None:   # sparse levels: compacted pairs on the tensor cores whenever the shape allows
                tc = _lib.ALGO_TC if self.deterministic else _lib.ALGO_TC_PAIRS
                algo = tc if core.tc_supported(L.conv.in_channels, L.conv.out_channels) else _lib.ALGO_SIMT
            L.cw = core.ConvWeights(
                L.conv.weight.to(device), bias=None if L.conv.bias is None else L.conv.bias.to(device),
                scale=scale, shift=shift, relu=L.relu, algo=algo,
            )
            L.sig = sig

    # ---- buffers -----------------------------------------------------------------
    def _build_state(self, cap0, spatial, batch, device):
        st = {"cap0": cap0, "spatial": tuple(spatial), "batch": batch, "device": device}
        n0 = torch.zeros(2, dtype=torch.int32, device=device)
        coors0 = torch.zeros((max(cap0, 1), 4), dtype=torch.int32, device=device)
        level = core.SparseLevel(coors0, n0, cap0, spatial, batch).build_hash_index()
        st["level0"] = level
        steps = []       # (layer, rulebook, build_fn or None)
        keyed = {}       # (indice_key) -> rulebook
        pools = {}
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
            pools.setdefault((rb.out_level.cap, conv.out_channels), [])
            steps.append((L, rb, build))
        st["steps"] = steps
        st["pools"] = pools
        st["final_level"] = cur
        c_last = self.plan[-1].conv.out_channels
        d, h, w = cur.spatial
        st["dense"] = torch.empty((batch, c_last, d, h, w), dtype=torch.float32, device=device)
        return st

    @staticmethod
    def _wants_pairs(st, rb):
        return any(M.cw.algo == _lib.ALGO_TC_PAIRS for M, r2, _b in st["steps"] if r2 is rb)

    @staticmethod
    def _take(pools, cap, c, busy, device):
        pool = pools[(cap, c)]
        for t in pool:
            if all(t is not b for b in busy):
                return t
        t = torch.empty((max(cap, 1), c), dtype=torch.float32, device=device)
        pool.append(t)
        return t

    # ---- run ------------------------------------------------------------------------
    def run(self, features, coors, batch_size, spatial, n_dev=None, row_cap=None, bev_rows=False):
        with _lib.on_device_of(features, coors, n_dev):
            return self._run(features, coors, batch_size, spatial, n_dev, row_cap, bev_rows)

    def _run(self, features, coors, batch_size, spatial, n_dev=None, row_cap=None, bev_rows=False):
        """features [M, C] f32, coors [M, 4] int (b,z,y,x) -> dense [B, C_out, D, H, W].

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
        if self.math == "fp16x3" and self.algo_override is None:
            return self._run16(st, features, coors, batch_size, n_dev, bev_rows)
        if bev_rows == "planes":
            raise ValueError("BEV planes are produced by the fp16x3 path only")
        self._refresh_weights(device)
        lvl0 = st["level0"]
        # adopt the caller's coordinate rows (zero-copy) for this run
        coors = coors.to(torch.int32).contiguous()
        feats = features.to(torch.float32).contiguous()
        if m == 0:  # keep pointers valid; the device row count (0) makes every kernel a no-op
            feats = torch.zeros((1, features.shape[1]), dtype=torch.float32, device=device)
        if m > 0:
            lvl0.coors[:m].copy_(coors)
        if n_dev is None:
            lvl0.n.fill_(m)
        else:
            lvl0.n[:1].copy_(n_dev.reshape(-1)[:1].to(torch.int32))
            lvl0.n[1:2].copy_(lvl0.n[:1])
        lvl0.rebuild_index()

        x = feats
        identity = None
        pending = None   # deferred epilogue (bias, scale, shift, relu) of the layer that produced raw sums in x
        x_level = lvl0

        def materialize():
            nonlocal pending
            if pending is not None:
                core.feature_epilogue(x, x_level, *pending[:3], relu=pending[3])
                pending = None

        # Rulebooks depend on coordinates only: build the whole chain (level 0 .. 3) on a side stream while the
        # main stream runs the convolutions of the levels already indexed.  Fork / join through events, so the
        # overlap is preserved as parallel branches when the forward is captured into a CUDA graph.
        main = torch.cuda.current_stream(device)
        ready = {}
        planes_cleared = None
        builds = [(rb, build) for _L, rb, build in st["steps"] if build is not None]
        # the pair-based kernel accumulates with atomics into a zeroed buffer: one dedicated output buffer per layer,
        # so that all of a resolution's targets can be cleared up front, off the critical path
        pair_outs = st.setdefault("pair_outs", {})
        for i, (L, rb, _b) in enumerate(st["steps"]):
            if L.cw.algo == _lib.ALGO_TC_PAIRS and i not in pair_outs:
                pair_outs[i] = torch.empty((max(rb.out_level.cap, 1), L.conv.out_channels), dtype=torch.float32, device=device)
        is_pairs = [L.cw.algo == _lib.ALGO_TC_PAIRS for L, _r, _b in st["steps"]]

        def prepare(rb, build):
            build(rb, with_pairs=self._wants_pairs(st, rb))
            bufs = [pair_outs[i] for i, (_L, r2, _b) in enumerate(st["steps"]) if r2 is rb and is_pairs[i]]
            if bufs:
                core.zero_rows(bufs, rb.out_level)

        if self.overlap_rulebooks and len(builds) > 1:
            side = st.get("side_stream")
            if side is None:
                side = st["side_stream"] = torch.cuda.Stream(device=device)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                for rb, build in builds:
                    prepare(rb, build)
                    ev = torch.cuda.Event()
                    ev.record(side)
                    ready[id(rb)] = ev
            builds = []
        waited = set()

        for i, (L, rb, build) in enumerate(st["steps"]):
            if build is not None and builds:   # single-stream order
                prepare(rb, build)
            if id(rb) in ready and id(rb) not in waited:
                main.wait_event(ready[id(rb)])
                waited.add(id(rb))
            pairs = L.cw.algo == _lib.ALGO_TC_PAIRS
            if L.save_identity:
                materialize()            # the block input is needed as activated values
                identity = x
            if not pairs:
                materialize()            # output-stationary kernels read activated inputs
            if pairs:
                out = pair_outs[i]
                core.sparse_conv(x, rb, L.cw, out, in_act=pending, out_zeroed=True)
                pending = (L.cw.bias, L.cw.scale, L.cw.shift, L.cw.relu)
                x, x_level = out, rb.out_level
                if L.residual:
                    core.feature_epilogue(x, x_level, *pending[:3], residual=identity, relu=pending[3])
                    pending, identity = None, None
            else:
                out = self._take(st["pools"], rb.out_level.cap, L.conv.out_channels, (x, identity), device)
                core.sparse_conv(x, rb, L.cw, out, residual=identity if L.residual else None)
                if L.residual:
                    identity = None
                x, x_level = out, rb.out_level
        materialize()
        if bev_rows:
            # channels-last [B*H*W, C*D] with channel = c*D + z: same values as dense.view(B, C*D, H, W)
            d, h, w = st["final_level"].spatial
            rows = st.get("bev_rows")
            if rows is None:
                rows = st["bev_rows"] = torch.empty((batch_size * h * w, x.shape[1] * d), dtype=torch.float32, device=device)
            rows.zero_()
            core.sparse_to_bev_rows(x, st["final_level"], rows)
            return rows
        dense = st["dense"]
        dense.zero_()
        core.sparse_to_dense(x, st["final_level"], out=dense)
        return dense

    # ---- FP16x3 path ------------------------------------------------------------------------
    def _refresh_weights16(self, device):
        for L in self.plan:
            tensors = [L.conv.weight, L.conv.bias]
            if L.bn is not None:
                tensors += [L.bn.weight, L.bn.bias, L.bn.running_mean, L.bn.running_var]
            sig = tuple((None if t is None else (t._version, t.data_ptr())) for t in tensors)
            if L.cw16 is not None and L.sig16 == sig:
                continue
            if L.bn is not None and L.bn.training:
                raise RuntimeError("det3d_b200 sparse encoders are inference-only: call .eval() first")
            scale = shift = None
            if L.bn is not None:
                scale, shift = _bn_fold(L.bn)
                scale, shift = scale.to(device), shift.to(device)
            L.cw16 = conv16.ConvWeights16(L.conv.weight.to(device), bias=None if L.conv.bias is None else L.conv.bias.to(device),
                                          scale=scale, shift=shift, relu=L.relu)
            L.sig16 = sig

    @staticmethod
    def _take16(pools, cap, c, busy, device):
        pool = pools.setdefault(("p16", cap, c), [])
        for t in pool:
            if all(t is not b for b in busy):
                return t
        t = conv16.Planes((max(cap, 1), c), device)
        pool.append(t)
        return t

    def _bev_planes(self, st, batch_size, device):
        """NHWC f16 planes [B, H, W, C * D] of the encoder output (scn.py:192-195: dense.view(N, C * D, H, W))."""
        planes = st.get("bev_planes")
        if planes is None or planes.shape[0] != batch_size:
            d, h, w = st["final_level"].spatial
            c = self.plan[-1].conv.out_channels
            planes = st["bev_planes"] = conv16.Planes((batch_size, h, w, c * d), device)
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

    def _run16(self, st, features, coors, batch_size, n_dev, bev_rows):
        device = features.device
        m = features.shape[0]
        self._refresh_weights16(device)
        lvl0 = st["level0"]
        coors = coors.to(torch.int32).contiguous()
        feats = features.to(torch.float32).contiguous()
        if m == 0:
            feats = torch.zeros((1, features.shape[1]), dtype=torch.float32, device=device)
        if m > 0:
            lvl0.coors[:m].copy_(coors)
        if n_dev is None:
            lvl0.n.fill_(m)
        else:
            lvl0.n[:1].copy_(n_dev.reshape(-1)[:1].to(torch.int32))
            lvl0.n[1:2].copy_(lvl0.n[:1])
        lvl0.rebuild_index()
        ovf = self.external_overflow
        if ovf is None:
            ovf = st.get("overflow")
            if ovf is None:
                ovf = st["overflow"] = torch.zeros(1, dtype=torch.int32, device=device)

        # rulebooks depend on coordinates only: the chain of all levels runs on a side stream (fork / join through
        # events, kept as parallel branches inside a CUDA graph) while the main stream convolves the levels already indexed
        main = torch.cuda.current_stream(device)
        ready = {}
        builds = [(rb, build) for _L, rb, build in st["steps"] if build is not None]
        if self.overlap_rulebooks and len(builds) > 1:
            side = st.get("side_stream")
            if side is None:
                side = st["side_stream"] = torch.cuda.Stream(device=device)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                for rb, build in builds:
                    build(rb, with_pairs=False)
                    ev = torch.cuda.Event()
                    ev.record(side)
                    ready[id(rb)] = ev
                if bev_rows:
                    # the BEV planes are cleared behind the rulebook chain, off the critical path (18 MB for SECOND)
                    self._bev_planes(st, batch_size, device).zero_()
                    planes_cleared = torch.cuda.Event()
                    planes_cleared.record(side)
            builds = []
        waited = set()

        first = self.plan[0].cw16
        x = feats if first.fp32_input else conv16.Planes.from_f32(feats, ovf)
        identity = None
        x_level = lvl0
        for L, rb, build in st["steps"]:
            if build is not None and builds:
                build(rb, with_pairs=False)
            if id(rb) in ready and id(rb) not in waited:
                main.wait_event(ready[id(rb)])
                waited.add(id(rb))
            if L.save_identity:
                identity = x
            out = self._take16(st["pools"], rb.out_level.cap, L.conv.out_channels, (x, identity), device)
            conv16.sparse_conv16(x, rb, L.cw16, out, residual=identity if L.residual else None, overflow=ovf)
            if L.residual:
                identity = None
            x, x_level = out, rb.out_level
        final = st["final_level"]
        d, h, w = final.spatial
        c = x.shape[-1]
        if bev_rows:
            planes = self._bev_planes(st, batch_size, device)
            assert tuple(planes.shape) == (batch_size, h, w, c * d)
            if planes_cleared is not None:
                main.wait_event(planes_cleared)
            else:
                planes.zero_()
            conv16.sparse_to_bev16(x, final, planes)
            if bev_rows == "planes":
                return planes
            rows = st.get("bev_rows")
            if rows is None:
                rows = st["bev_rows"] = torch.empty((batch_size * h * w, c * d), dtype=torch.float32, device=device)
            return planes.view(batch_size * h * w, c * d).to_f32(out=rows)
        rows32 = st.get("final_f32")
        if rows32 is None:
            rows32 = st["final_f32"] = torch.empty((max(final.cap, 1), c), dtype=torch.float32, device=device)
        x.to_f32(out=rows32)
        dense = st["dense"]
        dense.zero_()
        core.sparse_to_dense(rows32, final, out=dense)
        return dense

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
                               algo="fp16x3" if L.cw is None else L.cw.algo))
            tot_b += b
            tot_f += f
        return dict(layers=layers, bytes=tot_b, flops=tot_f, dense_bytes=int(self._state["dense"].numel() * 4))

    def last_levels(self):
        """(level, rulebook) pairs of the most recent run, for tests / roofline accounting."""
        return [(rb.out_level, rb, L) for (L, rb, _b) in self._state["steps"]]
