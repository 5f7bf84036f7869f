"""Device-resident sparse-convolution primitives over the det3d_b200 C ABI.

Everything here keeps the data-dependent row counts on the device (`n` is an
int32[2] tensor) and sizes buffers by a static capacity, so a whole middle
encoder runs without one host synchronisation and can be captured in a CUDA
graph.  The spconv-v1-style classes in `modules.py` and the fused encoder in
`fused.py` are thin layers over these functions.

Reference call sites being served: det3d/models/backbones/scn.py:106-157,
184-197, 323-370 (spconv.SparseConvTensor / SubMConv3d / SparseConv3d /
.dense()).  spconv itself is an un-vendored dependency of the reference.
"""
import ctypes as C

import numpy as np
import torch

from ... import _lib
from ..._lib import ConvParams, SiteIndex

TILE_M = 128


def _i3(v):
    return (C.c_int32 * 3)(*[int(x) for x in v])


def _triple(v):
    if isinstance(v, (list, tuple, np.ndarray)):
        assert len(v) == 3
        return tuple(int(x) for x in v)
    return (int(v),) * 3


def _pow2_at_least(n):
    c = 2
    while c < n:
        c <<= 1
    return c


class SparseLevel:
    """Active sites of one resolution: coordinates, device row count, lookup index."""

    def __init__(self, coors, n_dev, cap, spatial, batch):
        self.coors = coors          # [cap, 4] int32 (b, z, y, x)
        self.n = n_dev              # int32[2] device: [0] rows in use, [1] rows found
        self.cap = int(cap)
        self.spatial = tuple(int(s) for s in spatial)  # D, H, W
        self.batch = int(batch)
        self.index = None           # SiteIndex (ctypes) once built
        self._keep = []             # tensors backing the index

    @property
    def device(self):
        return self.coors.device

    def n_tiles(self):
        return (self.cap + TILE_M - 1) // TILE_M

    # -- level-0 index: hash --------------------------------------------------
    def build_hash_index(self):
        dev = self.device
        cap = _pow2_at_least(max(2 * self.cap, 1024))
        keys = torch.empty(cap, dtype=torch.int64, device=dev)
        vals = torch.empty(cap, dtype=torch.int32, device=dev)
        idx = SiteIndex()
        idx.spatial = _i3(self.spatial)
        idx.batch = self.batch
        idx.hash_keys = keys.data_ptr()
        idx.hash_vals = vals.data_ptr()
        idx.hash_cap = cap
        idx.bitmap = None
        idx.word_prefix = None
        idx.n_words = 0
        self.index = idx
        self._keep = [keys, vals]
        self.rebuild_index()
        return self

    def rebuild_index(self):
        """Re-run the hash insert for new coordinates in the same buffers."""
        assert self.index is not None and self.index.hash_keys
        with _lib.timed("rulebook", kind="hash"):
            st = _lib.lib().d3b_index_build_hash(
                self.coors.data_ptr(), self.n.data_ptr(), self.cap, C.byref(self.index), _lib.current_stream()
            )
        _lib.check(st, "d3b_index_build_hash")

    # -- strided-level index: bitmap ------------------------------------------
    def alloc_bitmap_index(self):
        dev = self.device
        cells = self.batch * self.spatial[0] * self.spatial[1] * self.spatial[2]
        n_words = (cells + 31) // 32
        n_alloc = (n_words + 3) // 4 * 4
        bitmap = torch.empty(n_alloc, dtype=torch.int32, device=dev)
        prefix = torch.empty(n_alloc, dtype=torch.int32, device=dev)
        idx = SiteIndex()
        idx.spatial = _i3(self.spatial)
        idx.batch = self.batch
        idx.hash_keys = None
        idx.hash_vals = None
        idx.hash_cap = 0
        idx.bitmap = bitmap.data_ptr()
        idx.word_prefix = prefix.data_ptr()
        idx.n_words = n_words
        self.index = idx
        self._keep = [bitmap, prefix]
        return self

    def count(self):
        """Host read of the row count (synchronises)."""
        return int(self.n[0].item())


class Rulebook:
    """Output-stationary neighbour map: nbr[k, o] = input row or -1."""

    def __init__(self, nbr, tile_mask, ksize, out_level, in_level, kind, stride=None, padding=None):
        self.nbr = nbr                # [K, out_cap] int32
        self.tile_mask = tile_mask    # [ceil(out_cap/128)] int32 (bit k = offset k used)
        self.ksize = ksize
        self.k_vol = ksize[0] * ksize[1] * ksize[2]
        self.out_level = out_level
        self.in_level = in_level
        self.kind = kind
        self.stride = stride
        self.padding = padding
        self._ws = None


def conv_out_spatial(spatial, ksize, stride, padding):
    return tuple((spatial[j] + 2 * padding[j] - (ksize[j] - 1) - 1) // stride[j] + 1 for j in range(3))


def max_outputs_per_input(ksize, stride):
    m = 1
    for k, s in zip(ksize, stride):
        m *= (k + s - 1) // s
    return m


def alloc_subm_rulebook(level, ksize):
    ksize = _triple(ksize)
    k_vol = ksize[0] * ksize[1] * ksize[2]
    dev = level.device
    nbr = torch.empty((k_vol, max(level.cap, 1)), dtype=torch.int32, device=dev)
    tile_mask = torch.empty(max(level.n_tiles(), 1), dtype=torch.int32, device=dev)
    return Rulebook(nbr, tile_mask, ksize, level, level, "subm")


def build_subm_rulebook(rb):
    level = rb.out_level
    with _lib.timed("rulebook", kind="subm", k_vol=rb.k_vol):
        st = _lib.lib().d3b_rulebook_subm(
            level.coors.data_ptr(), level.n.data_ptr(), level.cap, C.byref(level.index), _i3(rb.ksize),
            rb.nbr.data_ptr(), rb.tile_mask.data_ptr(), _lib.current_stream(),
        )
    _lib.check(st, "d3b_rulebook_subm")
    return rb


def alloc_conv_rulebook(in_level, ksize, stride, padding, out_cap=None):
    ksize, stride, padding = _triple(ksize), _triple(stride), _triple(padding)
    dev = in_level.device
    out_spatial = conv_out_spatial(in_level.spatial, ksize, stride, padding)
    cells = in_level.batch * out_spatial[0] * out_spatial[1] * out_spatial[2]
    if out_cap is None:
        out_cap = min(cells, in_level.cap * max_outputs_per_input(ksize, stride))
    out_cap = max(int(out_cap), 1)
    coors = torch.empty((out_cap, 4), dtype=torch.int32, device=dev)
    n = torch.zeros(2, dtype=torch.int32, device=dev)
    out_level = SparseLevel(coors, n, out_cap, out_spatial, in_level.batch).alloc_bitmap_index()
    k_vol = ksize[0] * ksize[1] * ksize[2]
    nbr = torch.empty((k_vol, out_cap), dtype=torch.int32, device=dev)
    tile_mask = torch.empty(out_level.n_tiles(), dtype=torch.int32, device=dev)
    rb = Rulebook(nbr, tile_mask, ksize, out_level, in_level, "conv", stride, padding)
    ws_bytes = _lib.lib().d3b_rulebook_workspace_bytes(out_level.index.n_words)
    rb._ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=dev)
    return rb


def build_conv_rulebook(rb):
    i, o = rb.in_level, rb.out_level
    with _lib.timed("rulebook", kind="conv", k_vol=rb.k_vol):
        st = _lib.lib().d3b_rulebook_conv(
            i.coors.data_ptr(), i.n.data_ptr(), i.cap, C.byref(i.index), _i3(rb.ksize), _i3(rb.stride),
            _i3(rb.padding), C.byref(o.index), o.coors.data_ptr(), o.n.data_ptr(), o.cap,
            rb.nbr.data_ptr(), rb.tile_mask.data_ptr(), rb._ws.data_ptr(), rb._ws.numel(),
            _lib.current_stream(),
        )
    _lib.check(st, "d3b_rulebook_conv")
    return rb


class ConvWeights:
    """Device-side parameters of one sparse conv with its fused epilogue."""

    def __init__(self, weight, bias=None, scale=None, shift=None, relu=False, algo=None):
        # weight: [kD, kH, kW, Cin, Cout] (spconv v1 layout) or [K, Cin, Cout]
        w = weight.detach().to(torch.float32)
        if w.dim() == 5:
            w = w.reshape(-1, w.shape[3], w.shape[4])
        self.c_in_logical = w.shape[1]
        if algo is None:
            algo = default_algo(w.shape[1], w.shape[2])
        if algo != _lib.ALGO_SIMT and w.shape[1] % 4 != 0:      # tensor-core kernels gather rows as float4
            w = torch.nn.functional.pad(w, (0, 0, 0, 4 - w.shape[1] % 4))
        self.weight = w.contiguous()
        self.k_vol, self.c_in, self.c_out = self.weight.shape
        f = lambda t: None if t is None else t.detach().to(torch.float32).contiguous()
        self.bias, self.scale, self.shift = f(bias), f(scale), f(shift)
        self.relu = bool(relu)
        self.packed = None
        self.algo = algo
        if self.algo != _lib.ALGO_SIMT:
            self._pack()

    def _pack(self):
        n = _lib.lib().d3b_conv_packed_weight_floats(self.c_in, self.c_out, self.k_vol)
        if n == 0:
            raise _lib.D3BError("tensor-core sparse conv does not support C_in=%d C_out=%d" % (self.c_in, self.c_out))
        self.packed = torch.empty(n, dtype=torch.float32, device=self.weight.device)
        st = _lib.lib().d3b_conv_pack_weight(
            self.weight.data_ptr(), self.c_in, self.c_out, self.k_vol, self.packed.data_ptr(), _lib.current_stream()
        )
        _lib.check(st, "d3b_conv_pack_weight")


def tc_supported(c_in, c_out):
    c_in = (int(c_in) + 3) // 4 * 4      # ConvWeights pads C_in to a multiple of 4 for the tensor-core kernels
    return _lib.lib().d3b_conv_packed_weight_floats(c_in, int(c_out), 27) > 0


def default_algo(c_in, c_out):
    return _lib.ALGO_TC if tc_supported(c_in, c_out) else _lib.ALGO_SIMT


def sparse_conv(feat_in, rb, cw, feat_out, residual=None):
    """feat_out[:n_out] = epilogue(sum_k feat_in[nbr[k]] @ W[k]).  All device-side."""
    if feat_in.shape[1] == cw.c_in_logical and cw.c_in != cw.c_in_logical:
        feat_in = torch.nn.functional.pad(feat_in, (0, cw.c_in - cw.c_in_logical))
    assert feat_in.dtype == torch.float32 and feat_in.is_contiguous() and feat_in.shape[1] == cw.c_in
    assert feat_out.shape[1] == cw.c_out and feat_out.is_contiguous()
    assert rb.k_vol == cw.k_vol, "kernel volume mismatch"
    assert feat_out.shape[0] >= rb.out_level.cap
    p = ConvParams()
    p.c_in, p.c_out, p.k_vol = cw.c_in, cw.c_out, cw.k_vol
    p.weight = cw.weight.data_ptr()
    p.weight_packed = None if cw.packed is None else cw.packed.data_ptr()
    p.bias = _lib.ptr(cw.bias)
    p.scale = _lib.ptr(cw.scale)
    p.shift = _lib.ptr(cw.shift)
    p.residual = _lib.ptr(residual)
    p.relu = 1 if cw.relu else 0
    p.algo = cw.algo
    dense = rb.kind == "dense2d"
    tag = ("bev3x3" if rb.k_vol == 9 else "bev1x1") if dense else "sparse"
    with _lib.timed(tag, c_in=cw.c_in, c_out=cw.c_out, k_vol=cw.k_vol, math="tf32x3"):
        st = _lib.lib().d3b_sparse_conv(
            feat_in.data_ptr(), rb.nbr.data_ptr(), rb.tile_mask.data_ptr(), rb.out_level.n.data_ptr(),
            rb.out_level.cap, C.byref(p), feat_out.data_ptr(), _lib.current_stream(),
        )
    _lib.check(st, "d3b_sparse_conv")
    return feat_out


def sparse_to_dense(feat, level, out=None):
    """rows -> [B, C, D, H, W]; `out` (if given) must be zero-filled by the caller."""
    c = feat.shape[1]
    d, h, w = level.spatial
    if out is None:
        out = torch.zeros((level.batch, c, d, h, w), dtype=torch.float32, device=feat.device)
    st = _lib.lib().d3b_sparse_to_dense(
        feat.data_ptr(), level.coors.data_ptr(), level.n.data_ptr(), level.cap, c, _i3(level.spatial),
        level.batch, out.data_ptr(), _lib.current_stream(),
    )
    _lib.check(st, "d3b_sparse_to_dense")
    return out


def sparse_to_bev_rows(feat, level, out):
    """rows -> channels-last BEV rows [B*H*W, C*D] (channel = c*D + z); `out` must be zero-filled."""
    c = feat.shape[1]
    st = _lib.lib().d3b_sparse_to_bev_rows(
        feat.data_ptr(), level.coors.data_ptr(), level.n.data_ptr(), level.cap, c, _i3(level.spatial),
        level.batch, out.data_ptr(), _lib.current_stream(),
    )
    _lib.check(st, "d3b_sparse_to_bev_rows")
    return out


def level_from_coors(coors, spatial, batch, n_dev=None):
    """Level 0 from caller coordinates ([M,4] int32 b,z,y,x) + hash index."""
    coors = coors.to(torch.int32).contiguous()
    cap = coors.shape[0]
    if n_dev is None:
        n_dev = torch.tensor([cap, cap], dtype=torch.int32, device=coors.device)
    if cap == 0:
        coors = torch.zeros((1, 4), dtype=torch.int32, device=coors.device)
    lvl = SparseLevel(coors, n_dev, cap, spatial, batch)
    return lvl.build_hash_index()
