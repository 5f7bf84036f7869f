"""TEST INFRASTRUCTURE -- sparse-convolution oracle (CPU, numpy + torch-CPU).

PARITY UNPINNED at this boundary: the reference delegates all sparse-conv
arithmetic to the external package `spconv` (fork github.com/poodarchu/spconv,
no pinned commit -- INSTALLATION.md:10-33; imported at
det3d/models/backbones/scn.py:4,9), which is neither vendored under
/root/reference nor installed here, and the reference has no tests or golden
vectors for it.  This file restates the published spconv v1.x algorithm
(`get_indice_pairs` + `indice_conv`: per kernel offset, gather rows ->
torch.mm -> scatter-add) and anchors it on (i) the reference's call sites --
layer lists, shapes and glue in scn.py:106-157,184-197,323-370 -- and (ii) a
self-validation every test run repeats: each layer must equal
torch.nn.functional.conv3d on the zero-filled dense tensor sampled at the
output active set (`check_against_dense`).

Conventions (SURVEY App. A.2):
  indices [N,4] int32 (batch, z, y, x); weight [kD,kH,kW,Cin,Cout];
  offset k enumerates (kz,ky,kx) row-major; input p feeds output o through k iff
  p = o*stride - padding + k;  SubM: outputs == inputs, same order;
  SparseConv3d: outputs = reachable in-bounds sites in ascending linear index
  ((b*D+z)*H+y)*W+x;  .dense() -> [B,C,D,H,W].
"""
import numpy as np
import torch


def _triple(v):
    return tuple(int(x) for x in v) if isinstance(v, (list, tuple, np.ndarray)) else (int(v),) * 3


def linear_index(coors, spatial):
    c = coors.astype(np.int64)
    d, h, w = spatial
    return ((c[:, 0] * d + c[:, 1]) * h + c[:, 2]) * w + c[:, 3]


def conv_out_spatial(spatial, ksize, stride, padding):
    return tuple((spatial[j] + 2 * padding[j] - (ksize[j] - 1) - 1) // stride[j] + 1 for j in range(3))


def _offsets(ksize):
    kz, ky, kx = np.meshgrid(np.arange(ksize[0]), np.arange(ksize[1]), np.arange(ksize[2]), indexing="ij")
    return np.stack([kz.ravel(), ky.ravel(), kx.ravel()], 1)  # [K,3], row-major k


class _Lookup:
    def __init__(self, coors, spatial):
        self.spatial = spatial
        lin = linear_index(coors, spatial)
        self.order = np.argsort(lin, kind="stable")
        self.sorted = lin[self.order]

    def find(self, b, zyx):
        d, h, w = self.spatial
        ok = ((zyx >= 0) & (zyx < np.array([d, h, w]))).all(1)
        lin = ((b.astype(np.int64) * d + zyx[:, 0]) * h + zyx[:, 1]) * w + zyx[:, 2]
        pos = np.searchsorted(self.sorted, lin)
        pos_c = np.minimum(pos, max(self.sorted.size - 1, 0))
        hit = ok & (pos < self.sorted.size)
        if self.sorted.size:
            hit &= self.sorted[pos_c] == lin
            row = np.where(hit, self.order[pos_c], -1)
        else:
            row = np.full(lin.shape, -1, np.int64)
        return row


def subm_neighbours(coors, spatial, ksize):
    """nbr [K, N] (input row or -1) for a submanifold conv (padding = k//2, stride 1)."""
    ksize = _triple(ksize)
    coors = np.asarray(coors)
    look = _Lookup(coors, spatial)
    offs = _offsets(ksize)
    pad = np.array([k // 2 for k in ksize])
    nbr = np.full((offs.shape[0], coors.shape[0]), -1, np.int64)
    for k, off in enumerate(offs):
        nbr[k] = look.find(coors[:, 0], coors[:, 1:4].astype(np.int64) - pad + off)
    return nbr


def conv_outputs(coors, spatial, ksize, stride, padding):
    """(out_coors [M,4] ascending linear index, out_spatial)."""
    ksize, stride, padding = _triple(ksize), _triple(stride), _triple(padding)
    coors = np.asarray(coors).astype(np.int64)
    out_sp = conv_out_spatial(spatial, ksize, stride, padding)
    cand = []
    s, p = np.array(stride), np.array(padding)
    for off in _offsets(ksize):
        t = coors[:, 1:4] + p - off
        ok = (t >= 0).all(1) & (t % s == 0).all(1)
        o = t // s
        ok &= (o < np.array(out_sp)).all(1)
        cand.append(np.concatenate([coors[ok, :1], o[ok]], 1))
    cand = np.concatenate(cand, 0) if cand else np.zeros((0, 4), np.int64)
    lin = linear_index(cand, out_sp)
    _, first = np.unique(lin, return_index=True)  # sorted ascending
    return cand[first].astype(np.int32), out_sp


def conv_neighbours(in_coors, in_spatial, out_coors, ksize, stride, padding):
    ksize, stride, padding = _triple(ksize), _triple(stride), _triple(padding)
    look = _Lookup(np.asarray(in_coors), in_spatial)
    offs = _offsets(ksize)
    oc = np.asarray(out_coors).astype(np.int64)
    nbr = np.full((offs.shape[0], oc.shape[0]), -1, np.int64)
    for k, off in enumerate(offs):
        nbr[k] = look.find(oc[:, 0], oc[:, 1:4] * np.array(stride) - np.array(padding) + off)
    return nbr


def pairs_of(nbr):
    """Rulebook in its canonical comparison form: sorted (k, in_row, out_row) triples."""
    k, o = np.nonzero(nbr >= 0)
    trip = np.stack([k, nbr[k, o], o], 1).astype(np.int64)
    return trip[np.lexsort((trip[:, 2], trip[:, 1], trip[:, 0]))]


def indice_conv(features, weight, nbr, n_out, bias=None, dtype=torch.float32):
    """spconv v1 indice_conv: for every offset with pairs, gather -> mm -> scatter-add (in `dtype`, fp32 by default)."""
    feats = torch.as_tensor(features, dtype=dtype)
    w = torch.as_tensor(weight, dtype=dtype)
    w = w.reshape(-1, w.shape[-2], w.shape[-1])
    out = torch.zeros((n_out, w.shape[2]), dtype=dtype)
    for k in range(w.shape[0]):
        o = np.nonzero(nbr[k] >= 0)[0]
        if o.size == 0:
            continue
        i = torch.from_numpy(nbr[k][o])
        out.index_add_(0, torch.from_numpy(o), feats[i] @ w[k])
    if bias is not None:
        out += torch.as_tensor(bias, dtype=dtype)
    return out


def dense(features, coors, spatial, batch, dtype=torch.float32):
    feats = torch.as_tensor(features, dtype=dtype)
    c = torch.as_tensor(np.asarray(coors)).long()
    d, h, w = spatial
    out = torch.zeros((batch, d, h, w, feats.shape[1]), dtype=dtype)
    out[c[:, 0], c[:, 1], c[:, 2], c[:, 3]] = feats
    return out.permute(0, 4, 1, 2, 3).contiguous()


def batchnorm_eval(x, bn):
    """nn.BatchNorm1d in eval mode on active rows (scn.py:103-104: eps 1e-3)."""
    return torch.nn.functional.batch_norm(x, bn["running_mean"], bn["running_var"], bn["weight"], bn["bias"],
                                          False, 0.0, bn["eps"])


def check_against_dense(features, coors, spatial, batch, weight, ksize, stride, padding, subm, bias=None):
    """Self-validation: sparse result == dense conv3d sampled at the output active set."""
    ksize, stride, padding = _triple(ksize), _triple(stride), _triple(padding)
    coors = np.asarray(coors)
    if subm:
        nbr = subm_neighbours(coors, spatial, ksize)
        out_coors, out_sp = coors, spatial
        dpad = tuple(k // 2 for k in ksize)
        dstride = (1, 1, 1)
    else:
        out_coors, out_sp = conv_outputs(coors, spatial, ksize, stride, padding)
        nbr = conv_neighbours(coors, spatial, out_coors, ksize, stride, padding)
        dpad, dstride = padding, stride
    sparse = indice_conv(features, weight, nbr, out_coors.shape[0], bias)
    x = dense(features, coors, spatial, batch)
    w = torch.as_tensor(weight, dtype=torch.float32).permute(4, 3, 0, 1, 2).contiguous()
    y = torch.nn.functional.conv3d(x, w, None, stride=dstride, padding=dpad)
    oc = torch.as_tensor(out_coors).long()
    sampled = y[oc[:, 0], :, oc[:, 1], oc[:, 2], oc[:, 3]]
    if bias is not None:
        sampled = sampled + torch.as_tensor(bias, dtype=torch.float32)
    if not subm:
        # every site the dense conv makes non-zero must be in the output active set
        nz = (y.abs().sum(1) > 0)
        act = torch.zeros_like(nz)
        act[oc[:, 0], oc[:, 1], oc[:, 2], oc[:, 3]] = True
        assert not (nz & ~act).any(), "dense conv produced a site missing from the sparse output set"
    return float((sparse - sampled).abs().max()) if sparse.numel() else 0.0


# ---- whole middle encoders (scn.py:106-157 and :323-355) -----------------------------
def _spec_fhd(cin):
    S, C = "subm", "conv"
    return [
        (S, cin, 16, 3, None, None, "subm0"), (S, 16, 16, 3, None, None, "subm0"),
        (C, 16, 32, 3, 2, 1, None),
        (S, 32, 32, 3, None, None, "subm1"), (S, 32, 32, 3, None, None, "subm1"),
        (C, 32, 64, 3, 2, 1, None),
        (S, 64, 64, 3, None, None, "subm2"), (S, 64, 64, 3, None, None, "subm2"), (S, 64, 64, 3, None, None, "subm2"),
        (C, 64, 64, 3, 2, [0, 1, 1], None),
        (S, 64, 64, 3, None, None, "subm3"), (S, 64, 64, 3, None, None, "subm3"), (S, 64, 64, 3, None, None, "subm3"),
        (C, 64, 64, (3, 1, 1), (2, 1, 1), 0, None),
    ]


def middle_encoder_forward(state_dict, voxel_features, coors, batch_size, input_shape, arch="SpMiddleFHD",
                           eps=1e-3, return_levels=False, dtype=torch.float32):
    """CPU forward of SpMiddleFHD / SpMiddleResNetFHD from a `middle_conv.*` state_dict, in `dtype` (fp32 by default;
    float64 gives a reference the fp32 device encoder can be measured against).

    Mirrors scn.py:184-197 / :357-370: sparse_shape = input_shape[::-1] + [1,0,0], the
    SparseSequential, .dense(), view(N, C*D, H, W).

    With return_levels=True, also returns one record per conv layer, in execution order: kind ("subm" / "conv"), the
    state_dict prefixes of its conv and BatchNorm, nbr [K, N_out] and the output coors / spatial shape, and the values
    around it -- `input` (the features it convolves), `identity` (the block input a residual layer adds before its ReLU,
    else None) and `output` (after BatchNorm, residual and ReLU: the next layer's input).
    """
    sd = {k: torch.as_tensor(v).to(dtype) if torch.is_tensor(v) or isinstance(v, np.ndarray) else v
          for k, v in state_dict.items()}
    spatial = tuple(int(s) for s in (np.array(input_shape[::-1]) + [1, 0, 0]))
    coors = np.asarray(coors).astype(np.int32)
    x = torch.as_tensor(voxel_features, dtype=dtype)
    cache = {}
    levels = []

    def bn(prefix, t):
        levels[-1]["bn"] = prefix
        return batchnorm_eval(t, dict(running_mean=sd[prefix + ".running_mean"], running_var=sd[prefix + ".running_var"],
                                      weight=sd[prefix + ".weight"], bias=sd[prefix + ".bias"], eps=eps))

    def conv(prefix, t, cur_coors, cur_sp, kind, k, s, p, key):
        w = sd[prefix + ".weight"]
        b = sd.get(prefix + ".bias")
        rec = dict(kind=kind, conv=prefix, bn=None, input=t, identity=None, output=None)
        levels.append(rec)
        if kind == "subm":
            ck = (key, cur_sp, cur_coors.shape[0])
            if key is None or ck not in cache:
                nbr = subm_neighbours(cur_coors, cur_sp, _triple(k))
                if key is not None:
                    cache[ck] = nbr
            else:
                nbr = cache[ck]
            rec.update(nbr=nbr, coors=cur_coors, spatial=cur_sp)
            return indice_conv(t, w, nbr, cur_coors.shape[0], b, dtype), cur_coors, cur_sp
        oc, osp = conv_outputs(cur_coors, cur_sp, k, s, p)
        nbr = conv_neighbours(cur_coors, cur_sp, oc, k, s, p)
        rec.update(nbr=nbr, coors=oc, spatial=osp)
        return indice_conv(t, w, nbr, oc.shape[0], b, dtype), oc, osp

    def done(t):
        levels[-1]["output"] = t
        return t

    cur_coors, cur_sp = coors, spatial
    if arch == "SpMiddleFHD":
        idx = 0
        for (kind, ci, co, k, s, p, key) in _spec_fhd(x.shape[1]):
            x, cur_coors, cur_sp = conv("middle_conv.%d" % idx, x, cur_coors, cur_sp, kind, k, s, p, key)
            x = done(torch.relu(bn("middle_conv.%d" % (idx + 1), x)))
            idx += 3
    elif arch == "SpMiddleResNetFHD":
        def block(i, t, key):
            pre = "middle_conv.%d" % i
            idt = t
            o, _, _ = conv(pre + ".conv1", t, cur_coors, cur_sp, "subm", 3, None, None, key)
            o = done(torch.relu(bn(pre + ".bn1", o)))
            o, _, _ = conv(pre + ".conv2", o, cur_coors, cur_sp, "subm", 3, None, None, key)
            levels[-1]["identity"] = idt
            o = bn(pre + ".bn2", o)
            return done(torch.relu(o + idt))

        def stem(i, t, kind, k, s, p, key):
            nonlocal cur_coors, cur_sp
            t, cur_coors, cur_sp = conv("middle_conv.%d" % i, t, cur_coors, cur_sp, kind, k, s, p, key)
            return done(torch.relu(bn("middle_conv.%d" % (i + 1), t)))

        x = stem(0, x, "subm", 3, None, None, "res0")
        x = block(3, x, "res0"); x = block(4, x, "res0")
        x = stem(5, x, "conv", 3, 2, 1, None)
        x = block(8, x, "res1"); x = block(9, x, "res1")
        x = stem(10, x, "conv", 3, 2, 1, None)
        x = block(13, x, "res2"); x = block(14, x, "res2")
        x = stem(15, x, "conv", 3, 2, [0, 1, 1], None)
        x = block(18, x, "res3"); x = block(19, x, "res3")
        x = stem(20, x, "conv", (3, 1, 1), (2, 1, 1), 0, None)
    else:
        raise ValueError(arch)
    out = dense(x, cur_coors, cur_sp, batch_size, dtype)
    n, c, d, h, w = out.shape
    out = out.view(n, c * d, h, w)
    if return_levels:
        return out, levels, (x, cur_coors, cur_sp)
    return out
