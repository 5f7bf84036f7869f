"""Single-pass FP16 without a GPU: the null-lo rule of the plane entry points (include/det3d_b200.h section 3b), the math
names, the pipeline's graph cache on a math switch, and wrap_fp16_model.

A plane entry point validates its arguments before any CUDA call, so every rejected combination below returns
D3B_ERR_INVALID_ARG (1) with a message on a host without a device.  The pointers are never dereferenced."""
import collections
import ctypes as C
import itertools
import os

import pytest
import torch

from conftest import ROOT

D3B_ERR_INVALID_ARG = 1
P = 0x10000            # a dummy "device" pointer: validation never dereferences it


def _lib():
    from det3d_b200 import _lib as L
    return L, L.lib()


def _rejected(lib, status, name):
    msg = (lib.d3b_last_error() or b"").decode()
    assert status == D3B_ERR_INVALID_ARG, "%s: status %d (%s)" % (name, status, msg)
    assert name in msg, msg
    return msg


def _conv16_params(L, **kw):
    p = L.Conv16Params()
    p.c_in, p.c_out, p.k_vol, p.acc_scale = 64, 64, 27, 1.0
    p.weight_packed = P
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _mixed(n):
    """Every on/off pattern of n lo pointers that is neither all on nor all off."""
    return [bits for bits in itertools.product((0, 1), repeat=n) if 0 < sum(bits) < n]


@pytest.mark.parametrize("bits", _mixed(3))
def test_sparse_conv16_rejects_mixed_lo_planes(bits):
    L, lib = _lib()
    in_lo, out_lo, res_lo = (P if b else None for b in bits)
    p = _conv16_params(L, in_hi=P, in_lo=in_lo, out_hi=P, out_lo=out_lo, residual_hi=P, residual_lo=res_lo)
    st = lib.d3b_sparse_conv16(P, P, P, 1000, C.byref(p), None)
    msg = _rejected(lib, st, "d3b_sparse_conv16")
    assert "single-pass" in msg


@pytest.mark.parametrize("bits", _mixed(2))
def test_sparse_conv16_first_layer_rejects_mixed_lo_planes(bits):
    """The fp32-input first layer: out and residual planes."""
    L, lib = _lib()
    out_lo, res_lo = (P if b else None for b in bits)
    p = _conv16_params(L, c_in=4, in_f32=P, weight=P, out_hi=P, out_lo=out_lo, residual_hi=P, residual_lo=res_lo)
    _rejected(lib, lib.d3b_sparse_conv16(P, P, P, 1000, C.byref(p), None), "d3b_sparse_conv16")


@pytest.mark.parametrize("which", ["in_lo", "out_lo", "residual_lo"])
def test_sparse_conv16_rejects_lo_without_hi(which):
    L, lib = _lib()
    kw = dict(in_hi=P, in_lo=P, out_hi=P, out_lo=P, residual_hi=P, residual_lo=P, out_f32=P)
    kw[which.replace("_lo", "_hi")] = None
    if which == "in_lo":
        kw.update(in_f32=P, weight=P, c_in=4)
    p = _conv16_params(L, **kw)
    _rejected(lib, lib.d3b_sparse_conv16(P, P, P, 1000, C.byref(p), None), "d3b_sparse_conv16")


def _bev16_params(L, **kw):
    p = L.Bev16Params()
    p.batch, p.h_in, p.w_in, p.c_in, p.c_out = 1, 16, 16, 64, 64
    p.ksize, p.stride, p.pad, p.groups, p.cgroups, p.up = 3, 1, 1, 1, 1, 1
    p.out_channels, p.acc_scale, p.weight_packed = 64, 1.0, P
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("in_lo,out_lo,out_hi", [(P, None, P), (None, P, P), (None, P, None), (P, P, None)])
def test_bev_conv16_rejects_mixed_lo_planes(in_lo, out_lo, out_hi):
    """in_lo without out_lo, out_lo without in_lo, and out_lo without out_hi (only out_f32 written)."""
    L, lib = _lib()
    p = _bev16_params(L, in_hi=P, in_lo=in_lo, out_hi=out_hi, out_lo=out_lo, out_f32=P)
    _rejected(lib, lib.d3b_bev_conv16(C.byref(p), None), "d3b_bev_conv16")


@pytest.mark.parametrize("in_hi,in_lo,in_f32,out_lo", [(P, P, None, None),     # plane rows, single-plane output
                                                       (P, None, None, P),     # single-plane rows, two-plane output
                                                       (None, P, P, P),        # fp32 rows with a stray in_lo
                                                       (None, P, P, None)])
def test_sparse_to_bev16_rejects_mixed_lo_planes(in_hi, in_lo, in_f32, out_lo):
    L, lib = _lib()
    sp = (C.c_int32 * 3)(1, 8, 8)
    st = lib.d3b_sparse_to_bev16(in_hi, in_lo, in_f32, P, P, 100, 64, sp, 1, P, out_lo, None, None)
    _rejected(lib, st, "d3b_sparse_to_bev16")


def test_split_merge_reject_lo_without_hi():
    L, lib = _lib()
    _rejected(lib, lib.d3b_split16(P, 100, None, P, None, None), "d3b_split16")
    _rejected(lib, lib.d3b_merge16(None, P, 100, P, None), "d3b_merge16")


def _model(name="second_kitti_car.py"):
    from det3d.models import build_detector
    from det3d.torchie import Config
    cfg = Config.fromfile(os.path.join(ROOT, "configs", name))
    return build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)


def test_set_math_names():
    model = _model()
    assert model.math == "fp16x3"
    for bad in ("fp32", "FP16", "bf16", "", None):
        with pytest.raises(ValueError):
            model.set_math(bad)
    assert model.math == "fp16x3"
    for m in ("fp16", "tf32x3", "fp16x3"):
        model.set_math(m)
        assert model.math == m and model.backbone.fused().math == m


def test_pipeline_set_math_drops_captured_graphs():
    from det3d_b200.apis.pipeline import InferencePipeline
    pipe = InferencePipeline.__new__(InferencePipeline)      # no device needed for the cache logic
    pipe.model = _model()
    pipe._graphs = collections.OrderedDict([((1, 1024, 4), object()), (("stream", 2, 3, 4096, 5, 5), object())])
    pipe.set_math("fp16")
    assert pipe.model.math == "fp16" and len(pipe._graphs) == 0
    with pytest.raises(ValueError):
        pipe.set_math("int8")


@pytest.mark.parametrize("name", ["second_kitti_car.py", "pointpillars_kitti_car.py", "cbgs_nusc.py"])
def test_wrap_fp16_model_selects_fp16_and_keeps_fp32_parameters(name):
    from det3d.core.fp16 import wrap_fp16_model
    model = _model(name)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    assert wrap_fp16_model(model) is model
    assert model.math == "fp16" and model.fp16_enabled
    assert model.n_planes() == 1
    fused = getattr(model.backbone, "fused", None)
    if fused is not None:
        assert fused().math == "fp16"
    after = model.state_dict()
    for k, v in before.items():
        assert after[k].dtype == v.dtype and torch.equal(after[k], v), k
    assert all(p.dtype == torch.float32 for p in model.parameters())
