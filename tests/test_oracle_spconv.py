"""Self-validation of the sparse-conv oracle (parity unpinned at the spconv boundary):
every layer type the Det3D encoders use must equal dense conv3d at the active output set."""
import numpy as np
import pytest
import torch

from oracle import spconv as osp


def _random_sites(rng, n, spatial, batch):
    d, h, w = spatial
    cells = rng.choice(batch * d * h * w, n, replace=False)
    b, r = cells // (d * h * w), cells % (d * h * w)
    return np.stack([b, r // (h * w), (r // w) % h, r % w], 1).astype(np.int32)


@pytest.mark.parametrize("k,s,p,subm", [(3, 1, 1, True), (3, 2, 1, False), (3, 2, [0, 1, 1], False),
                                        ((3, 1, 1), (2, 1, 1), 0, False), (1, 1, 0, True)])
def test_layer_equals_dense_conv3d(k, s, p, subm):
    rng = np.random.default_rng(7)
    spatial, batch = (9, 14, 11), 2
    coors = _random_sites(rng, 220, spatial, batch)
    feat = rng.standard_normal((220, 6)).astype(np.float32)
    kk = osp._triple(k)
    w = (rng.standard_normal((*kk, 6, 8)) * 0.2).astype(np.float32)
    err = osp.check_against_dense(feat, coors, spatial, batch, w, k, s, p, subm, bias=rng.standard_normal(8).astype(np.float32))
    assert err < 1e-5


def test_conv_outputs_sorted_and_unique():
    rng = np.random.default_rng(3)
    spatial = (11, 20, 16)
    coors = _random_sites(rng, 300, spatial, 3)
    oc, osp_ = osp.conv_outputs(coors, spatial, 3, 2, 1)
    lin = osp.linear_index(oc, osp_)
    assert (np.diff(lin) > 0).all()
    assert osp_ == (6, 10, 8)


def test_subm_centre_is_identity_and_symmetric():
    rng = np.random.default_rng(4)
    spatial = (8, 8, 8)
    coors = _random_sites(rng, 100, spatial, 1)
    nbr = osp.subm_neighbours(coors, spatial, 3)
    assert (nbr[13] == np.arange(100)).all()
    # (k, i -> o) exists iff (26-k, o -> i) exists
    for k in range(27):
        o = np.nonzero(nbr[k] >= 0)[0]
        assert (nbr[26 - k][nbr[k][o]] == o).all()


def test_middle_encoder_shapes():
    import sys
    from det3d_b200.models.backbones.scn import SpMiddleFHD, SpMiddleResNetFHD
    from det3d_b200.utils.synthetic import randomize_bn_
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    input_shape = [64, 80, 40]                      # x, y, z
    spatial = (17, 80, 64)
    coors = _random_sites(rng, 400, (40, 80, 64), 2)
    for cls, cin, cout in ((SpMiddleFHD, 4, 64), (SpMiddleResNetFHD, 5, 128)):
        m = randomize_bn_(cls(num_input_features=cin).eval())
        feats = rng.standard_normal((400, cin)).astype(np.float32)
        out = osp.middle_encoder_forward(m.state_dict(), feats, coors, 2, input_shape, arch=cls.__name__)
        assert out.shape == (2, cout * 2, 10, 8)
        assert torch.isfinite(out).all() and out.abs().sum() > 0


def _encoder_case(cls, cin, seed):
    from det3d_b200.utils.synthetic import randomize_bn_
    torch.manual_seed(seed)
    rng = np.random.default_rng(seed)
    m = randomize_bn_(cls(num_input_features=cin).eval(), seed)
    coors = _random_sites(rng, 400, (40, 80, 64), 2)
    feats = rng.standard_normal((400, cin)).astype(np.float32)
    return m.state_dict(), feats, coors, [64, 80, 40]


def _archs():
    from det3d_b200.models.backbones.scn import SpMiddleFHD, SpMiddleResNetFHD
    return ((SpMiddleFHD, 4), (SpMiddleResNetFHD, 5))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_middle_encoder_recorded_path_is_the_plain_path(dtype):
    """return_levels only records: the dense output has the same bits with and without it, in fp32 and float64."""
    for cls, cin in _archs():
        sd, feats, coors, shape = _encoder_case(cls, cin, 1)
        plain = osp.middle_encoder_forward(sd, feats, coors, 2, shape, arch=cls.__name__, dtype=dtype)
        rec, levels, _ = osp.middle_encoder_forward(sd, feats, coors, 2, shape, arch=cls.__name__, dtype=dtype,
                                                    return_levels=True)
        assert plain.dtype == dtype and torch.equal(plain, rec)
        assert len(levels) == (14 if cls.__name__ == "SpMiddleFHD" else 21)


def test_middle_encoder_float64_agrees_with_fp32():
    """The float64 oracle computes what the fp32 one does: within 1e-5 abs on every layer's output and the dense map
    (features are O(1) with randomized BatchNorm statistics; fp32 reorders alone stay far below that)."""
    for cls, cin in _archs():
        sd, feats, coors, shape = _encoder_case(cls, cin, 2)
        o32, l32, _ = osp.middle_encoder_forward(sd, feats, coors, 2, shape, arch=cls.__name__, return_levels=True)
        o64, l64, _ = osp.middle_encoder_forward(sd, feats, coors, 2, shape, arch=cls.__name__, return_levels=True,
                                                 dtype=torch.float64)
        assert o64.dtype == torch.float64 and float(o64.abs().max()) > 0.1
        assert float((o32.double() - o64).abs().max()) <= 1e-5
        for a, b in zip(l32, l64):
            assert a["output"].dtype == torch.float32 and b["output"].dtype == torch.float64
            assert np.array_equal(a["nbr"], b["nbr"]) and np.array_equal(a["coors"], b["coors"])
            assert float((a["output"].double() - b["output"]).abs().max()) <= 1e-5, a["conv"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_middle_encoder_levels_recompose_the_dense_map(dtype):
    """Every record is self-consistent and the chain is complete: each layer's output is indice_conv of its input
    through its nbr, its BatchNorm, its identity and a ReLU (same bits), each input is the previous output, each identity
    is the input of its block, and the last output scattered to dense is the returned map."""
    for cls, cin in _archs():
        sd, feats, coors, shape = _encoder_case(cls, cin, 3)
        out, levels, (x, c, sp) = osp.middle_encoder_forward(sd, feats, coors, 2, shape, arch=cls.__name__,
                                                             return_levels=True, dtype=dtype)
        sdd = {k: v.to(dtype) for k, v in sd.items()}
        assert torch.equal(levels[0]["input"], torch.as_tensor(feats, dtype=dtype))
        block_in = None
        for i, L in enumerate(levels):
            if i:
                assert L["input"] is levels[i - 1]["output"], L["conv"]
            if L["conv"].endswith("conv1"):
                block_in = L["input"]
            assert (L["identity"] is not None) == L["conv"].endswith("conv2")
            if L["identity"] is not None:
                assert L["identity"] is block_in
            y = osp.indice_conv(L["input"], sdd[L["conv"] + ".weight"], L["nbr"], L["coors"].shape[0],
                                sdd.get(L["conv"] + ".bias"), dtype)
            y = osp.batchnorm_eval(y, dict(running_mean=sdd[L["bn"] + ".running_mean"],
                                           running_var=sdd[L["bn"] + ".running_var"], weight=sdd[L["bn"] + ".weight"],
                                           bias=sdd[L["bn"] + ".bias"], eps=1e-3))
            if L["identity"] is not None:
                y = y + L["identity"]
            y = torch.relu(y)
            assert y.dtype == dtype and torch.equal(y, L["output"]), L["conv"]
            assert L["nbr"].shape == (int(np.prod(sdd[L["conv"] + ".weight"].shape[:3])), L["coors"].shape[0])
        assert x is levels[-1]["output"] and c is levels[-1]["coors"]
        d = osp.dense(levels[-1]["output"], levels[-1]["coors"], levels[-1]["spatial"], 2, dtype)
        assert torch.equal(d.view(out.shape), out)
