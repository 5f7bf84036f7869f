"""Rulebook (bit-exact) and sparse convolution (<= 1e-4 abs) vs the oracle; fused encoders vs
the oracle's SpMiddleFHD / SpMiddleResNetFHD forward."""
import numpy as np
import pytest
import torch

from oracle import spconv as osp

pytestmark = pytest.mark.gpu
TOL = 1e-4  # BASELINE.json north_star: float features within 1e-4 abs


def _sites(rng, n, spatial, batch):
    d, h, w = spatial
    cells = rng.choice(batch * d * h * w, n, replace=False)
    b, r = cells // (d * h * w), cells % (d * h * w)
    return np.stack([b, r // (h * w), (r // w) % h, r % w], 1).astype(np.int32)


def _nbr_to_numpy(rb, n_out):
    return rb.nbr[:, :n_out].cpu().numpy().astype(np.int64)


@pytest.mark.parametrize("n,spatial,batch", [(500, (9, 20, 24), 2), (5000, (41, 160, 140), 1), (1, (5, 5, 5), 1)])
@pytest.mark.parametrize("ksize", [3, (3, 1, 1), 1])
def test_subm_rulebook_bit_exact(n, spatial, batch, ksize):
    from det3d_b200.ops.spconv import core
    rng = np.random.default_rng(n)
    coors = _sites(rng, n, spatial, batch)
    lvl = core.level_from_coors(torch.from_numpy(coors).cuda(), spatial, batch)
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, ksize))
    got = _nbr_to_numpy(rb, n)
    want = osp.subm_neighbours(coors, spatial, ksize)
    assert np.array_equal(got, want)
    mask = rb.tile_mask.cpu().numpy().astype(np.uint32)
    for t in range((n + 127) // 128):
        bits = 0
        for k in range(want.shape[0]):
            if (want[k, t * 128:(t + 1) * 128] >= 0).any():
                bits |= 1 << k
        assert int(mask[t]) == bits


@pytest.mark.parametrize("k,s,p", [(3, 2, 1), (3, 2, [0, 1, 1]), ((3, 1, 1), (2, 1, 1), 0)])
@pytest.mark.parametrize("n,spatial,batch", [(800, (11, 40, 36), 2), (6000, (41, 200, 176), 1)])
def test_conv_rulebook_bit_exact(k, s, p, n, spatial, batch):
    from det3d_b200.ops.spconv import core
    rng = np.random.default_rng(n + 1)
    coors = _sites(rng, n, spatial, batch)
    lvl = core.level_from_coors(torch.from_numpy(coors).cuda(), spatial, batch)
    rb = core.build_conv_rulebook(core.alloc_conv_rulebook(lvl, k, s, p))
    want_coors, want_sp = osp.conv_outputs(coors, spatial, k, s, p)
    n_out = rb.out_level.count()
    assert rb.out_level.spatial == tuple(want_sp)
    assert n_out == want_coors.shape[0] and int(rb.out_level.n[1]) == n_out
    assert np.array_equal(rb.out_level.coors[:n_out].cpu().numpy(), want_coors)          # ascending linear index
    want = osp.conv_neighbours(coors, spatial, want_coors, k, s, p)
    assert np.array_equal(_nbr_to_numpy(rb, n_out), want)
    assert np.array_equal(osp.pairs_of(_nbr_to_numpy(rb, n_out)), osp.pairs_of(want))    # canonical triple form
    # second level through the bitmap index: SubM on the conv outputs
    rb2 = core.build_subm_rulebook(core.alloc_subm_rulebook(rb.out_level, 3))
    assert np.array_equal(_nbr_to_numpy(rb2, n_out), osp.subm_neighbours(want_coors, want_sp, 3))


def test_conv_rulebook_overflow_is_reported():
    from det3d_b200.ops.spconv import core
    rng = np.random.default_rng(5)
    spatial = (9, 30, 30)
    coors = _sites(rng, 400, spatial, 1)
    lvl = core.level_from_coors(torch.from_numpy(coors).cuda(), spatial, 1)
    rb = core.build_conv_rulebook(core.alloc_conv_rulebook(lvl, 3, 2, 1, out_cap=50))
    want_coors, _ = osp.conv_outputs(coors, spatial, 3, 2, 1)
    assert int(rb.out_level.n[0]) == 50 and int(rb.out_level.n[1]) == want_coors.shape[0]
    assert np.array_equal(rb.out_level.coors[:50].cpu().numpy(), want_coors[:50])


ALGOS = ["simt", "tc"]


def _algo(name):
    from det3d_b200 import _lib
    return {"simt": _lib.ALGO_SIMT, "tc": _lib.ALGO_TC}[name]


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("cin,cout,k,s,p,subm", [
    (4, 16, 3, 1, 1, True), (5, 16, 3, 1, 1, True), (16, 16, 3, 1, 1, True), (16, 32, 3, 2, 1, False),
    (32, 32, 3, 1, 1, True), (32, 64, 3, 2, 1, False), (64, 64, 3, 1, 1, True), (64, 64, 3, 2, [0, 1, 1], False),
    (64, 128, 3, 2, [0, 1, 1], False), (128, 128, 3, 1, 1, True), (64, 64, (3, 1, 1), (2, 1, 1), 0, False),
    (128, 128, (3, 1, 1), (2, 1, 1), 0, False),
    # partial and odd 32-channel slots, C_out < C_in, k_vol 1 and 9
    (48, 32, 3, 1, 1, True), (96, 128, 3, 1, 1, True), (128, 64, 3, 1, 1, True), (32, 16, 3, 2, 1, False),
    (64, 64, 1, 1, 0, True), (16, 32, (1, 3, 3), 1, 0, True)])
def test_output_stationary_layer_vs_oracle(algo, cin, cout, k, s, p, subm):
    from det3d_b200.ops.spconv import core
    if algo != "simt" and not core.tc_supported(cin, cout):
        pytest.skip("tensor-core kernels do not take C_in=%d" % cin)
    rng = np.random.default_rng(cin * 1000 + cout)
    spatial, batch, n = (11, 48, 40), 2, 3000
    coors = _sites(rng, n, spatial, batch)
    feat = rng.standard_normal((n, cin)).astype(np.float32)
    kk = osp._triple(k)
    w = (rng.standard_normal((*kk, cin, cout)) / np.sqrt(cin * np.prod(kk) / 3)).astype(np.float32)
    bias = rng.standard_normal(cout).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, cout).astype(np.float32)
    shift = rng.standard_normal(cout).astype(np.float32)
    lvl = core.level_from_coors(torch.from_numpy(coors).cuda(), spatial, batch)
    if subm:
        rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, k))
        nbr, n_out = osp.subm_neighbours(coors, spatial, k), n
    else:
        rb = core.build_conv_rulebook(core.alloc_conv_rulebook(lvl, k, s, p))
        oc, _ = osp.conv_outputs(coors, spatial, k, s, p)
        nbr, n_out = osp.conv_neighbours(coors, spatial, oc, k, s, p), oc.shape[0]
    res = rng.standard_normal((n_out, cout)).astype(np.float32)
    cw = core.ConvWeights(torch.from_numpy(w).cuda(), bias=torch.from_numpy(bias).cuda(),
                          scale=torch.from_numpy(scale).cuda(), shift=torch.from_numpy(shift).cuda(), relu=True,
                          algo=_algo(algo))
    out = torch.full((rb.out_level.cap, cout), float("nan"), device="cuda")
    res_dev = torch.zeros((rb.out_level.cap, cout), device="cuda")
    res_dev[:n_out] = torch.from_numpy(res).cuda()
    core.sparse_conv(torch.from_numpy(feat).cuda(), rb, cw, out, residual=res_dev)
    want = torch.relu((osp.indice_conv(feat, w, nbr, n_out, bias) * torch.from_numpy(scale) + torch.from_numpy(shift))
                      + torch.from_numpy(res))
    got = out[:n_out].cpu()
    assert torch.isfinite(got).all()
    assert float((got - want).abs().max()) <= TOL
    if rb.out_level.cap > n_out:
        assert torch.isnan(out[n_out:]).all()      # rows beyond the live count are never written


def _encoder_case(cls_name, cin, n, seed, spatial_xyz=(96, 112, 40), batch=2):
    from det3d_b200.models.backbones import scn
    from det3d_b200.utils.synthetic import randomize_bn_
    torch.manual_seed(seed)
    rng = np.random.default_rng(seed)
    model = randomize_bn_(getattr(scn, cls_name)(num_input_features=cin).eval(), seed)
    x, y, z = spatial_xyz
    coors = _sites(rng, n, (z, y, x), batch)
    feats = rng.standard_normal((n, cin)).astype(np.float32)
    return model, feats, coors, list(spatial_xyz), batch


@pytest.mark.parametrize("algo", ["auto", "simt", "tc"])
@pytest.mark.parametrize("cls_name,cin", [("SpMiddleFHD", 4), ("SpMiddleResNetFHD", 5)])
def test_fused_encoder_vs_oracle(cls_name, cin, algo):
    from det3d_b200 import _lib
    model, feats, coors, input_shape, batch = _encoder_case(cls_name, cin, 6000, 3)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    want = osp.middle_encoder_forward(sd, feats, coors, batch, input_shape, arch=cls_name)
    model = model.cuda()
    if algo != "auto":
        model.fused().algo_override = _lib.ALGO_SIMT if algo == "simt" else _lib.ALGO_TC
    got = model(torch.from_numpy(feats).cuda(), torch.from_numpy(coors).cuda(), batch, input_shape).cpu()
    assert got.shape == want.shape
    assert float((got - want).abs().max()) <= TOL
    # run again with fewer live rows in the same buffers (device-side count path)
    n2 = 2500
    want2 = osp.middle_encoder_forward(sd, feats[:n2], coors[:n2], batch, input_shape, arch=cls_name)
    n_dev = torch.tensor([n2], dtype=torch.int32, device="cuda")
    got2 = model(torch.from_numpy(feats).cuda(), torch.from_numpy(coors).cuda(), batch, input_shape, n_dev=n_dev).cpu()
    assert float((got2 - want2).abs().max()) <= TOL


def test_unfused_module_path_matches_fused():
    model, feats, coors, input_shape, batch = _encoder_case("SpMiddleFHD", 4, 3000, 5)
    model = model.cuda()
    f, c = torch.from_numpy(feats).cuda(), torch.from_numpy(coors).cuda()
    a = model(f, c, batch, input_shape)
    b = model.forward_unfused(f, c, batch, input_shape)
    assert float((a - b).abs().max()) <= 1e-5


def test_empty_input():
    from det3d_b200.models.backbones.scn import SpMiddleFHD
    model = SpMiddleFHD(num_input_features=4).eval().cuda()
    out = model(torch.zeros((0, 4), device="cuda"), torch.zeros((0, 4), dtype=torch.int32, device="cuda"), 1, [96, 112, 40])
    assert out.shape == (1, 128, 14, 12) and float(out.abs().sum()) == 0.0


def test_dense_matches_oracle():
    from det3d_b200.ops.spconv import SparseConvTensor
    rng = np.random.default_rng(2)
    spatial, batch = (5, 30, 20), 3
    coors = _sites(rng, 700, spatial, batch)
    feat = rng.standard_normal((700, 64)).astype(np.float32)
    t = SparseConvTensor(torch.from_numpy(feat).cuda(), torch.from_numpy(coors).cuda(), spatial, batch)
    assert torch.equal(t.dense().cpu(), osp.dense(feat, coors, spatial, batch))
