"""Rulebook, site index, dense 2-D rulebook and BEV scatters, bit for bit against the brute-force reference
(oracle/rulebook_brute.py) across their parameter space: every kernel size 1 .. 5, k_vol 1 .. 32, stride above the
kernel, padding up to k - 1, grids one cell wide, B up to 64, empty inputs, scans of thousands of blocks, capacity
clamps, colliding hash keys, out-of-grid and duplicate rows, and live counts below capacity with poisoned rows past
them.  Each case runs once."""
import ctypes as C

import numpy as np
import pytest
import torch

import rulebook_cases as cases
from oracle import rulebook_brute as brute
from oracle import spconv as osp

pytestmark = pytest.mark.gpu


def _level(rows, spatial, batch, poison, rng):
    """Level-0 hash level over `rows`; with `poison`, rows past the live count hold cells the reference must not see."""
    from det3d_b200.ops.spconv import core
    n = rows.shape[0]
    if poison:
        rows = np.concatenate([rows, cases.poison_rows(n // 4 + 5, spatial, batch, rng)])
    n_dev = torch.tensor([n, n], dtype=torch.int32, device="cuda")
    return core.level_from_coors(torch.from_numpy(np.ascontiguousarray(rows)).cuda(), spatial, batch, n_dev=n_dev)


def _mask(t):
    return t.cpu().numpy().view(np.uint32)


def _check_subm(level, rows, n, spatial, batch, ksize, occ=None):
    from det3d_b200.ops.spconv import core
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(level, ksize))
    want = brute.subm_map(rows, spatial, batch, ksize, n=n, occ=occ)
    assert np.array_equal(rb.nbr[:, :n].cpu().numpy(), want)
    mask = _mask(rb.tile_mask)
    assert np.array_equal(mask, brute.tile_masks(want, mask.shape[0]))
    return rb


def _check_conv(level, rows, n, spatial, batch, ksize, stride, padding, out_cap=None):
    """Strided build vs the reference: output grid, [rows kept, rows found], coordinates, map and tile masks.  Returns
    the rulebook and the output coordinates it keeps."""
    from det3d_b200.ops.spconv import core
    rb = core.build_conv_rulebook(core.alloc_conv_rulebook(level, ksize, stride, padding, out_cap))
    want, want_sp = brute.conv_outputs(rows, spatial, batch, ksize, stride, padding, n=n)
    m = min(want.shape[0], rb.out_level.cap)
    assert rb.out_level.spatial == tuple(want_sp)
    assert rb.out_level.n.cpu().tolist() == [m, want.shape[0]]
    assert np.array_equal(rb.out_level.coors[:m].cpu().numpy(), want[:m])
    nbr = brute.conv_map(rows, spatial, batch, want[:m], ksize, stride, padding, n_in=n)
    assert np.array_equal(rb.nbr[:, :m].cpu().numpy(), nbr)
    mask = _mask(rb.tile_mask)
    assert np.array_equal(mask, brute.tile_masks(nbr, mask.shape[0]))
    return rb, want[:m]


@pytest.mark.parametrize("poison", [False, True], ids=["all-live", "poisoned-tail"])
@pytest.mark.parametrize("density", cases.DENSITIES)
@pytest.mark.parametrize("ksize,stride,padding,spatial,batch", cases.strided_params())
def test_strided_rulebook(ksize, stride, padding, spatial, batch, density, poison):
    rng = np.random.default_rng(11)
    rows = cases.sites(density, spatial, batch, rng)
    lvl = _level(rows, spatial, batch, poison, rng)
    rb, out = _check_conv(lvl, rows, rows.shape[0], spatial, batch, ksize, stride, padding)
    # the next level's SubM rulebook reads the bitmap index the strided build left
    _check_subm(rb.out_level, out, out.shape[0], rb.out_level.spatial, batch, (3, 3, 3))


@pytest.mark.parametrize("poison", [False, True], ids=["all-live", "poisoned-tail"])
@pytest.mark.parametrize("density", cases.DENSITIES)
@pytest.mark.parametrize("spatial,batch", cases.GRIDS)
@pytest.mark.parametrize("ksize", cases.SUBM)
def test_subm_rulebook(ksize, spatial, batch, density, poison):
    rng = np.random.default_rng(12)
    rows = cases.sites(density, spatial, batch, rng)
    _check_subm(_level(rows, spatial, batch, poison, rng), rows, rows.shape[0], spatial, batch, ksize)


def test_empty_input():
    rng = np.random.default_rng(13)
    spatial, batch = (9, 10, 11), 3
    rows = np.zeros((0, 4), np.int32)
    lvl = _level(rows, spatial, batch, True, rng)
    _check_subm(lvl, rows, 0, spatial, batch, (3, 3, 3))
    rb, out = _check_conv(lvl, rows, 0, spatial, batch, (3, 3, 3), (2, 2, 2), (1, 1, 1))
    assert out.shape == (0, 4)
    _check_subm(rb.out_level, out, 0, rb.out_level.spatial, batch, (3, 3, 3))


@pytest.mark.parametrize("clamp", [False, True], ids=["fits", "clamped"])
@pytest.mark.parametrize("n_words", [4095, 4096, 4097, 8191, 8192, 8193])
def test_scan_word_counts(n_words, clamp):
    """Bitmaps of 4096*k - 1, 4096*k and 4096*k + 1 words: a scan block holds 4096 words, so the last block is one word
    short of full, exactly full, or holds a single word."""
    rng = np.random.default_rng(n_words)
    spatial, batch = (n_words, 1, 32), 1
    lin = rng.permutation(n_words * 32)[: n_words * 3]
    lin[0] = n_words * 32 - 1                                 # the scan's very last bit
    rows = cases.cells_to_coors(lin, spatial)
    lvl = _level(rows, spatial, batch, True, rng)
    total = brute.conv_outputs(rows, spatial, batch, (3, 1, 1), (1, 1, 1), (1, 0, 0))[0].shape[0]
    rb, out = _check_conv(lvl, rows, rows.shape[0], spatial, batch, (3, 1, 1), (1, 1, 1), (1, 0, 0),
                          out_cap=total - 37 if clamp else None)
    _check_subm(rb.out_level, out, out.shape[0], spatial, batch, (3, 1, 1))


@pytest.mark.parametrize("clamp", [False, True], ids=["fits", "clamped"])
def test_scan_thousands_of_blocks(clamp):
    """B = 8 over a 41 x 1600 x 1408 grid: 23.1 M bitmap words, 5638 scan blocks, sparse sites.  Too large for the
    reference's dense grids, so the expected rulebook of this 1x1x1 stride-1 conv is written from its definition:
    the outputs are the occupied cells in ascending linear index, each fed by its own row."""
    from det3d_b200.ops.spconv import core
    rng = np.random.default_rng(14)
    spatial, batch = (41, 1600, 1408), 8
    cells = batch * 41 * 1600 * 1408
    lin = np.unique(np.concatenate([rng.integers(0, cells, 160000), [0, cells - 1]]))
    rows = cases.cells_to_coors(rng.permutation(lin), spatial)
    order = np.argsort(brute.linear_index(rows, spatial), kind="stable")
    out_cap = lin.size - 1000 if clamp else None
    lvl = core.level_from_coors(torch.from_numpy(rows).cuda(), spatial, batch)
    rb = core.build_conv_rulebook(core.alloc_conv_rulebook(lvl, 1, 1, 0, out_cap))
    assert rb.out_level.index.n_words == cells // 32
    m = rb.out_level.cap
    assert rb.out_level.n.cpu().tolist() == [m, lin.size]
    assert np.array_equal(rb.out_level.coors[:m].cpu().numpy(), rows[order[:m]])
    assert np.array_equal(rb.nbr[0, :m].cpu().numpy(), order[:m])
    assert np.array_equal(_mask(rb.tile_mask), np.ones(rb.tile_mask.numel(), np.uint32))


@pytest.mark.parametrize("poison", [False, True], ids=["all-live", "poisoned-tail"])
@pytest.mark.parametrize("ksize,stride,padding", [((3, 3, 3), (2, 2, 2), (1, 1, 1)), ((1, 4, 8), (1, 2, 4), (0, 1, 3))])
def test_overflow_clamp(ksize, stride, padding, poison):
    """out_cap below the true count: the first out_cap outputs, the true count in n_out[1], and a SubM rulebook on the
    clamped level that never returns a rank >= out_cap although the bitmap still holds every output."""
    rng = np.random.default_rng(15)
    spatial, batch = (9, 30, 30), 2
    rows = cases.sites("random", spatial, batch, rng)[:900]
    lvl = _level(rows, spatial, batch, poison, rng)
    total = brute.conv_outputs(rows, spatial, batch, ksize, stride, padding)[0].shape[0]
    cap = total // 2 + 3
    rb, out = _check_conv(lvl, rows, rows.shape[0], spatial, batch, ksize, stride, padding, out_cap=cap)
    assert out.shape[0] == cap < total
    sub = _check_subm(rb.out_level, out, cap, rb.out_level.spatial, batch, (3, 3, 3))
    assert int(sub.nbr[:, :cap].max()) < cap


def _lookup(level, query, ksize):
    """SubM rulebook of the `query` rows looked up in `level`'s index (the C ABI takes them separately)."""
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import core
    q = torch.from_numpy(np.ascontiguousarray(query)).cuda()
    n = torch.tensor([q.shape[0]] * 2, dtype=torch.int32, device="cuda")
    k_vol = int(np.prod(ksize))
    nbr = torch.empty((k_vol, q.shape[0]), dtype=torch.int32, device="cuda")
    mask = torch.empty((q.shape[0] + 127) // 128, dtype=torch.int32, device="cuda")
    st = _lib.lib().d3b_rulebook_subm(q.data_ptr(), n.data_ptr(), q.shape[0], C.byref(level.index), core._i3(ksize),
                                      nbr.data_ptr(), mask.data_ptr(), _lib.current_stream())
    _lib.check(st, "d3b_rulebook_subm")
    return nbr.cpu().numpy(), _mask(mask)


def test_hash_collisions_at_half_load():
    """512 rows in a 1024-slot table (load 0.5), every key's home slot in 1020 .. 1023 or 0 .. 3: one probe run of
    512 slots that wraps around the table's end.  Every lookup -- the present keys, absent cells with the same home
    slots, and the 27 neighbours of each row -- matches the reference."""
    spatial, batch = (16, 64, 64), 2
    slots = [1020, 1021, 1022, 1023, 0, 1, 2, 3]
    coll = brute.colliding_cells(spatial, batch, 1024, slots)
    assert coll.shape[0] >= 900
    rng = np.random.default_rng(16)
    coll = coll[rng.permutation(coll.shape[0])]
    rows, absent = coll[:512], coll[512:]
    lvl = _level(rows, spatial, batch, False, rng)
    assert lvl.index.hash_cap == 1024 and lvl.cap == 512
    occ = brute.occupancy(rows, spatial, batch)
    query = np.concatenate([absent, rows, cases.sites("random", spatial, batch, rng)[:2000]])
    got, _ = _lookup(lvl, query, (1, 1, 1))
    want = brute.subm_map(query, spatial, batch, (1, 1, 1), occ=occ)
    assert np.array_equal(got, want)
    assert (want[0, :absent.shape[0]] == -1).all() and np.array_equal(want[0, absent.shape[0]:][:512], np.arange(512))
    got, mask = _lookup(lvl, rows, (3, 3, 3))
    want = brute.subm_map(rows, spatial, batch, (3, 3, 3), occ=occ)
    assert np.array_equal(got, want) and np.array_equal(mask, brute.tile_masks(want))


RULE_GRIDS = [((41, 8, 8), 2), ((2, 3, 33), 3), ((3, 4, 1), 5), ((1, 1, 5), 64)]


@pytest.mark.parametrize("poison", [False, True], ids=["all-live", "poisoned-tail"])
@pytest.mark.parametrize("spatial,batch", RULE_GRIDS)
@pytest.mark.parametrize("dups", [False, True], ids=["out-of-grid", "out-of-grid+duplicates"])
@pytest.mark.parametrize("path", ["subm", "strided"])
def test_out_of_grid_and_duplicate_rows(path, dups, spatial, batch, poison):
    """Rows with each coordinate at -1 and at its size and the batch at -1 and at B, and (with `dups`) duplicates
    before and after their originals: no out-of-grid row creates an output, is a neighbour or gets one; duplicates
    resolve to the lowest row.  Through SubM, or through strided builds and the SubM level above them."""
    rng = np.random.default_rng(17)
    rows = cases.with_rule_rows(cases.sites("random", spatial, batch, rng), spatial, batch, rng,
                                n_dup=None if dups else 0)
    lvl = _level(rows, spatial, batch, poison, rng)
    n = rows.shape[0]
    if path == "subm":
        for ksize in [(3, 3, 3), (1, 3, 3), (1, 1, 1)]:
            rb = _check_subm(lvl, rows, n, spatial, batch, ksize)
            assert (rb.nbr[:, :n].cpu().numpy()[:, ~brute.in_grid(rows, spatial, batch)] == -1).all()
        return
    for ksize, stride, padding in [((3, 3, 3), (2, 2, 2), (1, 1, 1)), ((3, 3, 3), (2, 2, 2), (0, 1, 1)),
                                   ((1, 1, 2), (1, 1, 2), (0, 0, 1)), ((2, 2, 2), (3, 3, 4), (0, 1, 1))]:
        if cases.valid(spatial, ksize, padding):
            rb, out = _check_conv(lvl, rows, n, spatial, batch, ksize, stride, padding)
            _check_subm(rb.out_level, out, out.shape[0], rb.out_level.spatial, batch, (3, 3, 3))


def test_duplicate_rows_are_deterministic():
    """Every site eight times at random positions: 20 builds give the same map bit for bit, the reference's lowest
    row."""
    from det3d_b200.ops.spconv import core
    rng = np.random.default_rng(18)
    spatial, batch = (11, 40, 36), 2
    sites = cases.sites("random", spatial, batch, rng)[:3000]
    rows = np.tile(sites, (8, 1))[rng.permutation(sites.shape[0] * 8)]
    n = rows.shape[0]
    want_subm = brute.subm_map(rows, spatial, batch, (3, 3, 3))
    want_out, _ = brute.conv_outputs(rows, spatial, batch, (3, 3, 3), (2, 2, 2), (1, 1, 1))
    want_conv = brute.conv_map(rows, spatial, batch, want_out, (3, 3, 3), (2, 2, 2), (1, 1, 1))
    lvl = _level(rows, spatial, batch, False, rng)
    subm = core.alloc_subm_rulebook(lvl, 3)
    conv = core.alloc_conv_rulebook(lvl, 3, 2, 1)
    m = want_out.shape[0]
    for _ in range(20):
        lvl.rebuild_index()
        core.build_subm_rulebook(subm)
        core.build_conv_rulebook(conv)
        assert np.array_equal(subm.nbr[:, :n].cpu().numpy(), want_subm)
        assert np.array_equal(conv.out_level.coors[:m].cpu().numpy(), want_out)
        assert np.array_equal(conv.nbr[:, :m].cpu().numpy(), want_conv)


@pytest.mark.parametrize("ksize", [(1, 1), (3, 3), (1, 3), (5, 5)])
@pytest.mark.parametrize("batch,height,width", [(1, 127, 1), (2, 8, 8), (3, 43, 1), (2, 5, 13)])
def test_dense2d_rulebook(ksize, batch, height, width):
    """B*H*W of 127, 128, 129 and 130 rows.  Every tile's mask has every offset of the kernel: the map holds -1 at the
    borders, which the convolution reads as zero padding."""
    from det3d_b200 import _lib
    n, k_vol = batch * height * width, ksize[0] * ksize[1]
    pad = (ksize[0] // 2, ksize[1] // 2)
    nbr = torch.full((k_vol * n + 64,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    tiles = (n + 127) // 128
    mask = torch.full((tiles + 4,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    n_rows = torch.full((4,), -7, dtype=torch.int32, device="cuda")
    st = _lib.lib().d3b_rulebook_dense2d(batch, height, width, (C.c_int32 * 2)(*ksize), (C.c_int32 * 2)(*pad),
                                         nbr.data_ptr(), mask.data_ptr(), n_rows.data_ptr(), _lib.current_stream())
    _lib.check(st, "d3b_rulebook_dense2d")
    want = brute.dense2d_map(batch, height, width, ksize, pad)
    got = nbr.cpu().numpy()
    assert np.array_equal(got[:k_vol * n].reshape(k_vol, n), want)
    assert (got[k_vol * n:] == 0x5A5A5A5A).all()
    full = (1 << k_vol) - 1
    m = _mask(mask)
    assert (m[:tiles] == full).all() and (m[tiles:] == 0x5A5A5A5A).all()
    assert not (brute.tile_masks(want) & ~np.uint32(full)).any()
    assert n_rows.cpu().tolist() == [n, n, -7, -7]


SCATTERS = ["dense", "bev_rows", "bev16_f32", "bev16_f32_one_plane", "bev16_planes"]


@pytest.mark.parametrize("poison", [False, True], ids=["all-live", "poisoned-tail"])
@pytest.mark.parametrize("channels", [1, 3, 64, 256])
@pytest.mark.parametrize("kind", SCATTERS)
def test_scatter(kind, channels, poison):
    """Each scatter writes exactly the in-grid live rows and leaves every other element of a NaN-filled output as it
    was; an out-of-grid row or a row past the live count with a value outside the f16 range raises no overflow."""
    from det3d_b200.ops.spconv import conv16, core
    rng = np.random.default_rng(channels)
    spatial, batch = (3, 5, 33), 2
    d, h, w = spatial
    rows = np.concatenate([cases.sites("random", spatial, batch, rng), cases.out_of_grid_rows(spatial, batch)])
    rows = rows[rng.permutation(rows.shape[0])]
    n = rows.shape[0]
    feat = rng.standard_normal((n, channels)).astype(np.float32)
    feat[~brute.in_grid(rows, spatial, batch)] = 1e6
    if poison:
        rows = np.concatenate([rows, cases.poison_rows(11, spatial, batch, rng)])
        feat = np.concatenate([feat, np.full((11, channels), 1e6, np.float32)])
    level = core.SparseLevel(torch.from_numpy(rows).cuda(), torch.tensor([n, n], dtype=torch.int32, device="cuda"),
                             rows.shape[0], spatial, batch)
    x = torch.from_numpy(feat).cuda()
    if kind == "dense":
        out = torch.full((batch, channels, d, h, w), float("nan"), device="cuda")
        core.sparse_to_dense(x, level, out)
        want = brute.scatter_dense(feat, rows, spatial, batch, np.full(out.shape, np.nan, np.float32), n=n)
        assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32))
        return
    if kind == "bev_rows":
        out = torch.full((batch * h * w, channels * d), float("nan"), device="cuda")
        core.sparse_to_bev_rows(x, level, out)
        want = brute.scatter_bev_rows(feat, rows, spatial, batch, np.full(out.shape, np.nan, np.float32), n=n)
        assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32))
        return
    n_planes = 1 if kind == "bev16_f32_one_plane" else 2
    hi = feat.astype(np.float16)
    lo = (feat - hi.astype(np.float32)).astype(np.float16)
    src = x
    if kind == "bev16_planes":
        src = conv16.Planes((rows.shape[0], channels), "cuda")
        src.buf.copy_(torch.from_numpy(np.stack([hi, lo])))
    out = conv16.Planes((batch, h, w, channels * d), "cuda", n_planes=n_planes)
    out.buf.fill_(float("nan"))
    overflow = torch.zeros(1, dtype=torch.int32, device="cuda")
    before = out.buf.cpu().numpy()
    conv16.sparse_to_bev16(src, level, out, overflow=overflow)
    got = out.buf.cpu().numpy()
    for p, plane in enumerate([hi, lo][:n_planes]):
        want = brute.scatter_bev_rows(plane, rows, spatial, batch, before[p].reshape(batch * h * w, -1), n=n)
        assert np.array_equal(got[p].reshape(batch * h * w, -1).view(np.uint16), want.view(np.uint16))
    assert int(overflow) == 0


def test_module_stack_with_duplicate_and_out_of_grid_rows():
    """SparseConvTensor -> SparseConv3d(k=2, s=2) -> SubMConv3d(k=(1,3,3)) on fp32 features, sites with duplicates and
    out-of-grid rows, against oracle.spconv.indice_conv on the reference's maps."""
    from det3d_b200.ops.spconv import SparseConv3d, SparseConvTensor, SubMConv3d
    torch.manual_seed(19)
    rng = np.random.default_rng(19)
    spatial, batch = (9, 22, 26), 2
    rows = cases.with_rule_rows(cases.sites("random", spatial, batch, rng)[:1200], spatial, batch, rng)
    feat = rng.standard_normal((rows.shape[0], 16)).astype(np.float32)
    conv = SparseConv3d(16, 32, 2, stride=2).cuda()
    subm = SubMConv3d(32, 32, (1, 3, 3)).cuda()
    t = SparseConvTensor(torch.from_numpy(feat).cuda(), torch.from_numpy(rows).cuda(), spatial, batch)
    t1 = conv(t)
    t2 = subm(t1)
    out, out_sp = brute.conv_outputs(rows, spatial, batch, (2, 2, 2), (2, 2, 2), (0, 0, 0))
    assert np.array_equal(t2.indices.cpu().numpy(), out) and list(out_sp) == t2.spatial_shape
    nbr1 = brute.conv_map(rows, spatial, batch, out, (2, 2, 2), (2, 2, 2), (0, 0, 0))
    f1 = osp.indice_conv(feat, conv.weight.detach().cpu(), nbr1, out.shape[0], conv.bias.detach().cpu())
    nbr2 = brute.subm_map(out, out_sp, batch, (1, 3, 3))
    f2 = osp.indice_conv(f1, subm.weight.detach().cpu(), nbr2, out.shape[0], subm.bias.detach().cpu())
    got = t2.features.cpu()
    assert torch.isfinite(got).all()
    assert float((got - f2).abs().max()) <= 1e-4
