"""The brute-force rulebook reference (oracle/rulebook_brute.py) against two independently built ones: oracle/spconv.py
(sorted linear indices + searchsorted) and dense torch conv3d of one-hot features, which tells which kernel offset
carried which input row to which output cell.  CPU only."""
import numpy as np
import pytest
import torch

from oracle import rulebook_brute as rb
from oracle import spconv as osp
import rulebook_cases as cases


@pytest.mark.parametrize("density", cases.DENSITIES)
@pytest.mark.parametrize("ksize,stride,padding,spatial,batch", cases.strided_params())
def test_strided_matches_spconv_oracle(ksize, stride, padding, spatial, batch, density):
    coors = cases.sites(density, spatial, batch, np.random.default_rng(7))
    out, out_sp = rb.conv_outputs(coors, spatial, batch, ksize, stride, padding)
    want, want_sp = osp.conv_outputs(coors, spatial, ksize, stride, padding)
    assert tuple(out_sp) == tuple(want_sp)
    assert np.array_equal(out, want)
    assert np.array_equal(rb.conv_map(coors, spatial, batch, out, ksize, stride, padding),
                          osp.conv_neighbours(coors, spatial, want, ksize, stride, padding))


@pytest.mark.parametrize("density", cases.DENSITIES)
@pytest.mark.parametrize("spatial,batch", cases.GRIDS)
@pytest.mark.parametrize("ksize", cases.SUBM)
def test_subm_matches_spconv_oracle(ksize, spatial, batch, density):
    coors = cases.sites(density, spatial, batch, np.random.default_rng(8))
    assert np.array_equal(rb.subm_map(coors, spatial, batch, ksize), osp.subm_neighbours(coors, spatial, ksize))


def _one_hot_conv(coors, spatial, batch, ksize, stride, padding):
    """Dense conv3d whose output channel i*K + k is 1 exactly where input row i reaches through offset k."""
    n, kv = coors.shape[0], int(np.prod(ksize))
    x = torch.zeros((batch, n, *spatial), dtype=torch.float64)
    c = torch.from_numpy(coors.astype(np.int64))
    x[c[:, 0], torch.arange(n), c[:, 1], c[:, 2], c[:, 3]] = 1.0
    w = torch.zeros((n * kv, n, *ksize), dtype=torch.float64)
    for k, (kz, ky, kx) in enumerate(rb.offsets(ksize)):
        w[torch.arange(n) * kv + k, torch.arange(n), kz, ky, kx] = 1.0
    y = torch.nn.functional.conv3d(x, w, stride=stride, padding=padding)
    return y.reshape(batch, n, kv, *y.shape[2:]).numpy()


def _nbr_from_one_hot(y, out_coors):
    b, z, yy, x = out_coors.astype(np.int64).T
    hits = y[b, :, :, z, yy, x]                          # [M, n, K]
    assert set(np.unique(hits)) <= {0.0, 1.0}
    assert (hits.sum(1) <= 1).all()                      # unique sites: at most one row per (output, offset)
    row = np.where(hits.any(1), hits.argmax(1), -1)      # [M, K]
    return row.T


SMALL = [((2, 3, 5), 2, 9), ((1, 4, 6), 3, 12), ((3, 3, 3), 1, 27), ((4, 1, 7), 2, 20)]


@pytest.mark.parametrize("ksize,stride,padding", cases.STRIDED)
@pytest.mark.parametrize("spatial,batch,n", SMALL)
def test_strided_matches_one_hot_conv3d(ksize, stride, padding, spatial, batch, n):
    if not cases.valid(spatial, ksize, padding):
        pytest.skip("kernel wider than the padded input")
    rng = np.random.default_rng(n)
    coors = cases.cells_to_coors(rng.permutation(batch * int(np.prod(spatial)))[:n], spatial)
    y = _one_hot_conv(coors, spatial, batch, ksize, stride, padding)
    out, out_sp = rb.conv_outputs(coors, spatial, batch, ksize, stride, padding)
    assert tuple(out_sp) == y.shape[3:]
    assert np.array_equal(out, np.argwhere(y.any(axis=(1, 2))))
    assert np.array_equal(rb.conv_map(coors, spatial, batch, out, ksize, stride, padding), _nbr_from_one_hot(y, out))


@pytest.mark.parametrize("ksize", cases.SUBM)
@pytest.mark.parametrize("spatial,batch,n", SMALL)
def test_subm_matches_one_hot_conv3d(ksize, spatial, batch, n):
    rng = np.random.default_rng(n + 1)
    coors = cases.cells_to_coors(rng.permutation(batch * int(np.prod(spatial)))[:n], spatial)
    y = _one_hot_conv(coors, spatial, batch, ksize, (1, 1, 1), tuple(k // 2 for k in ksize))
    assert np.array_equal(rb.subm_map(coors, spatial, batch, ksize), _nbr_from_one_hot(y, coors))


def _clean(rows, spatial, batch):
    """(unique in-grid coordinates, their row index in `rows`): each cell's lowest row, out-of-grid rows dropped."""
    ok = np.nonzero(rb.in_grid(rows, spatial, batch))[0]
    lin = rb.linear_index(rows[ok], spatial)
    _, first = np.unique(lin, return_index=True)        # first occurrence == lowest row (ok is ascending)
    keep = np.sort(ok[first])
    return rows[keep], keep


@pytest.mark.parametrize("spatial,batch", cases.GRIDS)
def test_row_rules_reduce_to_the_clean_rows(spatial, batch):
    """Out-of-grid rows change nothing and duplicates resolve to their lowest row: every map over the mixed rows is
    the map over the clean rows, renumbered."""
    rng = np.random.default_rng(batch)
    rows = cases.with_rule_rows(cases.sites("random", spatial, batch, rng), spatial, batch, rng)
    clean, keep = _clean(rows, spatial, batch)
    renum = lambda nbr: np.where(nbr >= 0, keep[np.maximum(nbr, 0)], -1)
    for ksize in cases.SUBM:
        got = rb.subm_map(rows, spatial, batch, ksize)
        ok = rb.in_grid(rows, spatial, batch)
        assert (got[:, ~ok] == -1).all()
        lin = rb.linear_index(rows, spatial)
        pos = {int(l): j for j, l in enumerate(rb.linear_index(clean, spatial))}
        for i in np.nonzero(ok)[0]:                       # every in-grid row, duplicate or not, sees its cell's map
            assert np.array_equal(got[:, i], renum(rb.subm_map(clean, spatial, batch, ksize))[:, pos[int(lin[i])]])
    for ksize, stride, padding in cases.STRIDED:
        if not cases.valid(spatial, ksize, padding):
            continue
        out, _ = rb.conv_outputs(rows, spatial, batch, ksize, stride, padding)
        want, _ = rb.conv_outputs(clean, spatial, batch, ksize, stride, padding)
        assert np.array_equal(out, want)
        assert np.array_equal(rb.conv_map(rows, spatial, batch, out, ksize, stride, padding),
                              renum(rb.conv_map(clean, spatial, batch, want, ksize, stride, padding)))


def test_out_of_grid_rows_mark_nothing():
    """The worked case of a 41-deep grid, k = 3, s = 2, p = 1: rows at z = -1 and z = 41 would reach output z 0 and 20
    by the offset arithmetic alone."""
    spatial = (41, 4, 4)
    rows = np.array([[0, -1, 1, 1], [0, 41, 2, 2]], np.int32)
    out, out_sp = rb.conv_outputs(rows, spatial, 1, (3, 3, 3), (2, 2, 2), (1, 1, 1))
    assert out_sp == (21, 2, 2) and out.shape == (0, 4)
    assert (rb.subm_map(rows, spatial, 1, (3, 3, 3)) == -1).all()


def test_live_count_hides_later_rows():
    spatial, batch = (3, 4, 5), 2
    rng = np.random.default_rng(3)
    coors = cases.sites("random", spatial, batch, rng)
    rows = np.concatenate([coors, cases.poison_rows(9, spatial, batch, rng)])
    n = coors.shape[0]
    assert np.array_equal(rb.subm_map(rows, spatial, batch, (3, 3, 3), n=n), rb.subm_map(coors, spatial, batch, (3, 3, 3)))
    assert np.array_equal(rb.conv_outputs(rows, spatial, batch, (3, 3, 3), (2, 2, 2), (1, 1, 1), n=n)[0],
                          rb.conv_outputs(coors, spatial, batch, (3, 3, 3), (2, 2, 2), (1, 1, 1))[0])
    assert np.array_equal(rb.occupancy(np.zeros((0, 4), np.int32), spatial, batch), np.full((batch, *spatial), -1))


def test_tile_masks():
    nbr = np.full((32, 300), -1, np.int64)
    nbr[31, 127] = 5          # bit 31 in tile 0
    nbr[0, 128] = 1           # bit 0 in tile 1
    nbr[7, 299] = 2           # bit 7 in tile 2
    assert rb.tile_masks(nbr).tolist() == [1 << 31, 1, 1 << 7]
    assert rb.tile_masks(nbr, 5).tolist() == [1 << 31, 1, 1 << 7, 0, 0]


@pytest.mark.parametrize("ksize", [(1, 1), (3, 3), (1, 3), (5, 5)])
@pytest.mark.parametrize("batch,height,width", [(1, 127, 1), (2, 8, 8), (3, 43, 1), (2, 5, 13)])
def test_dense2d_is_the_subm_map_of_a_full_grid(ksize, batch, height, width):
    spatial = (1, height, width)
    full = cases.cells_to_coors(np.arange(batch * height * width), spatial)
    want = rb.neighbour_map(full, spatial, rb.occupancy(full, spatial, batch), (1, *ksize), (1, 1, 1),
                            (0, ksize[0] // 2, ksize[1] // 2))
    assert np.array_equal(rb.dense2d_map(batch, height, width, ksize, (ksize[0] // 2, ksize[1] // 2)), want)


@pytest.mark.parametrize("channels", [1, 3, 64])
def test_scatters_match_spconv_dense(channels):
    spatial, batch = (3, 5, 7), 2
    rng = np.random.default_rng(channels)
    coors = cases.sites("random", spatial, batch, rng)
    feat = rng.standard_normal((coors.shape[0], channels)).astype(np.float32)
    dense = rb.scatter_dense(feat, coors, spatial, batch, np.zeros((batch, channels, *spatial), np.float32))
    assert np.array_equal(dense, osp.dense(feat, coors, spatial, batch).numpy())
    rows = rb.scatter_bev_rows(feat, coors, spatial, batch, np.zeros((batch * 35, channels * 3), np.float32))
    assert np.array_equal(rows, dense.reshape(batch, channels * 3, 5, 7).transpose(0, 2, 3, 1).reshape(batch * 35, -1))


def test_mix64_is_the_splitmix64_finaliser():
    # splitmix64's first output from state 0 is mix64(0x9E3779B97F4A7C15)
    assert int(rb.mix64(0x9E3779B97F4A7C15)) == 0xE220A8397B1DCDAF
    cells = rb.colliding_cells((5, 16, 16), 2, 1024, [1022, 1023, 0, 1])
    assert cells.shape[0] > 0
    home = rb.mix64(rb.linear_index(cells, (5, 16, 16))) & np.uint64(1023)
    assert set(int(h) for h in home) <= {1022, 1023, 0, 1}
