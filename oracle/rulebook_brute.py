"""TEST INFRASTRUCTURE -- brute-force rulebook, site-index and scatter reference (CPU, numpy).

Written straight from the definition in the header of csrc/rulebook.cu (spconv v1.x `get_indice_pairs`, dilation 1):
input p feeds output o through kernel offset k = (kz, ky, kx) (row-major, k = (kz*kH + ky)*kW + kx) iff

    p = o * stride - padding + k.

Every structure is a dense occupancy grid of row indices per batch, so the cases it serves must be small enough for a
[B, D, H, W] int64 array.  It deliberately shares no code with oracle/spconv.py (which finds sites by `searchsorted`
over sorted linear indices): the tests hold the two against each other.

Row rules, the same everywhere:
  * only the first `n` rows are live (`n` defaults to every row); rows past it are never read;
  * a live row whose batch index or coordinate lies outside its grid is ignored: it occupies no cell, marks no
    output, is nobody's neighbour, and as an output row of a SubM map it gets -1 for every offset;
  * among live rows that share a cell the lowest row index is the one found.
"""
import numpy as np

TILE_M = 128


def offsets(ksize):
    """[K, 3] (kz, ky, kx) in kernel-offset order."""
    return np.array([(z, y, x) for z in range(ksize[0]) for y in range(ksize[1]) for x in range(ksize[2])],
                    np.int64).reshape(-1, 3)


def conv_out_spatial(spatial, ksize, stride, padding):
    """Output extent per axis: floor((size + 2*padding - ksize) / stride) + 1, the number of o >= 0 whose window
    o*stride - padding + [0, ksize) ends inside the padded input."""
    return tuple((spatial[j] + 2 * padding[j] - ksize[j]) // stride[j] + 1 for j in range(3))


def in_grid(coors, spatial, batch):
    """[n] bool: batch index in [0, batch) and every coordinate in [0, size)."""
    c = np.asarray(coors, np.int64).reshape(-1, 4)
    hi = np.array([batch, *spatial], np.int64)
    return ((c >= 0) & (c < hi)).all(1)


def occupancy(coors, spatial, batch, n=None):
    """[B, D, H, W] int64: the row index that owns each cell, -1 where none does (row rules above)."""
    c = np.asarray(coors, np.int64).reshape(-1, 4)
    n = c.shape[0] if n is None else int(n)
    c = c[:n]
    big = np.iinfo(np.int64).max
    grid = np.full((batch, *spatial), big, np.int64)
    ok = in_grid(c, spatial, batch)
    rows = np.nonzero(ok)[0]
    np.minimum.at(grid, tuple(c[ok].T), rows)
    grid[grid == big] = -1
    return grid


def _lookup(occ, b, zyx):
    """occ[b, z, y, x] where the cell is inside the grid, else -1."""
    bsz, d, h, w = occ.shape
    ok = (b >= 0) & (b < bsz) & ((zyx >= 0) & (zyx < np.array([d, h, w]))).all(1)
    out = np.full(b.shape, -1, np.int64)
    out[ok] = occ[b[ok], zyx[ok, 0], zyx[ok, 1], zyx[ok, 2]]
    return out


def neighbour_map(out_coors, out_spatial, in_occ, ksize, stride, padding, n_out=None):
    """nbr [K, n_out]: nbr[k, o] = row at o*stride - padding + k, or -1.  An output row outside its own grid gets -1
    for every offset."""
    oc = np.asarray(out_coors, np.int64).reshape(-1, 4)
    n_out = oc.shape[0] if n_out is None else int(n_out)
    oc = oc[:n_out]
    live = in_grid(oc, out_spatial, in_occ.shape[0])
    offs = offsets(ksize)
    nbr = np.full((offs.shape[0], n_out), -1, np.int64)
    for k, off in enumerate(offs):
        p = oc[:, 1:] * np.array(stride) - np.array(padding) + off
        nbr[k] = np.where(live, _lookup(in_occ, oc[:, 0], p), -1)
    return nbr


def subm_map(coors, spatial, batch, ksize, n=None, occ=None):
    """SubM rulebook (stride 1, padding k // 2): nbr [K, n] over the same rows.  `occ` (default: the occupancy of
    `coors` itself) is the index the rows are looked up in."""
    if occ is None:
        occ = occupancy(coors, spatial, batch, n)
    return neighbour_map(coors, spatial, occ, ksize, (1, 1, 1), tuple(k // 2 for k in ksize), n)


def conv_outputs(coors, spatial, batch, ksize, stride, padding, n=None):
    """(out_coors [M, 4] int32 in ascending linear index ((b*D+z)*H+y)*W+x, out_spatial): every output cell o of the
    output grid with at least one occupied input cell o*stride - padding + k."""
    occ = occupancy(coors, spatial, batch, n) >= 0
    out_sp = conv_out_spatial(spatial, ksize, stride, padding)
    hit = np.zeros((batch, *out_sp), bool)
    for off in offsets(ksize):
        sel_o, sel_p = [], []
        for j in range(3):
            p = np.arange(out_sp[j]) * stride[j] - padding[j] + off[j]
            ok = (p >= 0) & (p < spatial[j])
            sel_o.append(np.nonzero(ok)[0])
            sel_p.append(p[ok])
        hit[np.ix_(np.arange(batch), *sel_o)] |= occ[np.ix_(np.arange(batch), *sel_p)]
    return np.argwhere(hit).astype(np.int32), out_sp      # argwhere walks C order == ascending linear index


def conv_map(in_coors, in_spatial, batch, out_coors, ksize, stride, padding, n_in=None, n_out=None):
    """Strided rulebook nbr [K, n_out] from the input rows to the given output rows."""
    occ = occupancy(in_coors, in_spatial, batch, n_in)
    out_sp = conv_out_spatial(in_spatial, ksize, stride, padding)
    return neighbour_map(out_coors, out_sp, occ, ksize, stride, padding, n_out)


def tile_masks(nbr, n_tiles=None):
    """[n_tiles] uint32: bit k of tile t set iff some row of t (rows t*128 ... t*128+127) has nbr[k] >= 0."""
    k_vol, n = nbr.shape
    n_tiles = (n + TILE_M - 1) // TILE_M if n_tiles is None else int(n_tiles)
    mask = np.zeros(n_tiles, np.uint32)
    for t in range(min(n_tiles, (n + TILE_M - 1) // TILE_M)):
        used = (nbr[:, t * TILE_M:(t + 1) * TILE_M] >= 0).any(1)
        mask[t] = np.uint32(sum(1 << k for k in range(k_vol) if used[k]))
    return mask


def dense2d_map(batch, height, width, ksize, padding):
    """Rulebook of a dense stride-1 2-D conv over rows (b*H + y)*W + x: nbr [kh*kw, B*H*W], k = ky*kw + kx."""
    kh, kw = ksize
    n = batch * height * width
    nbr = np.full((kh * kw, n), -1, np.int64)
    for row in range(n):
        b, y, x = row // (height * width), (row // width) % height, row % width
        for ky in range(kh):
            for kx in range(kw):
                yy, xx = y + ky - padding[0], x + kx - padding[1]
                if 0 <= yy < height and 0 <= xx < width:
                    nbr[ky * kw + kx, row] = (b * height + yy) * width + xx
    return nbr


def scatter_dense(feat, coors, spatial, batch, out, n=None):
    """rows -> `out` [B, C, D, H, W] (a copy): every occupied cell gets its owner row; nothing else is touched.  The
    device scatters leave the winner among duplicate rows open, so they are held to this on unique cells only."""
    out = np.array(out, copy=True)
    occ = occupancy(coors, spatial, batch, n)
    b, z, y, x = np.nonzero(occ >= 0)
    out[b, :, z, y, x] = np.asarray(feat)[occ[b, z, y, x]]
    return out


def scatter_bev_rows(feat, coors, spatial, batch, out, n=None):
    """rows -> `out` [B*H*W, C*D] (a copy), channel c*D + z; nothing else is touched."""
    d, h, w = spatial
    feat = np.asarray(feat)
    out = np.array(out, copy=True).reshape(batch * h * w, feat.shape[1], d)
    occ = occupancy(coors, spatial, batch, n)
    b, z, y, x = np.nonzero(occ >= 0)
    out[(b * h + y) * w + x, :, z] = feat[occ[b, z, y, x]]
    return out.reshape(batch * h * w, feat.shape[1] * d)


# ---- the level-0 hash's slot function (csrc/common.cuh mix64, the splitmix64 finaliser) ---------------------------------
def mix64(x):
    x = np.asarray(x).astype(np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(30))
        x = x * np.uint64(0xBF58476D1CE4E5B9)
        x = x ^ (x >> np.uint64(27))
        x = x * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return x


def linear_index(coors, spatial):
    c = np.asarray(coors, np.int64).reshape(-1, 4)
    d, h, w = spatial
    return ((c[:, 0] * d + c[:, 1]) * h + c[:, 2]) * w + c[:, 3]


def colliding_cells(spatial, batch, hash_cap, slots):
    """[M, 4] int32: every cell of the grid whose home slot (mix64(linear index) & (hash_cap - 1)) is in `slots`, in
    ascending linear index."""
    lin = np.arange(batch * int(np.prod(spatial)), dtype=np.int64)
    home = (mix64(lin) & np.uint64(hash_cap - 1)).astype(np.int64)
    lin = lin[np.isin(home, np.asarray(slots, np.int64))]
    d, h, w = spatial
    return np.stack([lin // (d * h * w), lin // (h * w) % d, lin // w % h, lin % w], 1).astype(np.int32)
