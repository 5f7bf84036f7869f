"""Rulebook edge cases shared by the brute-force reference's CPU test and the device tests: kernel / stride / padding
geometries, small grids and site layouts (no pytest hooks here)."""
import numpy as np

# (ksize, stride, padding) of the strided build: k_vol 1 .. 32 (exactly 32 reaches tile-mask bit 31), every kernel
# size 1 .. 5, strides 1 .. 4 including stride > kernel, padding 0 .. k - 1 including the deployed [0, 1, 1].
STRIDED = [
    ((1, 1, 1), (1, 1, 1), (0, 0, 0)),
    ((1, 1, 2), (1, 1, 2), (0, 0, 1)),
    ((3, 3, 3), (2, 2, 2), (1, 1, 1)),
    ((3, 3, 3), (2, 2, 2), (0, 1, 1)),
    ((3, 1, 1), (2, 1, 1), (0, 0, 0)),
    ((2, 2, 2), (2, 2, 2), (0, 0, 0)),
    ((1, 4, 8), (1, 2, 4), (0, 1, 3)),
    ((2, 4, 4), (2, 3, 2), (1, 3, 0)),
    ((2, 2, 2), (3, 3, 4), (0, 1, 1)),
    ((1, 1, 1), (4, 3, 2), (0, 0, 0)),
    ((5, 1, 5), (1, 4, 2), (4, 0, 2)),
    ((4, 2, 4), (3, 1, 4), (3, 1, 2)),
    ((3, 5, 2), (4, 1, 3), (2, 4, 1)),
]

# SubM kernels: every odd size with k_vol <= 32.
SUBM = [(1, 1, 1), (3, 1, 1), (1, 3, 3), (3, 3, 3), (1, 5, 5), (1, 1, 31)]

# (spatial (D, H, W), batch): W in {1, 2, 3, 31, 32, 33}, D and H equal to 1, B up to 64, and D*H*W mostly not a
# multiple of 32 so batches change inside one 32-cell bitmap word.
GRIDS = [
    ((3, 4, 1), 5),
    ((2, 3, 2), 3),
    ((5, 1, 3), 4),
    ((1, 7, 31), 2),
    ((3, 2, 32), 3),
    ((2, 3, 33), 2),
    ((1, 1, 5), 64),
    ((4, 6, 7), 1),
]

DENSITIES = ["one", "full", "last", "random"]


def valid(spatial, ksize, padding):
    """The strided geometry has an output cell along every axis (the padded input is at least the kernel)."""
    return all(spatial[j] + 2 * padding[j] >= ksize[j] for j in range(3))


def strided_params():
    """pytest params (ksize, stride, padding, spatial, batch): every strided geometry on every grid it fits."""
    import pytest
    return [pytest.param(k, s, p, sp, b, id="k%s-s%s-p%s-g%s-b%d" % (k, s, p, sp, b))
            for (k, s, p) in STRIDED for (sp, b) in GRIDS if valid(sp, k, p)]


def cells_to_coors(lin, spatial):
    d, h, w = spatial
    lin = np.asarray(lin, np.int64)
    return np.stack([lin // (d * h * w), lin // (h * w) % d, lin // w % h, lin % w], 1).astype(np.int32)


def sites(density, spatial, batch, rng):
    """[n, 4] int32 unique in-grid sites (b, z, y, x) in random row order."""
    d, h, w = spatial
    cells = batch * d * h * w
    if density == "one":
        lin = rng.integers(0, cells, 1)
    elif density == "full":
        lin = rng.permutation(cells)
    elif density == "last":
        lin = rng.permutation(np.arange(batch) * (d * h * w) + d * h * w - 1)
    else:
        lin = rng.permutation(cells)[: max(1, int(0.35 * cells))]
    return cells_to_coors(lin, spatial)


def out_of_grid_rows(spatial, batch):
    """One row per way of leaving the grid: each coordinate at -1 and at its size, the batch at -1 and at B; the
    other coordinates are in the grid."""
    d, h, w = spatial
    base = [0, d // 2, h // 2, w // 2]
    rows = []
    for j, size in enumerate([batch, d, h, w]):
        for v in (-1, size):
            r = list(base)
            r[j] = v
            rows.append(r)
    return np.array(rows, np.int32)


def with_rule_rows(coors, spatial, batch, rng, n_dup=None):
    """`coors` with every out-of-grid row and duplicates of some of its sites mixed in at random positions (so a
    duplicate can come before or after its original)."""
    n = coors.shape[0]
    n_dup = max(1, n // 3) if n_dup is None else n_dup
    dup = coors[rng.integers(0, n, n_dup)]
    rows = np.concatenate([coors, dup, out_of_grid_rows(spatial, batch)], 0)
    return rows[rng.permutation(rows.shape[0])]


def poison_rows(n, spatial, batch, rng):
    """Rows to place past the live count: random in-grid cells alternating with out-of-grid and huge coordinates, so
    a kernel that read one would mark an output or find a neighbour the reference does not have."""
    d, h, w = spatial
    big = np.iinfo(np.int32).max
    pool = np.array([[batch, d, h, w], [-1, -1, -1, -1], [big, big, big, big], [0, big, 0, 0],
                     [0, 0, 0, -big - 1], [batch - 1, d - 1, h - 1, w]], np.int32)
    rows = pool[np.arange(n) % pool.shape[0]]
    rows[::2] = cells_to_coors(rng.integers(0, batch * d * h * w, (n + 1) // 2), spatial)
    return rows
