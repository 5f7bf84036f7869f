"""The PointPillars reader's forward-error model (`csrc/pillars.cu`: `d3b_pillar_features` and `_lists`), a float64
restatement of the operation that can be mutated rule by rule, and the synthetic inputs the GPU sweep and the CPU
sensitivity test share.  A helper module, not a test file: `tests/test_pillar_reader_error_model_gpu.py` runs the
kernels against `error_bound`, `tests/test_pillar_error_model.py` shows that the bound and the data catch every rule."""
import numpy as np
import torch

U = 2.0 ** -24            # fp32 unit roundoff (round to nearest)
U64 = 2.0 ** -53          # float64 unit roundoff: the reference's own rounding
EPS = 1e-3                # BatchNorm1d eps of every PointPillars config
SENTINEL = 0x7F000000     # csrc/voxelize.cu: point-list slots at or above this value are empty

KITTI = dict(vs=(0.2, 0.2, 4.0), pcr=(0.0, -40.0, -3.0, 70.4, 40.0, 1.0))          # x up to 70.4 m
NUSC = dict(vs=(0.2, 0.2, 8.0), pcr=(-51.2, -51.2, -5.0, 51.2, 51.2, 3.0))        # +-51.2 m

MUTATIONS = ("pad_dropped", "pad_on_full", "pad_unmasked", "mean_over_P", "xy_swapped", "no_half_voxel", "no_eps")

# (ndim, units) of the two kernels: the ndim-templated one runs units 64 at ndim 4 / 5, the generic one everything
# else, including ndim 4 / 5 at other widths so both kernels see the same point layouts
FIXED = [(4, 64), (5, 64)]
GENERIC = [(nd, u) for nd in (3, 4, 6, 11) for u in (32, 64, 96, 128) if (nd, u) != (4, 64)] + [(5, 32), (5, 96), (5, 128)]
SWEEP_P = (1, 20, 32, 33, 100)
# (ndim, units, P) whose staging needs the dynamic shared-memory opt-in above 48 KB
OPT_IN = [(8, 128, 400), (5, 64, 600), (4, 64, 800)]


def staging_bytes(ndim, units, P, warps=4):
    return ((ndim + 5) * units + warps * P * ndim) * 4


def sweep_cases():
    """(name, ndim, units, P, clouds, regime, seed) of the synthetic sweep: every kernel shape at every P, KITTI and
    nuScenes coordinates alternating, two clouds (41 rows: not a multiple of the 4 warps of a CTA); then the
    shared-memory opt-in shapes."""
    out = []
    for nd, u in FIXED + GENERIC:
        for i, P in enumerate(SWEEP_P):
            kitti = (i + nd) % 2 == 0
            out.append(("nd%d_u%d_P%d_%s" % (nd, u, P, "kitti" if kitti else "nusc"), nd, u, P, [23, 18],
                        KITTI if kitti else NUSC, 1000 * nd + 7 * u + P))
    for nd, u, P in OPT_IN:
        out.append(("nd%d_u%d_P%d_optin" % (nd, u, P), nd, u, P, [9, 7], KITTI, 1000 * nd + 7 * u + P))
    return out


def gamma(n, u=U):
    """gamma_n = n u / (1 - n u): the relative error of n chained roundings (Higham, Accuracy and Stability, 3.1)."""
    return n * u / (1 - n * u)


def grid_of(regime):
    vs, pcr = regime["vs"], regime["pcr"]
    return [int(np.round(np.float32(pcr[3 + j] - pcr[j]) / np.float32(vs[j]))) for j in range(2)]


def offsets_of(vs, pcr):
    """The module's pillar-centre offsets, as Python doubles (pillar_encoder.py: vx / 2 + pc_range[0])."""
    return float(vs[0]) / 2 + float(pcr[0]), float(vs[1]) / 2 + float(pcr[1])


def make_params(ndim, units, seed):
    """PFN parameters that exercise every term of the bound: mixed-sign weights; BatchNorm with negative gammas, a
    quarter of the units at variances far below eps (scale up to ~30), means and betas that give shifts of both signs.
    fp32 values, as the module holds them."""
    g = torch.Generator().manual_seed(seed)
    n_in = ndim + 5
    w = (torch.rand(units, n_in, generator=g) * 2 - 1) / n_in ** 0.5
    gam = (0.5 + torch.rand(units, generator=g)) * torch.where(torch.rand(units, generator=g) < 0.35, -1.0, 1.0)
    tiny = torch.rand(units, generator=g) < 0.25
    var = torch.where(tiny, 10 ** (-5 + 1.5 * torch.rand(units, generator=g)), 10 ** (-1 + 1.5 * torch.rand(units, generator=g)))
    mu = torch.randn(units, generator=g) * 2
    beta = torch.randn(units, generator=g) * 2
    return {"linear.weight": w.float(), "norm.running_mean": mu.float(), "norm.running_var": var.float(),
            "norm.weight": gam.float(), "norm.bias": beta.float()}


def fold(par, device=None):
    """Scale and shift of the folded BatchNorm, computed in float64 and rounded once to fp32 (as PillarFeatureNet does)."""
    var, gam = par["norm.running_var"].double(), par["norm.weight"].double()
    s = gam / torch.sqrt(var + EPS)
    t = par["norm.bias"].double() - par["norm.running_mean"].double() * s
    return s.float().to(device), t.float().to(device)


def _counts(n, P, rng):
    """1, 2, P-1 and P, then uniform draws: every count class in every launch."""
    base = [1, 2, P - 1, P]
    c = [base[i] if i < 4 else int(rng.integers(1, P + 1)) for i in range(n)]
    return [min(max(x, 1), P) for x in c]


def make_case(ndim, P, clouds, regime, seed, max_voxels=None):
    """Synthetic clouds already grouped into pillars.  clouds: pillars per cloud (0 = an empty cloud).  Per cloud: the
    four corner cells of the grid first (first / last row and column), then distinct random cells; point counts
    1, 2, P-1, P, then random; the P-count pillar has all its points at one coordinate; every third pillar carries
    intensity / time columns of magnitude up to 1e3.  The points of the whole batch are shuffled, so list order and row
    order differ.  Returns host tensors: points [N, ndim], lists [B, max_voxels, P] (the layout csrc/voxelize.cu
    writes, empty slots >= SENTINEL), counts [B], and per row nums [T], coors [T, 4] (b, z, y, x), voxels [T, P, ndim]
    (zero padded)."""
    rng = np.random.default_rng(seed)
    vs, pcr = regime["vs"], regime["pcr"]
    nx, ny = grid_of(regime)
    mv = max_voxels if max_voxels is not None else max(max(clouds), 1) + 2
    assert max(clouds) <= mv
    corners = [(0, 0), (0, nx - 1), (ny - 1, 0), (ny - 1, nx - 1)]
    pts, rows = [], []                       # rows: (b, j, iy, ix, [point ids])
    for b, m in enumerate(clouds):
        cells = corners[:m]
        if m > 4:
            taken = {iy * nx + ix for iy, ix in corners}
            pick = [int(c) for c in rng.choice(nx * ny, m + 4, replace=False) if int(c) not in taken][:m - 4]
            cells = cells + [(c // nx, c % nx) for c in pick]
        for j, ((iy, ix), cnt) in enumerate(zip(cells, _counts(m, P, rng))):
            p = np.zeros((cnt, ndim), np.float64)
            p[:, 0] = pcr[0] + (ix + rng.uniform(0, 1, cnt)) * vs[0]
            p[:, 1] = pcr[1] + (iy + rng.uniform(0, 1, cnt)) * vs[1]
            p[:, 2] = rng.uniform(pcr[2], pcr[5], cnt)
            big = 1e3 if j % 3 == 2 else 1.0
            if ndim > 3:
                p[:, 3] = rng.uniform(0, 1, cnt) * big
            if ndim > 4:
                p[:, 4] = rng.uniform(-0.5, 0.5, cnt) * big
            if ndim > 5:
                p[:, 5:] = rng.normal(0, 1, (cnt, ndim - 5))
            if j == 3:
                p[:] = p[0]
            start = sum(x.shape[0] for x in pts)
            ids = list(range(start, start + cnt))
            pts.append(p.astype(np.float32))
            rows.append((b, j, iy, ix, ids))
    allp = np.concatenate(pts, 0) if pts else np.zeros((0, ndim), np.float32)
    perm = rng.permutation(allp.shape[0])                 # new position of every point
    points = np.zeros_like(allp)
    points[perm] = allp
    B, T = len(clouds), len(rows)
    lists = SENTINEL + (np.arange(B * mv * P, dtype=np.int64) % 4096).reshape(B, mv, P).astype(np.int32)
    nums = np.zeros(T, np.int32)
    coors = np.zeros((T, 4), np.int32)
    voxels = np.zeros((T, P, ndim), np.float32)
    for r, (b, j, iy, ix, ids) in enumerate(rows):
        lists[b, j, :len(ids)] = perm[ids]
        nums[r] = len(ids)
        coors[r] = (b, 0, iy, ix)
        voxels[r, :len(ids)] = points[perm[ids]]
    return dict(points=torch.from_numpy(points), lists=torch.from_numpy(lists),
                counts=torch.tensor(clouds, dtype=torch.int32), nums=torch.from_numpy(nums),
                coors=torch.from_numpy(coors), voxels=torch.from_numpy(voxels), vs=vs, pcr=pcr, P=P, ndim=ndim,
                max_voxels=mv)


def _decorate(v, nums, coors, vs, pcr, mutation=None):
    """[M, P, ndim] float64 -> the nine-or-more decorated features [M, P, ndim + 5] (before the padding mask)."""
    P = v.shape[1]
    vx, vy = float(vs[0]), float(vs[1])
    x_off, y_off = offsets_of(vs, pcr)
    if mutation == "no_half_voxel":
        x_off = float(pcr[0])
    div = float(P) if mutation == "mean_over_P" else nums.double().view(-1, 1, 1)
    mean = v[:, :, :3].sum(dim=1, keepdim=True) / div
    ix, iy = (coors[:, 2], coors[:, 3]) if mutation == "xy_swapped" else (coors[:, 3], coors[:, 2])
    cx = (ix.double() * vx + x_off).view(-1, 1, 1)
    cy = (iy.double() * vy + y_off).view(-1, 1, 1)
    return torch.cat([v, v[:, :, :3] - mean, v[:, :, 0:1] - cx, v[:, :, 1:2] - cy], dim=-1)


def reference(par, voxels, nums, coors, vs, pcr, mutation=None):
    """The operation in float64 (pillar_encoder.py:115-155, :33-47), with one rule optionally broken (MUTATIONS).
    Unmutated it is `oracle.pillars_cpu.pillar_features(..., dtype=torch.float64)` restated in terms the mutations can
    reach; tests/test_pillar_error_model.py pins the two together."""
    v = voxels.double()
    dev = v.device
    P = v.shape[1]
    f = _decorate(v, nums, coors, vs, pcr, mutation)
    occ = torch.arange(P, device=dev).view(1, -1) < nums.to(dev).view(-1, 1)
    if mutation != "pad_unmasked":
        f = f * occ.unsqueeze(-1).double()
    p = {k: x.double().to(dev) for k, x in par.items()}
    eps = 0.0 if mutation == "no_eps" else EPS
    x = f @ p["linear.weight"].t()
    y = torch.relu((x - p["norm.running_mean"]) / torch.sqrt(p["norm.running_var"] + eps) * p["norm.weight"] + p["norm.bias"])
    if mutation == "pad_dropped":
        y = y * occ.unsqueeze(-1).double()             # relu output >= 0: 0 is neutral in the max
    out = y.max(dim=1)[0]
    if mutation == "pad_on_full":
        t = p["norm.bias"] - p["norm.running_mean"] * p["norm.weight"] / torch.sqrt(p["norm.running_var"] + EPS)
        out = torch.maximum(out, torch.relu(t).view(1, -1))
    return out


def error_bound(par, voxels, nums, coors, vs, pcr):
    """|got - y64| <= error_bound elementwise, for the fp32 kernel's output `got` and the float64 operation `y64`, from
    per-operation roundings (u = 2^-24, round to nearest; gamma_n = n u / (1 - n u); no fast-math) -- derived, not
    fitted.  Per pillar with n = num_points points q_p (exact fp32 inputs; n <= P here) and per output unit c:

    * Mean.  The kernel's fp32 sum of the n values, in any order and tree, is within gamma_n A_k of the exact sum,
      A_k = sum_p |q_pk|; times fl(1/n) (or divided: the reference's form) and one more rounding, possibly contracted
      into the cluster offset's subtraction: |mean^_k - mean_k| <= e_mean_k = gamma_{n+2} A_k / n.
    * Cluster offset fl(q - mean^): |f^ - f| <= (1 + u) e_mean + u |q - mean|.
    * Centre offset fl(q - c^x), c^x = coor * fl32(vx) + fl32(x_offset) in fp32 (product and sum rounded, or one FMA):
      |c^x - cx| <= e_c = gamma_3 (|coor vx| + |x_offset|); |f^ - f| <= (1 + u) e_c + u |q - cx|.  Raw columns are
      exact (D = 0).
    * Dot product, n_in = ndim + 5 chained FMAs from 0 over the decorated features f^ (|f^| <= |f| + D):
      |acc^ - acc| <= e_acc = gamma_{n_in} sum_d |w_d| (|f_d| + D_d) + sum_d |w_d| D_d.
    * Folded BatchNorm.  s = gamma / sqrt(var + eps) and t = beta - mean s, evaluated in float64 (3 / 4 roundings) and
      rounded once to fp32: e_s = (u + 2 gamma64_3) |s|, e_t = u |t| + 2 gamma64_4 (|beta| + |mean s|).  Then one
      fmaf(acc^, s^, t^): |y^ - y| <= (1 + u)(|s^| e_acc + |acc| e_s + e_t) + u (|acc| |s| + |t|), |s^| <= |s| + e_s.
    * ReLU and the max over the point slots are 1-Lipschitz, so the output's error is at most the largest per-point
      bound, and, when n < P, at most e_t for the padded slots' relu(t^) as well.
    * The float64 reference's own rounding: gamma64_{P + n_in + 8} times the magnitudes of every intermediate (the
      features and their sums, |s| sum |w| G, |mean s|, |beta|).  ~1e-14 relative: it only keeps the bound honest.

    Evaluated in float64 on the device of `voxels` ([M, P, ndim], zero padded); returns [M, units]."""
    v = voxels.double()
    dev = v.device
    M, P, ndim = v.shape
    n_in = ndim + 5
    n = nums.to(dev).double()
    occ = torch.arange(P, device=dev).view(1, -1) < nums.to(dev).view(-1, 1)
    p = {k: x.double().to(dev) for k, x in par.items()}
    W = p["linear.weight"]
    Wa = W.abs()
    s = p["norm.weight"] / torch.sqrt(p["norm.running_var"] + EPS)
    t = p["norm.bias"] - p["norm.running_mean"] * s
    f = _decorate(v, nums.to(dev), coors.to(dev), vs, pcr) * occ.unsqueeze(-1).double()
    F_ = f.abs()
    A = v[:, :, :3].abs().sum(dim=1)                                            # [M, 3]
    e_mean = gamma(n + 2).view(-1, 1) * A / n.view(-1, 1)
    vx, vy = float(vs[0]), float(vs[1])
    x_off, y_off = offsets_of(vs, pcr)
    cmag = torch.stack([(coors[:, 3].to(dev).double() * vx).abs() + abs(x_off),
                        (coors[:, 2].to(dev).double() * vy).abs() + abs(y_off)], 1)   # [M, 2]
    e_c = gamma(3) * cmag
    D = torch.zeros_like(f)
    D[:, :, ndim:ndim + 3] = (1 + U) * e_mean.unsqueeze(1) + U * F_[:, :, ndim:ndim + 3]
    D[:, :, ndim + 3:] = (1 + U) * e_c.unsqueeze(1) + U * F_[:, :, ndim + 3:]
    acc = (f @ W.t()).abs()
    e_acc = gamma(n_in) * ((F_ + D) @ Wa.t()) + D @ Wa.t()
    sa, ta, ms = s.abs(), t.abs(), (p["norm.running_mean"] * s).abs()
    e_s = (U + 2 * gamma(3, U64)) * sa
    e_t = U * ta + 2 * gamma(4, U64) * (p["norm.bias"].abs() + ms)
    e_y = (1 + U) * ((sa + e_s) * e_acc + acc * e_s + e_t) + U * (acc * sa + ta)
    G = F_.clone()
    G[:, :, ndim:ndim + 3] += (A / n.view(-1, 1)).unsqueeze(1)
    G[:, :, ndim + 3:] += cmag.unsqueeze(1)
    e_ref = gamma(P + n_in + 8, U64) * (sa * (G @ Wa.t()) + ms + p["norm.bias"].abs())
    per_point = (e_y + e_ref).masked_fill(~occ.unsqueeze(-1), 0.0)
    bound = per_point.amax(dim=1)
    pad = e_t + gamma(8, U64) * (ms + p["norm.bias"].abs())
    padded = (nums.to(dev) < P).view(-1, 1)
    return torch.where(padded, torch.maximum(bound, pad.view(1, -1)), bound)
