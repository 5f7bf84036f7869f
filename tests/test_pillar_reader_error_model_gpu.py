"""The PointPillars reader (`csrc/pillars.cu`) against the float64 operation and its own error model
(`tests/pillar_error_model.py: error_bound`), through both point sources: the materialised [rows, P, ndim] voxel
tensor (`d3b_pillar_features`) and the voxelizer's point-index lists (`d3b_pillar_features_lists`).  The two sources
must give the same bits; both must be within the bound on every output; rows past the live count must be exactly 0
whatever the output buffer held, and poisoned inputs past it must not matter."""
import os

import numpy as np
import pytest
import torch

import pillar_error_model as pem
from conftest import ROOT

pytestmark = pytest.mark.gpu

NAN_POISON = (float("nan"), 1e30)
INT_POISON = 1 << 30


def _kernel(ndim, units):
    return "fixed" if (ndim, units) in pem.FIXED else "generic"


def _poisoned(case, n, R):
    """Row arrays of capacity R for the kernels: the case's rows below n, poison from n on (NaN / 1e30 in the voxels,
    2^30 in num_points and coors)."""
    T, P, nd = case["nums"].shape[0], case["P"], case["ndim"]
    vox = torch.empty((R, P, nd), dtype=torch.float32)
    vox.view(R, -1)[:, 0::2] = NAN_POISON[0]
    vox.view(R, -1)[:, 1::2] = NAN_POISON[1]
    nums = torch.full((R,), INT_POISON, dtype=torch.int32)
    coors = torch.full((R, 4), INT_POISON, dtype=torch.int32)
    k = min(n, T)
    vox[:k], nums[:k], coors[:k] = case["voxels"][:k], case["nums"][:k], case["coors"][:k]
    return vox.cuda(), nums.cuda(), coors.cuda()


def _folded(par):
    scale, shift = pem.fold(par, "cuda")
    return par["linear.weight"].cuda().contiguous(), scale.contiguous(), shift.contiguous()


def _launch_dense(vox, nums, coors, n_dev, R, P, ndim, par, vs, pcr):
    from det3d_b200 import _lib
    units = par["linear.weight"].shape[0]
    w, scale, shift = _folded(par)
    out = torch.full((max(R, 1), units), float("nan"), device="cuda")
    nd = torch.tensor([n_dev], dtype=torch.int32, device="cuda")
    x_off, y_off = pem.offsets_of(vs, pcr)
    st = _lib.lib().d3b_pillar_features(vox.data_ptr(), nums.data_ptr(), coors.data_ptr(), nd.data_ptr(), R, P, ndim, units,
                                        w.data_ptr(), scale.data_ptr(), shift.data_ptr(), float(vs[0]), float(vs[1]),
                                        x_off, y_off, out.data_ptr(), _lib.current_stream())
    _lib.check(st, "d3b_pillar_features")
    torch.cuda.synchronize()
    return out[:R]


def _launch_lists(points, lists, counts, nums, coors, n_dev, R, P, ndim, par, vs, pcr):
    from det3d_b200 import _lib
    units = par["linear.weight"].shape[0]
    w, scale, shift = _folded(par)
    out = torch.full((max(R, 1), units), float("nan"), device="cuda")
    nd = torch.tensor([n_dev], dtype=torch.int32, device="cuda")
    x_off, y_off = pem.offsets_of(vs, pcr)
    st = _lib.lib().d3b_pillar_features_lists(
        points.data_ptr(), lists.data_ptr(), counts.data_ptr(), lists.shape[0], lists.shape[1], nums.data_ptr(),
        coors.data_ptr(), nd.data_ptr(), R, P, ndim, units, w.data_ptr(), scale.data_ptr(), shift.data_ptr(),
        float(vs[0]), float(vs[1]), x_off, y_off, out.data_ptr(), _lib.current_stream())
    _lib.check(st, "d3b_pillar_features_lists")
    torch.cuda.synchronize()
    return out[:R]


def _within_bound(got, par, voxels, nums, coors, vs, pcr, chunk=4096):
    """max |got - y64| / bound over the rows of `got` (float64 oracle and bound on the device, in chunks); exact
    equality wherever the bound is 0.  Never runs the kernel under test."""
    from oracle.pillars_cpu import pillar_features
    sd = {"reader.pfn_layers.0." + k: v for k, v in par.items()}
    worst = 0.0
    for a in range(0, got.shape[0], chunk):
        b = min(a + chunk, got.shape[0])
        args = (voxels[a:b].cuda(), nums[a:b].cuda(), coors[a:b].cuda(), vs, pcr)
        y = pillar_features(sd, *args, dtype=torch.float64)
        bound = pem.error_bound(par, *args)
        err = (got[a:b].double() - y).abs()
        assert bool(torch.isfinite(err).all()), "non-finite output in rows %d..%d" % (a, b)
        assert bool((err[bound == 0] == 0).all())
        worst = max(worst, float((err / bound.clamp_min(1e-300)).max()))
    return worst


def _run(case, par, n_dev, R, name):
    """Both sources on the same rows; returns the output.  Asserts bit-identity, the zero rows and the bound."""
    P, nd, vs, pcr = case["P"], case["ndim"], case["vs"], case["pcr"]
    T = case["nums"].shape[0]
    n = max(min(n_dev, R), 0)
    assert n <= T <= R
    vox, nums, coors = _poisoned(case, n, R)
    dense = _launch_dense(vox, nums, coors, n_dev, R, P, nd, par, vs, pcr)
    lists = _launch_lists(case["points"].cuda(), case["lists"].cuda(), case["counts"].cuda(), nums, coors, n_dev, R, P,
                          nd, par, vs, pcr)
    assert torch.equal(dense, lists), "%s: the voxel tensor and the point lists give different bits" % name
    assert bool((dense[n:] == 0).all()), "%s: rows past the live count are not 0" % name
    if n:
        ratio = _within_bound(dense[:n], par, case["voxels"][:n], case["nums"][:n], case["coors"][:n], vs, pcr)
        units = par["linear.weight"].shape[0]
        print("pillars %s (%s kernel, n %d / cap %d): worst |got - y64| / bound = %.3g"
              % (name, _kernel(nd, units), n, R, ratio))
        assert ratio <= 1.0, "%s: %.3g x the error bound" % (name, ratio)
    return dense


@pytest.mark.parametrize("ndim,units", pem.FIXED + pem.GENERIC)
def test_kernel_shapes_within_error_model(ndim, units):
    """Every kernel shape at P = 1, 20, 32, 33, 100, KITTI and nuScenes coordinates, counts 1 / 2 / P-1 / P mixed in one
    launch, a row capacity of 43 (not a multiple of 4 warps) with 41 live rows."""
    cases = [c for c in pem.sweep_cases() if c[1:3] == (ndim, units) and not c[0].endswith("optin")]
    assert len(cases) == len(pem.SWEEP_P)
    for name, nd, u, P, clouds, regime, seed in cases:
        case = pem.make_case(nd, P, clouds, regime, seed)
        T = case["nums"].shape[0]
        _run(case, pem.make_params(nd, u, seed), T, T + 2, name)


@pytest.mark.parametrize("ndim,units,P", pem.OPT_IN)
def test_shared_memory_opt_in_within_error_model(ndim, units, P):
    """Point staging above the 48 KB default: the dynamic shared-memory opt-in of both kernels."""
    assert pem.staging_bytes(ndim, units, P) > 48 * 1024
    (name, nd, u, P_, clouds, regime, seed), = [c for c in pem.sweep_cases() if c[1:4] == (ndim, units, P)]
    case = pem.make_case(nd, P, clouds, regime, seed)
    T = case["nums"].shape[0]
    _run(case, pem.make_params(nd, u, seed), T, T + 1, name)


@pytest.mark.parametrize("ndim,units", [(4, 64), (5, 64), (6, 96)])
@pytest.mark.parametrize("mode", ["zero", "cap_minus_1", "cap", "above_cap"])
def test_live_count(ndim, units, mode):
    """n_dev = 0, row_cap - 1, row_cap and above it, with an empty cloud in the middle of the batch: only the first
    min(n_dev, row_cap) rows are computed, the rest are exactly 0 in an output buffer that held NaN."""
    case = pem.make_case(ndim, 20, [13, 0, 10], pem.NUSC if ndim == 5 else pem.KITTI, 17 * ndim + units)
    R = case["nums"].shape[0]
    assert R % 4 != 0
    n_dev = {"zero": 0, "cap_minus_1": R - 1, "cap": R, "above_cap": R + 5}[mode]
    out = _run(case, pem.make_params(ndim, units, 5 + ndim), n_dev, R, "live_%s_nd%d_u%d" % (mode, ndim, units))
    if mode == "zero":
        assert bool((out == 0).all())
        # and no rows at all, through the module: an empty [0, units] result, no launch
        from det3d.models.readers import PillarFeatureNet
        net = PillarFeatureNet(num_input_features=ndim, num_filters=[units], voxel_size=pem.KITTI["vs"],
                               pc_range=pem.KITTI["pcr"]).eval().cuda()
        with torch.no_grad():
            empty = net(case["voxels"][:0].cuda(), case["nums"][:0].cuda(), case["coors"][:0].cuda())
        assert empty.shape == (0, units)


LIST_BATCHES = {
    1: ((4, 64, 100), [24]),
    3: ((5, 64, 20), [0, 24, 0]),
    8: ((4, 96, 33), [0, 9, 3, 0, 0, 24, 4, 0]),
    64: ((4, 64, 20), [0 if b in (0, 31, 63) else 24 if b == 17 else 1 + b % 5 for b in range(64)]),
}


@pytest.mark.parametrize("B", sorted(LIST_BATCHES))
def test_list_batches(B):
    """List mode over B = 1, 3, 8, 64 clouds (the limit), empty clouds first, in the middle and last, one cloud at its
    max_voxels cap: within the bound, and each cloud's rows bit-identical whether it runs alone or inside the batch."""
    (nd, units, P), clouds = LIST_BATCHES[B]
    case = pem.make_case(nd, P, clouds, pem.NUSC if nd == 5 else pem.KITTI, 100 + B, max_voxels=24)
    assert max(clouds) == case["max_voxels"]
    par = pem.make_params(nd, units, B)
    T = case["nums"].shape[0]
    batch = _run(case, par, T, T + 3, "lists_B%d" % B)
    pts = case["points"].cuda()
    r = 0
    for b, m in enumerate(clouds):
        if m == 0:
            continue
        nums, coors = case["nums"][r:r + m].cuda(), case["coors"][r:r + m].cuda()
        alone = _launch_lists(pts, case["lists"][b:b + 1].cuda(), case["counts"][b:b + 1].cuda(), nums, coors, m, m,
                              P, nd, par, case["vs"], case["pcr"])
        assert torch.equal(alone, batch[r:r + m]), "cloud %d of %d" % (b, B)
        r += m


DEPLOYED = {
    # PointPillars KITTI (configs/pointpillars_kitti_car.py): 20k points x B = 8, P = 100, 12000 pillars per cloud
    "kitti": dict(cfg="pointpillars_kitti_car.py", ndim=4, n_points=20000, B=8),
    # nuScenes PointPillars (configs/pointpillars_nusc.py): 35k 5-feature points x B = 4, P = 20, 30000 pillars per cloud
    "nusc": dict(cfg="pointpillars_nusc.py", ndim=5, n_points=35000, B=4),
}


@pytest.mark.parametrize("config", sorted(DEPLOYED))
def test_deployed_within_error_model(config):
    """The deployed reader on the device voxelizer's voxels and lists, uniform (even) and LiDAR-like (odd) clouds: both
    sources bit-identical and within the bound, rows past the live count 0, two runs bit-identical."""
    from det3d.models.readers import PillarFeatureNet
    from det3d.torchie import Config
    from det3d_b200.ops.point_cloud.voxelize import Voxelizer
    from det3d_b200.utils.synthetic import lidar_like_cloud, uniform_cloud
    d = DEPLOYED[config]
    cfg = Config.fromfile(os.path.join(ROOT, "configs", d["cfg"]))
    vg, rd = cfg.voxel_generator, cfg.model["reader"]
    nd, B, P, mv = d["ndim"], d["B"], vg.max_points_in_voxel, vg.max_voxel_num
    vs, pcr = list(vg.voxel_size), list(vg.range)
    assert nd == rd.get("num_input_features", 4) and list(rd["num_filters"]) == [64]
    rng = np.random.default_rng(0)
    clouds = []
    for i in range(B):
        c = (uniform_cloud if i % 2 == 0 else lidar_like_cloud)(d["n_points"], pcr, nd, 40 + i)
        if nd > 4:
            c[:, 4] = rng.uniform(0, 0.5, c.shape[0]).astype(np.float32)          # sweep time lag
        clouds.append(c)
    net = PillarFeatureNet(num_input_features=nd, num_filters=[64], voxel_size=vs, pc_range=pcr).eval()
    par = pem.make_params(nd, 64, 7)
    layer = net.pfn_layers[0]
    with torch.no_grad():
        layer.linear.weight.copy_(par["linear.weight"])
        for k in ("running_mean", "running_var", "weight", "bias"):
            getattr(layer.norm, k).copy_(par["norm." + k])
    assert layer.norm.eps == pem.EPS
    net = net.cuda()
    pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    offsets = [d["n_points"] * i for i in range(B + 1)]
    vox = Voxelizer(vs, pcr, P, mv, want_voxels=True, want_mean=False)(pts, offsets)
    counts = vox["counts"]
    n, cap = int(counts[B]), B * mv
    assert int(counts[0]) == mv, "the uniform cloud must fill max_voxels"
    with torch.no_grad():
        dense = net.forward_fused(vox["voxels"], vox["num_points"], vox["coors"], n_dev=counts[B:B + 1]).clone()
        pl = dict(vox["point_lists"], counts=counts)
        lists = net.forward_lists(pl, vox["num_points"], vox["coors"], cap, counts[B:B + 1]).clone()
        net.__dict__["_out_bufs"][(cap, pts.device)].fill_(float("nan"))
        lists2 = net.forward_lists(pl, vox["num_points"], vox["coors"], cap, counts[B:B + 1]).clone()
        dense2 = net.forward_fused(vox["voxels"], vox["num_points"], vox["coors"], n_dev=counts[B:B + 1])
    torch.cuda.synchronize()
    assert dense.shape == (cap, 64)
    assert torch.equal(dense, lists), "the voxel tensor and the point lists give different bits"
    assert torch.equal(lists, lists2) and torch.equal(dense, dense2), "two runs differ"
    assert bool((dense[n:] == 0).all()) and bool((lists2[n:] == 0).all()), "rows past the live count are not 0"
    nums = vox["num_points"][:n]
    assert int(nums.min()) >= 1 and int(nums.max()) <= P and bool((nums < P).any())
    ratio = _within_bound(dense[:n], par, vox["voxels"][:n], nums, vox["coors"][:n], vs, pcr)
    print("pillars deployed %s (B %d, %d pillars, %d full, P %d): worst |got - y64| / bound = %.3g"
          % (config, B, n, int((nums == P).sum()), P, ratio))
    assert ratio <= 1.0
