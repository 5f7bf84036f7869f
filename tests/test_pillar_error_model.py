"""CPU, no GPU needed: the PointPillars reader's error model (tests/pillar_error_model.py) is tight enough to catch every
rule of the operation on the sweep's own inputs, and its float64 restatement is the oracle's."""
import functools

import pytest
import torch

import pillar_error_model as pem


@functools.lru_cache(maxsize=None)
def _case(i):
    name, nd, units, P, clouds, regime, seed = pem.sweep_cases()[i]
    c = pem.make_case(nd, P, clouds, regime, seed)
    par = pem.make_params(nd, units, seed)
    args = (c["voxels"], c["nums"], c["coors"], c["vs"], c["pcr"])
    return name, par, args, pem.reference(par, *args), pem.error_bound(par, *args)


def test_sweep_covers_both_kernels_and_the_opt_in():
    cases = pem.sweep_cases()
    shapes = {(nd, u) for _, nd, u, *_ in cases}
    assert {(4, 64), (5, 64)} <= shapes and {(4, 32), (5, 128), (3, 96), (11, 128)} <= shapes
    assert {P for *_, P, _, _, _ in cases} >= set(pem.SWEEP_P)
    fixed = [(nd, u, P) for nd, u, P in pem.OPT_IN if (nd, u) in pem.FIXED]
    generic = [(nd, u, P) for nd, u, P in pem.OPT_IN if (nd, u) not in pem.FIXED]
    assert fixed and generic
    for nd, u, P in pem.OPT_IN:
        assert 48 * 1024 < pem.staging_bytes(nd, u, P) <= 200 * 1024


def test_case_layout():
    """The lists hold the shuffled points of each row in slot order, empty slots at or above the sentinel; counts
    1, 2, P-1 and P and the four grid corners are present; one full pillar has all its points at one coordinate."""
    c = pem.make_case(5, 20, [0, 11, 0, 6, 0], pem.NUSC, 3)
    nums, lists, pts = c["nums"], c["lists"], c["points"]
    assert c["counts"].tolist() == [0, 11, 0, 6, 0] and nums.shape[0] == 17
    assert {1, 2, 19, 20} <= set(nums.tolist())
    nx, ny = pem.grid_of(pem.NUSC)
    cells = {(int(y), int(x)) for y, x in c["coors"][:, 2:].tolist()}
    assert {(0, 0), (0, nx - 1), (ny - 1, 0), (ny - 1, nx - 1)} <= cells
    r = 0
    for b, m in enumerate(c["counts"].tolist()):
        for j in range(m):
            k = int(nums[r])
            idx = lists[b, j, :k].long()
            assert torch.equal(pts[idx], c["voxels"][r, :k]) and bool((lists[b, j, k:] >= pem.SENTINEL).all())
            assert not torch.equal(idx, torch.arange(int(idx[0]), int(idx[0]) + k)) or k == 1
            if j == 3:
                assert k == 20 and bool((c["voxels"][r] == c["voxels"][r, 0]).all())
            r += 1
    assert bool((c["voxels"][nums == 1][:, 1:] == 0).all())


def test_reference_is_the_oracle_in_float64():
    """The mutable restatement, unmutated, is oracle.pillars_cpu.pillar_features(dtype=torch.float64)."""
    from oracle.pillars_cpu import pillar_features
    for i in (0, 7, 33, len(pem.sweep_cases()) - 1):
        name, par, args, y, _ = _case(i)
        voxels, nums, coors, vs, pcr = args
        sd = {"reader.pfn_layers.0." + k: v for k, v in par.items()}
        want = pillar_features(sd, voxels, nums, coors, vs, pcr, dtype=torch.float64)
        assert want.dtype == torch.float64
        assert float((want - y).abs().max()) <= 1e-12 * max(1.0, float(y.abs().max())), name


def test_bound_is_tight():
    """The bound is a few ulps of the outputs, not a flat tolerance: its median is below 1e-5 of the case's largest
    output on every case (the old flat 1e-4 was ~100x the kernel's error at O(1) features)."""
    for i in range(len(pem.sweep_cases())):
        name, _, _, y, b = _case(i)
        assert bool((b > 0).all()), name
        assert float(b.median()) <= 1e-5 * float(y.abs().max()), name


@pytest.mark.parametrize("mutation", pem.MUTATIONS)
def test_error_model_rejects_mutations(mutation):
    """Each rule of the operation decides some output of the sweep's data by far more than the bound: a kernel that
    broke the rule would be >= 10x outside it (its own rounding is within 1x)."""
    worst, where = 0.0, None
    for i in range(len(pem.sweep_cases())):
        name, par, args, y, b = _case(i)
        r = float(((pem.reference(par, *args, mutation=mutation) - y).abs() / b).max())
        if r > worst:
            worst, where = r, name
    print("mutation %s: worst |y_mut - y64| / bound = %.3g (%s)" % (mutation, worst, where))
    assert worst >= 10.0, "%s stays within %.3g x the bound: the data do not exercise it" % (mutation, worst)
