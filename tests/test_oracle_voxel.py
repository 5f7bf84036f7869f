"""Pins the voxelizer oracle (C restatement + numpy restatement) to the reference numba
function through the committed golden fixtures (tests/golden/make_golden.py)."""
import os

import numpy as np
import pytest

from boundary_golden import voxel_clouds
from conftest import golden_voxel_cases, load_golden
from oracle import voxel as ovoxel


@pytest.mark.parametrize("case", golden_voxel_cases())
def test_c_oracle_matches_reference_golden(case):
    g = load_golden("voxel_" + case)
    v, c, n = ovoxel.points_to_voxel(g["points"], g["voxel_size"], g["pcr"], int(g["max_points"]), True,
                                     int(g["max_voxels"]))
    assert np.array_equal(c, g["coors"])
    assert np.array_equal(n, g["num_points"])
    assert np.array_equal(v, g["voxels"])


@pytest.mark.parametrize("case", [c for c in golden_voxel_cases() if c not in ("kitti_empty", "kitti_all_outside")])
def test_numpy_restatement_matches_reference_golden(case):
    g = load_golden("voxel_" + case)
    v, c, n = ovoxel.points_to_voxel_numpy(g["points"], g["voxel_size"], g["pcr"], int(g["max_points"]),
                                           int(g["max_voxels"]))
    assert np.array_equal(c, g["coors"]) and np.array_equal(n, g["num_points"]) and np.array_equal(v, g["voxels"])


def test_overflow_break_drops_late_points_of_open_voxels():
    # 3 voxels allowed; the 4th new voxel appears at point 3 -> points 4.. are dropped even
    # though point 4 belongs to voxel 0 (point_cloud_ops.py:46-47 is a `break`).
    vs, pcr = [1.0, 1.0, 1.0], [0, 0, 0, 10, 10, 1]
    pts = np.array([[0.5, 0.5, 0.5], [1.5, 0.5, 0.5], [2.5, 0.5, 0.5], [3.5, 0.5, 0.5], [0.6, 0.5, 0.5]], np.float32)
    v, c, n = ovoxel.points_to_voxel(pts, vs, pcr, 5, True, 3)
    assert n.tolist() == [1, 1, 1] and c[:, 2].tolist() == [0, 1, 2]


def test_dense_map_scratch_is_restored():
    vs, pcr = np.float32([0.5, 0.5, 0.5]), np.float32([0, 0, 0, 4, 4, 2])
    grid = ovoxel.grid_size(vs, pcr)
    scratch = -np.ones(int(np.prod(grid)), np.int32)
    pts = np.random.default_rng(0).uniform(0, 2, (100, 3)).astype(np.float32)
    a = ovoxel.points_to_voxel(pts, vs, pcr, 4, True, 50, dense_map=scratch)
    b = ovoxel.points_to_voxel(pts, vs, pcr, 4, True, 50)
    assert (scratch == -1).all()
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_c_oracle_matches_live_reference_on_fresh_seeds():
    """The C restatement vs the reference's own points_to_voxel on three seeded clouds (its outputs:
    tests/golden/live_voxel_reference.npz, tests/golden/make_golden_boundary.py)."""
    g = load_golden("live_voxel_reference")
    for seed, (pts, vs, pcr, max_pts, max_vox) in enumerate(voxel_clouds()):
        got = ovoxel.points_to_voxel(pts, vs, pcr, max_pts, True, max_vox)
        for name, a in zip(("voxels", "coors", "num_points"), got):
            want = g["%s_%d" % (name, seed)]
            assert a.dtype == want.dtype and np.array_equal(a, want), (seed, name)


def test_c_oracle_equals_aot_reference_kernel_on_random_inputs():
    """Beyond the committed goldens: the C restatement must reproduce the reference's own numba kernel (compiled ahead of
    time, oracle/build.py; its outputs stored as digests in tests/golden/aot_voxel_reference.json) bit for bit on seeded
    clouds -- boundary-snapped points, overflow `break`, ndim 3/4/5, an empty cloud."""
    import json

    from boundary_golden import GOLDEN, aot_voxel_cases, digest
    from oracle import voxel

    with open(os.path.join(GOLDEN, "aot_voxel_reference.json")) as fh:
        want = json.load(fh)
    for i, (pts, vs, pcr, max_pts, max_vox) in enumerate(aot_voxel_cases()):
        got = voxel.points_to_voxel(pts, vs, pcr, max_pts, True, max_vox)
        assert [digest(a) for a in got] == want[i], i
