"""d3b_voxelize_dev (cloud offsets in device memory) at any point capacity >= the live total against the same call at
exactly the live total (the values themselves are pinned by the reference goldens: test_voxelize_gpu.py,
test_oracle_voxel.py): bit for bit on every output and on the per-voxel point-index lists, with NaN / huge padding past
the total, through the Voxelizer's host-offsets call, inside a CUDA graph replayed over offsets of different sizes, and
with malformed offsets (flagged in `status`, then run clamped)."""
import numpy as np
import pytest
import torch

from conftest import golden_voxel_cases, load_golden

pytestmark = pytest.mark.gpu

KITTI = dict(vs=[0.05, 0.05, 0.1], pcr=[0, -40.0, -3.0, 70.4, 40.0, 1.0])
MODES = [(True, True), (True, False), (False, True), (False, False)]     # (want_voxels, want_mean)


def _voxelizer(vs, pcr, max_points, max_voxels, want_voxels=True, want_mean=True):
    from det3d_b200.ops.point_cloud.voxelize import Voxelizer
    return Voxelizer(vs, pcr, max_points, max_voxels, want_voxels=want_voxels, want_mean=want_mean)


def _bits(t):
    a = t.cpu().numpy()
    return a.view(np.int32) if a.dtype == np.float32 else a


def _result(vox, out, batch):
    """Every defined output of one call as host arrays (floats as their bit patterns), point lists included."""
    counts = out["counts"].cpu().numpy()
    m = int(counts[batch])
    res = {"counts": counts}
    for k in ("voxels", "coors", "num_points", "mean"):
        if out[k] is not None:
            res[k] = _bits(out[k][:m])
    pl = out["point_lists"]
    ws = pl["keepalive"]
    start = pl["lists_ptr"] - ws.data_ptr()
    n = pl["batch"] * pl["max_voxels"] * pl["max_points"]
    res["point_lists"] = ws[start:start + 4 * n].view(torch.int32).cpu().numpy()
    return res


def _assert_same(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k].shape == b[k].shape, k
        assert np.array_equal(a[k], b[k]), k


def _host(vox, clouds):
    """The clouds through the Voxelizer's host-offsets call."""
    offs = np.cumsum([0] + [c.shape[0] for c in clouds]).tolist()
    pts = torch.from_numpy(np.concatenate(clouds).astype(np.float32)).cuda()
    return _result(vox, vox(pts, offs), len(clouds))


def _dev(vox, clouds, capacity=None, pad=np.nan):
    """The clouds through d3b_voxelize_dev at `capacity` (default: exactly their total), rows past the live total
    filled with `pad`."""
    offs = np.cumsum([0] + [c.shape[0] for c in clouds])
    total = int(offs[-1])
    capacity = total if capacity is None else capacity
    ndim = clouds[0].shape[1]
    pts = np.full((capacity, ndim), pad, np.float32)
    pts[:total] = np.concatenate(clouds)
    out = vox(torch.from_numpy(pts).cuda(), torch.from_numpy(offs.astype(np.int32)).cuda())
    res = _result(vox, out, len(clouds))
    assert int(out["status"].item()) == 0
    return res


@pytest.mark.parametrize("case", golden_voxel_cases())
def test_golden_cases_match_the_host_offsets_call(case):
    g = load_golden("voxel_" + case)
    vox = _voxelizer(g["voxel_size"], g["pcr"], int(g["max_points"]), int(g["max_voxels"]))
    want = _dev(vox, [g["points"]])
    n = g["points"].shape[0]
    _assert_same(_host(vox, [g["points"]]), want)
    for capacity, pad in ((n + 1, np.nan), (n + 5000, 1e30), (4 * n + 1024, np.nan)):
        _assert_same(_dev(vox, [g["points"]], capacity, pad), want)


def _mixed_clouds(ndim=4):
    from det3d_b200.utils.synthetic import lidar_like_cloud, uniform_cloud
    return [lidar_like_cloud(7000, KITTI["pcr"], ndim, 1), np.zeros((0, ndim), np.float32),
            lidar_like_cloud(1, KITTI["pcr"], ndim, 2), uniform_cloud(9000, KITTI["pcr"], ndim, 3),
            np.zeros((0, ndim), np.float32), lidar_like_cloud(300, KITTI["pcr"], ndim, 4)]


@pytest.mark.parametrize("want_voxels,want_mean", MODES)
def test_mixed_batch_with_a_max_voxels_cut(want_voxels, want_mean):
    """Empty and single-point clouds, and max_voxels = 2500 cutting the 9k-point uniform cloud short (the reference
    `break`)."""
    clouds = _mixed_clouds()
    vox = _voxelizer(KITTI["vs"], KITTI["pcr"], 5, 2500, want_voxels, want_mean)
    want = _dev(vox, clouds)
    assert want["counts"][3] == 2500 and want["counts"][1] == 0 and want["counts"][2] <= 1
    total = sum(c.shape[0] for c in clouds)
    _assert_same(_host(vox, clouds), want)
    _assert_same(_dev(vox, clouds, total + 3000, np.nan), want)
    _assert_same(_dev(vox, clouds, 1 << 16, 1e30), want)


@pytest.mark.parametrize("want_voxels,want_mean", MODES)
def test_batch_1_and_batch_64(want_voxels, want_mean):
    from det3d_b200.utils.synthetic import lidar_like_cloud
    vox = _voxelizer(KITTI["vs"], KITTI["pcr"], 5, 20000, want_voxels, want_mean)
    one = [lidar_like_cloud(20000, KITTI["pcr"], 4, 7)]
    _assert_same(_dev(vox, one, 32768, 1e30), _dev(vox, one))
    rng = np.random.default_rng(5)
    many = [lidar_like_cloud(int(n), KITTI["pcr"], 4, 100 + i) if n else np.zeros((0, 4), np.float32)
            for i, n in enumerate(rng.integers(0, 3000, 64))]
    many[10] = np.zeros((0, 4), np.float32)
    many[63] = lidar_like_cloud(1, KITTI["pcr"], 4, 9)
    vox64 = _voxelizer(KITTI["vs"], KITTI["pcr"], 5, 400, want_voxels, want_mean)
    want = _dev(vox64, many)
    total = sum(c.shape[0] for c in many)
    _assert_same(_host(vox64, many), want)
    _assert_same(_dev(vox64, many, total + 777, np.nan), want)


def test_one_graph_replays_offsets_of_any_size():
    """One captured d3b_voxelize_dev call, replayed with 6 different offset vectors (batch 3), equals the eager call
    on the exactly sized points each time."""
    from det3d_b200.utils.synthetic import lidar_like_cloud
    capacity, batch = 1 << 15, 3
    vox = _voxelizer(KITTI["vs"], KITTI["pcr"], 5, 3000)
    ref = _voxelizer(KITTI["vs"], KITTI["pcr"], 5, 3000)
    pts = torch.full((capacity, 4), float("nan"), device="cuda")
    offs = torch.zeros(batch + 1, dtype=torch.int32, device="cuda")
    vox(pts, offs)                                   # allocates the capacity's buffers outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = vox(pts, offs)
    rng = np.random.default_rng(3)
    sizes = [(1000, 2000, 3000), (0, 10000, 1), (9000, 9000, 9000), (1, 0, 0), (20000, 500, 12000), (0, 0, 0)]
    for step, ns in enumerate(sizes):
        clouds = [lidar_like_cloud(n, KITTI["pcr"], 4, 10 * step + j) if n else np.zeros((0, 4), np.float32)
                  for j, n in enumerate(ns)]
        o = np.cumsum([0] + list(ns)).astype(np.int32)
        if o[-1]:
            pts[:o[-1]].copy_(torch.from_numpy(np.concatenate(clouds)))
        pts[o[-1]:int(rng.integers(o[-1], capacity + 1))] = 1e30
        offs.copy_(torch.from_numpy(o))
        graph.replay()
        got = _result(vox, out, batch)
        assert int(out["status"].item()) == 0
        _assert_same(got, _dev(ref, clouds))


@pytest.mark.parametrize("raw,clamped", [
    ([0, 3000, 2000, 5000], [0, 3000, 3000, 5000]),           # not monotone
    ([0, 3000, 5000, 9000], [0, 3000, 5000, 8192]),           # past the capacity
    ([0, 9000, 100, 20000], [0, 8192, 8192, 8192]),           # both
    ([5, 3000, 4000, 6000], [0, 3000, 4000, 6000]),           # off[0] != 0
    ([0, -7, 4000, 6000], [0, 0, 4000, 6000]),                # negative
    ([0, 3000, 3000, 2 ** 31 - 1], [0, 3000, 3000, 8192]),
])
def test_malformed_offsets_set_status_and_run_clamped(raw, clamped):
    """The clamp comes before any point index is formed: the outputs are those of the clamped offsets."""
    from det3d_b200.utils.synthetic import uniform_cloud
    capacity = 8192
    pts_np = uniform_cloud(capacity, KITTI["pcr"], 4, 21)
    vox = _voxelizer(KITTI["vs"], KITTI["pcr"], 5, 4000)
    ref = _voxelizer(KITTI["vs"], KITTI["pcr"], 5, 4000)
    out = vox(torch.from_numpy(pts_np).cuda(), torch.tensor(raw, dtype=torch.int32, device="cuda"))
    assert int(out["status"].item()) == 1
    got = _result(vox, out, 3)
    want = _dev(ref, [pts_np[a:b] for a, b in zip(clamped[:-1], clamped[1:])])
    _assert_same(got, want)
    # a well-formed call on the same buffers clears the status again
    ok = vox(torch.from_numpy(pts_np).cuda(), torch.tensor(clamped, dtype=torch.int32, device="cuda"))
    assert int(ok["status"].item()) == 0
