"""Seeded synthetic inputs (SURVEY 8d): point clouds, NMS box sets, random BN statistics."""
import numpy as np


def uniform_cloud(n, point_cloud_range, ndim=4, seed=0):
    """x,y,z ~ U[lo,hi) per axis, intensity ~ U[0,1), further features 0 (worst case for dilation)."""
    rng = np.random.default_rng(seed)
    r = np.asarray(point_cloud_range, np.float64)
    pts = np.zeros((n, ndim), np.float32)
    for j in range(3):
        pts[:, j] = rng.uniform(r[j], r[3 + j], n)
    if ndim > 3:
        pts[:, 3] = rng.uniform(0, 1, n)
    return pts


def lidar_like_cloud(n, point_cloud_range, ndim=4, seed=0):
    """64-beam spinning-lidar look-alike: rays from a sensor 1.73 m above the ground hit the
    ground plane or (35 %) an obstacle at 5-70 m; cropped to the range, shuffled, first n kept."""
    rng = np.random.default_rng(seed)
    r = np.asarray(point_cloud_range, np.float64)
    front_only = r[0] >= 0
    out = []
    need = n
    while need > 0:
        m = max(4 * need, 4096)
        beam = rng.integers(0, 64, m)
        elev = np.deg2rad(-24.8 + beam * (26.8 / 63.0))
        azim = rng.uniform(-np.pi / 4, np.pi / 4, m) if front_only else rng.uniform(-np.pi, np.pi, m)
        h = 1.73
        with np.errstate(divide="ignore"):
            ground_d = np.where(elev < -1e-3, h / np.tan(-elev), np.inf)
        obst = rng.uniform(0, 1, m) < 0.35
        obst_d = rng.uniform(5, 70, m)
        d = np.where(obst, np.minimum(obst_d, ground_d), ground_d)
        ok = np.isfinite(d) & (d < 120)
        d = np.where(ok, d, 1.0)
        z = -h + np.where(obst & (obst_d < ground_d), rng.uniform(0, 1.6, m), 0.0) + rng.normal(0, 0.02, m)
        x, y = d * np.cos(azim), d * np.sin(azim)
        ok &= (x >= r[0]) & (x < r[3]) & (y >= r[1]) & (y < r[4]) & (z >= r[2]) & (z < r[5])
        p = np.zeros((int(ok.sum()), ndim), np.float32)
        p[:, 0], p[:, 1], p[:, 2] = x[ok], y[ok], z[ok]
        if ndim > 3:
            p[:, 3] = rng.uniform(0, 1, p.shape[0])
        out.append(p)
        need -= p.shape[0]
    pts = np.concatenate(out, 0)
    rng.shuffle(pts)
    return np.ascontiguousarray(pts[:n])


def lidar_like_sweeps(sizes, point_cloud_range, seed=0, raw_stride=5, max_yaw=0.1, max_shift=5.0, lag_step=0.05,
                      close_fraction=0.0):
    """One nuScenes-style multi-sweep sample: (raw_sweeps, transforms, time_lags) for ingest_sweeps.  Sweep s is a seeded
    lidar_like_cloud of sizes[s] raw records (raw_stride floats), the key frame (s = 0) untransformed, every other
    sweep under a seeded rigid motion (yaw <= max_yaw rad, translation <= max_shift m) with lag lag_step * s.
    close_fraction of each sweep's points are moved inside the 1 m remove_close box."""
    rng = np.random.default_rng(seed)
    raws, tms, lags = [], [], []
    for s, n in enumerate(sizes):
        p = lidar_like_cloud(int(n), point_cloud_range, raw_stride, seed * 1000 + s) if n else np.zeros((0, raw_stride), np.float32)
        k = int(round(close_fraction * p.shape[0]))
        if k:
            p[:k, :2] = rng.uniform(-0.99, 0.99, (k, 2)).astype(np.float32)
        raws.append(p)
        if s == 0:
            tms.append(None)
        else:
            a = rng.uniform(-max_yaw, max_yaw)
            t = np.eye(4)
            t[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
            t[:3, 3] = rng.uniform(-1, 1, 3) * (max_shift / np.sqrt(3))
            tms.append(t)
        lags.append(lag_step * s)
    return raws, tms, lags


def nms_boxes_xyxyr(n, seed=0, clustered=False, extent=100.0):
    """[n,5] x1,y1,x2,y2,ry + distinct scores (SURVEY 8d C5)."""
    rng = np.random.default_rng(seed)
    if clustered:
        centres = rng.uniform(0, extent, (max(n // 50, 1), 2))
        c = centres[rng.integers(0, centres.shape[0], n)] + rng.normal(0, 3.0, (n, 2))
    else:
        c = rng.uniform(0, extent, (n, 2))
    w = rng.uniform(1.5, 2.5, n)
    l = rng.uniform(3.5, 5.0, n)
    ry = rng.uniform(-np.pi, np.pi, n)
    boxes = np.stack([c[:, 0] - w / 2, c[:, 1] - l / 2, c[:, 0] + w / 2, c[:, 1] + l / 2, ry], 1).astype(np.float32)
    scores = (rng.permutation(n).astype(np.float32) + 1) / n
    return boxes, scores


def xyxyr_to_xywlr(boxes):
    b = np.asarray(boxes, np.float32)
    return np.stack([(b[:, 0] + b[:, 2]) / 2, (b[:, 1] + b[:, 3]) / 2, b[:, 2] - b[:, 0], b[:, 3] - b[:, 1], b[:, 4]],
                    1).astype(np.float32)


def randomize_bn_(model, seed=0):
    """Random running stats / affine so BN folding is exercised (mean~N(0,.1), var~U[.5,1.5])."""
    import torch

    g = torch.Generator().manual_seed(seed)
    for m in model.modules():
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=g) * 0.1)
            m.running_var.copy_(torch.rand(m.running_var.shape, generator=g) + 0.5)
            if m.weight is not None:
                m.weight.data.copy_(1.0 + 0.2 * torch.randn(m.weight.shape, generator=g))
                m.bias.data.copy_(0.1 * torch.randn(m.bias.shape, generator=g))
    return model


def variance_preserving_init_(model, seed=0, sparse_fan_in_taps=6.0):
    """He-style re-initialisation so that random-weight activations keep O(1) variance through the
    sparse encoder and the RPN (the default inits shrink the signal to a spatially constant map, which
    would leave NMS with ~70k tied scores -- a degenerate benchmark workload)."""
    import torch

    g = torch.Generator().manual_seed(seed)
    for m in model.modules():
        w = getattr(m, "weight", None)
        if w is None or w.dim() < 4:
            continue
        if w.dim() == 5:                      # sparse conv [kd,kh,kw,Cin,Cout]: only a few taps are occupied
            k = w.shape[0] * w.shape[1] * w.shape[2]
            fan_in = w.shape[3] * min(float(k), sparse_fan_in_taps)
        else:                                 # Conv2d / ConvTranspose2d [Cout,Cin,kh,kw]
            fan_in = w.shape[1] * w.shape[2] * w.shape[3]
        with torch.no_grad():
            w.copy_(torch.randn(w.shape, generator=g) * (2.0 / fan_in) ** 0.5)
    return model


def demo_weights_(model, seed=0, cls_scale=0.005, cls_bias=-1.05, box_scale=0.005):
    """Random-init weights of the configured architecture that give a *non-degenerate* detection
    workload (no checkpoints exist offline): variance-preserving conv init, random BN statistics, and
    head scales calibrated (on 20k-point lidar-like clouds, CPU oracle) so that ~3 % of the anchors pass
    the 0.3 score threshold with well-spread scores and finite decoded boxes."""
    import torch

    variance_preserving_init_(model, seed)
    randomize_bn_(model, seed)
    with torch.no_grad():
        for m in model.modules():          # residual blocks: damp the branch so activations stay O(1..10)
            if hasattr(m, "bn2") and hasattr(m, "conv2"):
                m.bn2.weight.mul_(0.25)
        for task in model.bbox_head.tasks:
            task.conv_cls.weight.mul_(cls_scale)
            task.conv_cls.bias.fill_(cls_bias)
            task.conv_box.weight.mul_(box_scale)
            task.conv_box.bias.zero_()
    return model


def calibrate_demo_weights_(model, cfg, clouds, seed=0, pass_fraction=0.03, box_std=0.1):
    """Data-driven finish of `demo_weights_` (GPU): makes the random-weight network behave like a trained one --
    every BatchNorm's running statistics are set from the activations it actually sees (then perturbed, so folding a
    non-trivial mean / variance is still exercised), which keeps features O(1) through all ~22 layers, and the heads
    are scaled so that `pass_fraction` of the anchors clear the score threshold with spread-out scores.

    Why: with random running statistics the features of `demo_weights_` grow to ~1e3 by the last layer, where fp32
    itself resolves only ~1e-4 -- the north_star's "1e-4 abs on float features" is only a meaningful bar for O(1)
    features, which is what trained BatchNorm layers produce.  One streaming pass through the layer-by-layer module path
    (forward pre-hooks on the BN modules, upstream layers already calibrated when a layer is reached)."""
    import torch

    from det3d_b200.ops.point_cloud.voxelize import Voxelizer

    assert torch.cuda.is_available(), "calibrate_demo_weights_ streams activations through the CUDA module path"
    dev = torch.device("cuda")
    model.to(dev).eval()
    g = torch.Generator().manual_seed(seed + 12345)
    hooks = []

    def pre_hook(bn, args):
        x = args[0].detach().float()
        if x.numel() == 0:
            return
        dims = [d for d in range(x.dim()) if d != 1]
        mean = x.mean(dim=dims)
        var = x.var(dim=dims, unbiased=False).clamp_min(1e-3)
        c = mean.shape[0]
        bn.running_mean.copy_(mean + 0.1 * var.sqrt() * torch.randn(c, generator=g).to(dev))
        bn.running_var.copy_(var * (0.8 + 0.45 * torch.rand(c, generator=g).to(dev)))
        if not getattr(bn, "_d3b_gamma_scaled", False):     # trained gammas sit below 1: keeps the activations' tails within ~10
            bn.weight.mul_(0.6)
            bn._d3b_gamma_scaled = True

    for m in model.modules():
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            hooks.append(m.register_forward_pre_hook(pre_hook))
    vg = cfg.voxel_generator
    takes_points = cfg.model["reader"]["type"] != "VoxelFeatureExtractorV3"
    vox = Voxelizer(vg["voxel_size"], vg["range"], vg["max_points_in_voxel"], vg["max_voxel_num"], want_voxels=takes_points,
                    want_mean=not takes_points)
    offsets = [0]
    for c in clouds:
        offsets.append(offsets[-1] + c.shape[0])
    pts = torch.from_numpy(np.concatenate(clouds)).to(dev)
    out = vox(pts, offsets)
    batch = len(clouds)
    m_rows = int(out["counts"][batch])
    coors = out["coors"][:m_rows]
    grid = [int(v) for v in vox.grid_size]
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            if takes_points:
                feats = model.reader.forward_torch(out["voxels"][:m_rows], out["num_points"][:m_rows], coors)
                x = model.backbone(feats.reshape(m_rows, -1), coors, batch, grid)
            else:
                # the reader's leading columns (Lyft: 3 of the 4 point columns)
                c = int(cfg.model["reader"].get("num_input_features", out["mean"].shape[1]))
                x = model.backbone.forward_unfused(out["mean"][:m_rows, :c].clone(), coors, batch, grid)
            if getattr(model, "with_neck", False):
                x = model.neck(x)
            thr = float(cfg.test_cfg["score_threshold"])
            for task in model.bbox_head.tasks:
                logit = task.conv_cls(x)
                # realistic logit range: the 99.99 % quantile of |logit - mean| lands on 6 (sigmoid(6) = 0.9975)
                dev_abs = (logit.float() - logit.float().mean()).abs().reshape(-1)
                spread = dev_abs.kthvalue(max(1, int(dev_abs.numel() * 0.9999)))[0]
                task.conv_cls.weight.mul_(6.0 / spread.clamp_min(1e-6))
                task.conv_cls.bias.zero_()
                logit = task.conv_cls(x)
                best = logit.float().amax(dim=1).reshape(-1) if logit.shape[1] > 1 else logit.float().reshape(-1)
                # the (1 - pass_fraction) quantile of the best logit lands on the score threshold
                k = max(1, int(best.numel() * (1.0 - pass_fraction)))
                q = best.kthvalue(k)[0]
                task.conv_cls.bias.fill_(float(np.log(thr / (1.0 - thr)) - q))
                box = task.conv_box(x)
                task.conv_box.weight.mul_(box_std / box.std().clamp_min(1e-6))
                task.conv_box.bias.zero_()
                if getattr(task, "use_dir", False):
                    d = task.conv_dir(x).float().abs().reshape(-1)
                    task.conv_dir.weight.mul_(6.0 / d.kthvalue(max(1, int(d.numel() * 0.9999)))[0].clamp_min(1e-6))
                    task.conv_dir.bias.zero_()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
        for h in hooks:
            h.remove()
    return model


def raw_velodyne_scan(n=120000, ndim=4, seed=0, max_range=120.0):
    """A full 360° scan of a 64-beam spinning LiDAR, KITTI-style: no range or field-of-view crop, ordered beam by beam
    and by azimuth within a beam (as a raw velodyne file).  Beams at -24.8° .. +2° elevation from 1.73 m above the
    ground hit the ground or (35 %) an obstacle at 2 m .. max_range; rays that hit nothing within max_range are dropped,
    so the scan holds about n points (n / 64 azimuth steps per beam)."""
    rng = np.random.default_rng(seed)
    per_beam = max(int(n) // 64, 1)
    beam = np.repeat(np.arange(64), per_beam)
    elev = np.deg2rad(-24.8 + beam * (26.8 / 63.0)) + rng.normal(0, 1e-3, beam.shape[0])
    azim = np.tile(np.linspace(-np.pi, np.pi, per_beam, endpoint=False), 64) + rng.normal(0, 1e-4, beam.shape[0])
    h = 1.73
    with np.errstate(divide="ignore"):
        ground_d = np.where(elev < -1e-3, h / np.tan(-elev), np.inf)
    obst = rng.uniform(0, 1, beam.shape[0]) < 0.35
    obst_d = rng.uniform(2.0, max_range, beam.shape[0])
    d = np.where(obst, np.minimum(obst_d, ground_d), ground_d)
    ok = d < max_range
    z = -h + np.where(obst & (obst_d < ground_d), rng.uniform(0, 2.5, beam.shape[0]), 0.0) + rng.normal(0, 0.02, beam.shape[0])
    pts = np.zeros((int(ok.sum()), ndim), np.float32)
    pts[:, 0], pts[:, 1], pts[:, 2] = (d * np.cos(azim))[ok], (d * np.sin(azim))[ok], z[ok]
    if ndim > 3:
        pts[:, 3] = rng.uniform(0, 1, pts.shape[0])
    return pts


KITTI_IMAGE_SHAPES = ((375, 1242), (370, 1224), (374, 1238), (376, 1241))


def kitti_like_calib(seed=0, image_shape=(375, 1242), perturb=True):
    """A synthetic KITTI calibration in the info files' form: dict(rect, Trv2c, P2, image_shape), 4x4 float64 matrices.
    P2 = K [I | t] with KITTI-like intrinsics (f ≈ 721.5, c ≈ (609.6, 172.9)) and P2[:, 3] ≈ (44.86, 0.216, 0.0027);
    R0_rect a small rotation; Tr_velo_to_cam the velodyne -> camera axis permutation times a small rotation, plus a
    translation of about (-0.004, -0.076, -0.27).  `perturb` adds seeded jitter to every parameter."""
    rng = np.random.default_rng(seed)
    j = (lambda s: rng.normal(0, s)) if perturb else (lambda s: 0.0)

    def rot(ax, ay, az):
        cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
        return (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
                @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]))

    f = 721.5377 * (1 + j(0.01))
    K = np.array([[f, 0, 609.5593 + j(3.0)], [0, f, 172.854 + j(3.0)], [0, 0, 1.0]])
    t = np.linalg.solve(K, np.array([44.85728 + j(0.5), 0.2163791 + j(0.01), 0.002745884 + j(1e-4)]))
    P2 = np.eye(4)
    P2[:3, :3], P2[:3, 3] = K, K @ t
    rect = np.eye(4)
    rect[:3, :3] = rot(0.0042 + j(0.002), -0.0099 + j(0.002), 0.0074 + j(0.002))
    axes = np.array([[0, -1.0, 0], [0, 0, -1.0], [1.0, 0, 0]])             # velodyne x fwd, y left, z up -> camera
    Trv2c = np.eye(4)
    Trv2c[:3, :3] = axes @ rot(j(0.01), j(0.01), j(0.01))
    Trv2c[:3, 3] = [-0.004069766 + j(0.002), -0.07631618 + j(0.005), -0.2717806 + j(0.01)]
    return dict(rect=rect, Trv2c=Trv2c, P2=P2, image_shape=np.array(image_shape, np.int64))
