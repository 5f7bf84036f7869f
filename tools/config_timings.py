"""Device timings of the other BASELINE.json configurations (they are parity-test cases, not bench lines; this is the
evidence table in profiles/).  CUDA events, 3 warm-up + 10 timed iterations, inputs resident in HBM.
    python tools/config_timings.py > profiles/r1_config_timings.md
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import det3d_b200  # noqa: E402,F401
from det3d.models import build_detector  # noqa: E402
from det3d.torchie import Config  # noqa: E402
from det3d_b200.apis import InferencePipeline  # noqa: E402
from det3d_b200.ops.iou3d import iou3d_utils  # noqa: E402
from det3d_b200.ops.point_cloud.voxelize import Voxelizer  # noqa: E402
from det3d_b200.utils.synthetic import demo_weights_, lidar_like_cloud, nms_boxes_xyxyr, uniform_cloud  # noqa: E402


def timed(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    rows = []
    kitti = dict(vs=[0.05, 0.05, 0.1], pcr=[0, -40.0, -3.0, 70.4, 40.0, 1.0])
    # C1: voxelizer only, 1k points
    vox = Voxelizer(kitti["vs"], kitti["pcr"], 5, 20000, want_voxels=True, want_mean=False)
    pts = torch.from_numpy(uniform_cloud(1000, kitti["pcr"], 4, 0)).cuda()
    rows.append(("C1 VoxelGenerator, 1k points, KITTI-car grid", "%.1f us / cloud" % (1e3 * timed(lambda: vox(pts, None))), "6 launches, latency bound"))
    pts20 = torch.from_numpy(lidar_like_cloud(20000, kitti["pcr"], 4, 0)).cuda()
    rows.append(("voxelizer, 20k lidar-like points", "%.1f us / cloud" % (1e3 * timed(lambda: vox(pts20, None))), ""))

    # C3: PointPillars B=8 x 20k (uniform clouds hit the 12000-pillar cap)
    cfg = Config.fromfile(os.path.join(ROOT, "configs", "pointpillars_kitti_car.py"))
    torch.manual_seed(0)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 0, cls_scale=0.3, cls_bias=-3.6, box_scale=0.02)
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    clouds = [uniform_cloud(20000, cfg.voxel_generator.range, 4, s) for s in range(8)]
    p8 = torch.from_numpy(np.concatenate(clouds)).cuda()
    off = [20000 * i for i in range(9)]
    ms = timed(lambda: pipe.pack(pipe.forward_device(p8, off)), iters=5)
    rows.append(("C3 PointPillars KITTI, 8 x 20k uniform points", "%.2f ms / batch = %.0f clouds/s" % (ms, 8e3 / ms),
                 "fused pillar reader + scatter; RPN [3,5,5] on cuDNN fp32; eager launches"))
    del pipe, model

    # C4: CBGS nuScenes, 4 clouds per GPU (32 over 8 GPUs), 35k points, 5 features
    cfg = Config.fromfile(os.path.join(ROOT, "configs", "cbgs_nusc.py"))
    torch.manual_seed(1)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), 1, cls_bias=-2.4)
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    clouds = [lidar_like_cloud(35000, cfg.voxel_generator.range, 5, s) for s in range(4)]
    p4 = torch.from_numpy(np.concatenate(clouds)).cuda()
    off = [35000 * i for i in range(5)]
    ms = timed(lambda: pipe.pack(pipe.forward_device(p4, off)), iters=5)
    rows.append(("C4 CBGS nuScenes (SpMiddleResNetFHD, 6 task heads), 4 x 35k lidar-like points per GPU", "%.2f ms / batch = %.0f clouds/s per GPU" % (ms, 4e3 / ms),
                 "21 sparse convs on the FP16x3 kernels (spconv_first16_kernel for the 5-channel input layer, "
                 "spconv_os16_kernel for the other 20); strided RPN2 on cuDNN fp32; eager launches"))
    del pipe, model

    # C5: rotated NMS stress, 100k boxes
    for kind, thr in (("uniform", 0.2), ("clustered", 0.2)):
        b, s = nms_boxes_xyxyr(100000, 0, clustered=(kind == "clustered"))
        bt, st = torch.from_numpy(b).cuda(), torch.from_numpy(s).cuda()
        ms = timed(lambda: iou3d_utils.nms_gpu(bt, st, thr), iters=3, warm=1)
        rows.append(("C5 iou3d NMS, 100k %s boxes, thr %.1f" % (kind, thr), "%.1f ms" % ms,
                     "%.2e pair tests/s; mask 1.25 GB stays on the device" % (100000 * 99999 / 2 / (ms * 1e-3))))

    print("# r1: timings of the other BASELINE configurations (H100, CUDA events, inputs resident)\n")
    print("| configuration | time | note |\n|---|---|---|")
    for r in rows:
        print("| %s | %s | %s |" % r)


if __name__ == "__main__":
    main()
