#!/usr/bin/env python
"""SECOND KITTI three-class (configs/second_kitti_all.py) and CBGS Lyft (configs/cbgs_lyft.py) on one GPU: clouds/s of
the whole forward with the RPN and heads on the FP16x3 BEV kernels, against the same model with `use_fused_bev = False`
(RPN and heads through the torch modules on cuDNN fp32, `allow_tf32 = False`), and the in-graph stage times.

    python tools/bench_stock_more.py [--steps 20] [--warmup 5] [--runs 3] [--out profiles/h100_bench_stock_more.json]

bench.py's method: seeded synthetic clouds resident on the device, the forward replayed from a CUDA graph, L2 flushed
(256 MiB write) before every step, CUDA events around each step, warm-up first.  KITTI three-class: B = 2 LiDAR-like
clouds of 20k points.  Lyft: B = 2 clouds of 60k-100k LiDAR-like points over the +-100.8 m range.  The two paths run in
the same process, alternating, `--runs` times each, on the same clouds.  The in-graph stage times come from a second
capture with an event at every stage boundary (bench.py's in-graph pass), replayed with L2 flushed.  The card's name,
power limit and maximum SM clock are read in the same call.  Writes one JSON line per config to --out and prints them.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_pillars_nusc import gpu_info, near_ties, unmatched  # noqa: E402

B = 2
N_POOL = 6
CONFIGS = {
    # name: (config file, points per cloud (lo, hi), calibration points, seed, pass fraction, metric label)
    "second_kitti_all": ("second_kitti_all.py", (20000, 20000), 20000, 0, 0.03,
                         "SECOND kitti_all_vfev3_spmiddlefhd_rpn1_mghead (Car, Pedestrian, Cyclist) forward, 20k synthetic "
                         "pts, batch=2"),
    "cbgs_lyft": ("cbgs_lyft.py", (60000, 100000), 80000, 1, 0.01,
                  "CBGS lyft_all_vfev3_spmiddleresnetfhd_rpn2_mghead forward, 60k-100k synthetic pts, batch=2"),
}


def build_model(cfg, n_calib, seed, pass_fraction):
    import torch
    from det3d.models import build_detector
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud
    torch.manual_seed(seed)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), seed)
    calibrate_demo_weights_(model, cfg, [lidar_like_cloud(n_calib, cfg.voxel_generator.range, 4, 777 + i)
                                         for i in range(2)], seed, pass_fraction=pass_fraction)
    return model


def bench_config(name, args, gpu):
    import numpy as np
    import torch
    from det3d.torchie import Config
    from det3d_b200 import _lib
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import lidar_like_cloud

    fname, (n_lo, n_hi), n_calib, seed, pf, label = CONFIGS[name]
    dev = torch.device("cuda", 0)
    cfg = Config.fromfile(os.path.join(ROOT, "configs", fname))
    model = build_model(cfg, n_calib, seed, pf)
    pipes = {"fused": InferencePipeline(cfg, model=model, device=dev), "cudnn": InferencePipeline(cfg, model=model, device=dev)}
    model = pipes["fused"].model
    assert type(model.fused_bev()).__name__ == "FusedBevStack"
    rng = np.random.default_rng(42)
    sizes = [int(rng.integers(n_lo, n_hi + 1)) for _ in range(N_POOL)]
    clouds = [lidar_like_cloud(n, cfg.voxel_generator.range, 4, 1000 + i) for i, n in enumerate(sizes)]
    resident = [torch.from_numpy(c).to(dev) for c in clouds]
    cap = 2 * n_hi
    dev_pts = torch.empty((cap, 4), dtype=torch.float32, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def batch(step):
        ids = [(step * B + j) % N_POOL for j in range(B)]
        return ids, np.cumsum([0] + [sizes[i] for i in ids]).tolist()

    def load(step):
        ids, off = batch(step)
        for j, i in enumerate(ids):
            dev_pts[off[j]:off[j + 1]].copy_(resident[i], non_blocking=True)
        return dev_pts[:off[-1]], off

    def use(mode):
        model.use_fused_bev = mode == "fused"         # read by fused_bev() while a graph is captured, not at replay

    def timed(mode, steps):
        use(mode)
        pipe = pipes[mode]
        evs = []
        torch.cuda.synchronize()
        for s in range(steps):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            pts, off = load(s)
            pipe.forward_graphed(pts, off)
            b.record()
            evs.append((a, b))
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in evs)

    for mode in ("fused", "cudnn"):
        timed(mode, max(args.warmup, 3))
    if int(pipes["fused"].overflow_flag().item()):
        raise SystemExit("%s: the FP16x3 kernels flagged an f16-range overflow on the synthetic workload" % name)
    runs = {"fused": [], "cudnn": []}
    for _ in range(args.runs):
        for mode in ("fused", "cudnn"):
            runs[mode].append(B * args.steps / (timed(mode, args.steps) * 1e-3))

    # the two paths' detections on the same batch, near-ties counted on the fused head scores
    pts, off = load(0)
    dets = {}
    for mode in ("fused", "cudnn"):
        use(mode)
        dets[mode] = pipes[mode].unpack(pipes[mode].forward_graphed(pts, off).cpu())
    use("fused")
    pipe = pipes["fused"]
    with torch.no_grad():
        vox = pipe.voxelizer(pts, off)
        planes = model.backbone.forward_planes(model.reader(vox["mean"], None), vox["coors"], B,
                                               [int(g) for g in pipe.grid_size], n_dev=vox["counts"][B:B + 1])
        cls = [p["cls_preds"].clone() for p in model.fused_bev().run(planes)]
    thr, pre = cfg.test_cfg.score_threshold, cfg.test_cfg.nms.nms_pre_max_size
    agreement = []
    for b in range(B):
        f, c = dets["fused"][b]["box3d_lidar"], dets["cudnn"][b]["box3d_lidar"]
        agreement.append({"fused": int(f.shape[0]), "cudnn": int(c.shape[0]), "missing": unmatched(c, f),
                          "extra": unmatched(f, c), "near_ties": near_ties(cls, b, thr, pre)})
    agree = all(a["missing"] <= a["near_ties"] and a["extra"] <= a["near_ties"] for a in agreement)

    # in-graph stage times: a second capture with an event at every stage boundary, replayed with L2 flushed
    graph_ms, n_rep = {}, args.steps + 2
    pipe._graphs.clear()
    _lib.GRAPH_MARKS = marks = []
    try:
        for s in range(n_rep):
            pts, off = load(0)
            flush.zero_()
            pipe.forward_graphed(pts, off)
            torch.cuda.synchronize()
            if s >= 2:
                for (tag, ev, _st), (_t1, ev1, _s1) in zip(marks[:-1], marks[1:]):
                    graph_ms[tag] = graph_ms.get(tag, 0.0) + ev.elapsed_time(ev1) / (n_rep - 2)
    finally:
        _lib.GRAPH_MARKS = None
        pipe._graphs.clear()

    value = statistics.median(runs["fused"])
    return {
        "metric": "point-clouds/sec " + label, "config": "configs/" + fname, "value": value, "unit": "clouds/s",
        "n_gpus": 1, "batch": B, "points_per_cloud": sizes, "steps": args.steps, "warmup": max(args.warmup, 3),
        "runs": args.runs, "ms_per_step": 1e3 * B / value,
        "runs_clouds_per_s": {"fp16x3_bev_kernels": runs["fused"], "cudnn_fp32_use_fused_bev_false": runs["cudnn"]},
        "speedup_vs_cudnn_median": value / statistics.median(runs["cudnn"]),
        "stage_ms_per_step_in_graph": graph_ms,
        "method": "graph replay, inputs resident on the device, L2 flushed (256 MiB write) before every step, CUDA events "
                  "around each step; the two paths alternate in one process on the same seeded clouds",
        "detections_agree": agree, "agreement_per_sample": agreement,
        "gpu": gpu, "dtype": "f32", "data": "synthetic",
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bench_stock_more.json"))
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_stock_more.py needs a CUDA device")
    torch.cuda.set_device(0)
    gpu = gpu_info()
    lines = [bench_config(name, args, gpu) for name in args.configs.split(",")]
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
        for line in lines:
            fh.write(json.dumps(line) + "\n")
    for line in lines:
        print(json.dumps(line))


if __name__ == "__main__":
    main()
