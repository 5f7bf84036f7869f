#!/usr/bin/env python
"""FP16x3 (the default) against single-pass FP16 (`set_math("fp16")`) on one GPU: clouds/s of the whole forward and the
in-graph stage times, for SECOND KITTI car (B = 1), PointPillars KITTI car (B = 8) and CBGS nuScenes (B = 4).

    python tools/bench_math.py [--steps 20] [--warmup 5] [--runs 2] [--out profiles/h100_math.json]

bench.py's method: seeded synthetic clouds resident on the device, the forward replayed from a CUDA graph, L2 flushed
(256 MiB write) before every step, CUDA events around each step, warm-up first.  Both maths run the same calibrated
weights on the same clouds in one process, alternating, `--runs` times each.  The in-graph stage times come from a
second capture with an event at every stage boundary (bench.py's in-graph pass), replayed with L2 flushed.  The card's
name, power limit and maximum SM clock are read in the same call.  Writes one JSON line per config to --out.
"""
import argparse
import copy
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_pillars_nusc import gpu_info  # noqa: E402

MATHS = ("fp16x3", "fp16")
N_POOL = 8
CONFIGS = {
    # name: (config file, batch, points per cloud, point features, seed, calibration pass fraction)
    "second": ("second_kitti_car.py", 1, 20000, 4, 0, None),
    "pillars": ("pointpillars_kitti_car.py", 8, 20000, 4, 0, 0.02),
    "cbgs": ("cbgs_nusc.py", 4, 35000, 5, 1, 0.01),
}


def bench_config(name, args, gpu):
    import numpy as np
    import torch
    from det3d.models import build_detector
    from det3d.torchie import Config
    from det3d_b200 import _lib
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import calibrate_demo_weights_, demo_weights_, lidar_like_cloud

    fname, B, n_pts, nf, seed, pf = CONFIGS[name]
    dev = torch.device("cuda", 0)
    cfg = Config.fromfile(os.path.join(ROOT, "configs", fname))
    r = cfg.voxel_generator.range
    torch.manual_seed(seed)
    model = demo_weights_(build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg).eval(), seed)
    calibrate_demo_weights_(model, cfg, [lidar_like_cloud(n_pts, r, nf, 777 + i) for i in range(2)], seed,
                            **({} if pf is None else {"pass_fraction": pf}))
    pipes = {}
    for m in MATHS:
        pipes[m] = InferencePipeline(cfg, model=copy.deepcopy(model), device=dev)
        pipes[m].set_math(m)
    resident = [torch.from_numpy(lidar_like_cloud(n_pts, r, nf, 1000 + i)).to(dev) for i in range(N_POOL)]
    dev_pts = torch.empty((B * n_pts, nf), dtype=torch.float32, device=dev)
    off = [n_pts * j for j in range(B + 1)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def load(step):
        for j in range(B):
            dev_pts[off[j]:off[j + 1]].copy_(resident[(step * B + j) % N_POOL], non_blocking=True)
        return dev_pts, off

    def timed(m, steps):
        pipe = pipes[m]
        evs = []
        torch.cuda.synchronize()
        for s in range(steps):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            pts, o = load(s)
            pipe.forward_graphed(pts, o)
            b.record()
            evs.append((a, b))
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in evs)

    for m in MATHS:
        timed(m, max(args.warmup, 3))
    for m in MATHS:
        if int(pipes[m].overflow_flag().item()) or pipes[m].model.math != m:
            raise SystemExit("%s: the %s kernels flagged an f16-range overflow on the synthetic workload" % (name, m))
    runs = {m: [] for m in MATHS}
    for _ in range(args.runs):
        for m in MATHS:
            runs[m].append(B * args.steps / (timed(m, args.steps) * 1e-3))

    stages = {}
    for m in MATHS:
        pipe, graph_ms, n_rep = pipes[m], {}, args.steps + 2
        pipe._graphs.clear()
        _lib.GRAPH_MARKS = marks = []
        try:
            for s in range(n_rep):
                pts, o = load(0)
                flush.zero_()
                pipe.forward_graphed(pts, o)
                torch.cuda.synchronize()
                if s >= 2:
                    for (tag, ev, _st), (_t1, ev1, _s1) in zip(marks[:-1], marks[1:]):
                        graph_ms[tag] = graph_ms.get(tag, 0.0) + ev.elapsed_time(ev1) / (n_rep - 2)
        finally:
            _lib.GRAPH_MARKS = None
            pipe._graphs.clear()
        stages[m] = graph_ms

    med = {m: statistics.median(runs[m]) for m in MATHS}
    return {
        "metric": "point-clouds/sec %s forward, fp16x3 vs single-pass fp16" % fname, "config": "configs/" + fname,
        "batch": B, "points_per_cloud": n_pts, "steps": args.steps, "warmup": max(args.warmup, 3), "runs": args.runs,
        "clouds_per_s": runs, "median_clouds_per_s": med, "speedup_fp16_over_fp16x3": med["fp16"] / med["fp16x3"],
        "stage_ms_per_step_in_graph": stages,
        "method": "graph replay, inputs resident on the device, L2 flushed (256 MiB write) before every step, CUDA events "
                  "around each step; the two maths alternate in one process on the same seeded clouds and weights",
        "gpu": gpu, "data": "synthetic",
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_math.json"))
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_math.py needs a CUDA device")
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
