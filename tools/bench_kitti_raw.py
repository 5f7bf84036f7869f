#!/usr/bin/env python
"""Clouds/s from raw KITTI velodyne scans to host detections: the camera-frustum crop on the host against the crop on the
device inside the replayed graph.

SECOND car (configs/second_kitti_car.py) at B = 1 and PointPillars KITTI (configs/pointpillars_kitti_car.py) at B = 8.
Every scan is a full 360° 64-beam scan (utils/synthetic.raw_velodyne_scan, about 111k points of 4 floats, no crop),
held in pinned host memory; its size varies from step to step.  Each slot of the batch has its own synthetic KITTI
calibration (a drive), fixed over the run.  Modes, both from the pinned raw scans to the detections in host memory:
  a  host_crop  the crop on the host (the plane test in float64 numpy, in the reference's order; planes computed once
                per calibration), then infer_host(graphed=True) on the cropped clouds
  b  infer_raw  infer_raw(graphed=True): crop, voxelize and forward replayed from one CUDA graph
Steps are timed with CUDA events, the L2 flushed before each, the modes interleaved step by step after a warm-up that
captures every graph.  The detections of every step must be identical in both modes; the run fails otherwise.  A second
pass replays the infer_raw graph with external timing events at its stage boundaries and reports the crop's time inside
the graph.

    python tools/bench_kitti_raw.py --steps 20 --out profiles/h100_kitti_raw.json
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

MODES = ("host_crop", "infer_raw")
CONFIGS = {"second": 1, "pillars": 8}


def host_crop(points, planes):
    """The reference's plane test on the host: s = ((x*n0 + y*n1) + z*n2) + d in float64, dropped when s >= 0."""
    import numpy as np
    x, y, z = (points[:, j].astype(np.float64) for j in range(3))
    keep = np.ones(points.shape[0], bool)
    for n0, n1, n2, d in planes:
        keep &= ~(((x * n0 + y * n1) + z * n2) + d >= 0)
    return points[keep]


def run(config, batch, n_scan, steps, warmup, seed):
    import numpy as np
    import torch
    import bench
    from bench_variable_clouds import card
    from det3d.torchie import Config
    from det3d_b200 import _lib
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import KITTI_IMAGE_SHAPES, kitti_like_calib, raw_velodyne_scan

    wl = bench.WORKLOADS[config]
    args = argparse.Namespace(config=config, wl=wl, dist="lidar_like")
    cfg = Config.fromfile(os.path.join(ROOT, "configs", wl["cfg"]))
    pipe = InferencePipeline(cfg, model=bench.build_model(cfg, args), device="cuda")
    calibs = [kitti_like_calib(seed + b, KITTI_IMAGE_SHAPES[b % 4]) for b in range(batch)]
    pool = [torch.from_numpy(raw_velodyne_scan(n_scan, 4, seed=seed * 100 + i)).pin_memory() for i in range(2 * batch)]
    rng = np.random.default_rng(seed)
    n_steps = warmup + steps
    # a step's scans are leading rows of pinned pool scans (slices of pinned memory are pinned)
    frames = [[pool[int(rng.integers(len(pool)))][:int(rng.integers(int(0.9 * n_scan), n_scan))] for _ in range(batch)]
              for _ in range(n_steps)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    pinned_out = {m: None for m in MODES}

    def step(mode, scans):
        if mode == "host_crop":
            clouds = [torch.from_numpy(host_crop(s.numpy(), pipe.frustum_planes(c))) for s, c in zip(scans, calibs)]
            out = pipe.infer_host(clouds, pinned_out=pinned_out[mode], graphed=True)
        else:
            out = pipe.infer_raw(scans, calibs, pinned_out=pinned_out[mode], graphed=True)
        pinned_out[mode] = out
        return out

    for s in range(warmup):
        for mode in MODES:
            step(mode, frames[s])
    n_graphs = len(pipe._graphs)
    ms = {m: 0.0 for m in MODES}
    wall = {m: 0.0 for m in MODES}
    equal, dets, kept = True, 0, []
    torch.cuda.synchronize()
    for s in range(warmup, n_steps):
        outs = {}
        for k in range(len(MODES)):
            mode = MODES[(s + k) % len(MODES)]                  # alternate the order step by step
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0.record()
            out = step(mode, frames[s])
            e1.record()
            e1.synchronize()
            wall[mode] += time.perf_counter() - t0
            ms[mode] += e0.elapsed_time(e1)
            outs[mode] = out.clone()
        equal &= torch.equal(outs["host_crop"], outs["infer_raw"])
        dets += int((outs["infer_raw"][..., -1] > 0.5).sum())
    assert len(pipe._graphs) == n_graphs, "a timed step captured a graph"
    graph_keys = [list(k) for k in pipe._graphs]          # (the stage pass below recaptures and then drops them)
    for s in range(warmup, n_steps):
        kept += [host_crop(sc.numpy(), pipe.frustum_planes(c)).shape[0] for sc, c in zip(frames[s], calibs)]
    raw = [int(sc.shape[0]) for f in frames[warmup:] for sc in f]

    # in-graph stage times of the infer_raw graph (recaptured with timing events at its stage boundaries)
    graph_ms = {}
    pipe._graphs.clear()
    _lib.GRAPH_MARKS = marks = []
    try:
        n_rep = min(steps, 10) + 2
        for s in range(n_rep):
            flush.zero_()
            pipe.infer_raw(frames[warmup + s % steps], calibs, pinned_out=pinned_out["infer_raw"], graphed=True)
            torch.cuda.synchronize()
            if s >= 2:
                for (tag, ev, _st), (_t1, ev1, _s1) in zip(marks[:-1], marks[1:]):
                    graph_ms[tag] = graph_ms.get(tag, 0.0) + ev.elapsed_time(ev1) / (n_rep - 2)
    except RuntimeError as ex:            # (timing of externally recorded events unsupported)
        print("[bench_kitti_raw] in-graph stage pass unavailable: %s" % ex, file=sys.stderr)
    finally:
        _lib.GRAPH_MARKS = None
        pipe._graphs.clear()

    res = {m: {"ms_per_step": ms[m] / steps, "clouds_per_s": steps * batch / (ms[m] * 1e-3),
               "wall_ms_per_step": wall[m] * 1e3 / steps} for m in MODES}
    return dict(config=wl["cfg"], batch=batch, steps=steps, warmup_steps=warmup,
                raw_points_per_scan=[min(raw), max(raw)], kept_points_per_scan=[min(kept), max(kept)],
                graphs_captured=n_graphs, graph_keys=graph_keys,
                detections_equal_all_modes=bool(equal), detections=dets, modes=res,
                speedup_infer_raw_vs_host_crop=res["host_crop"]["ms_per_step"] / res["infer_raw"]["ms_per_step"],
                in_graph_stage_ms=graph_ms, crop_in_graph_ms=graph_ms.get("frustum_crop")), card()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--points-per-scan", type=int, default=120000)
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_kitti_raw.py needs a CUDA device: det3d_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    runs, card = [], None
    for config, batch in CONFIGS.items():
        r, card = run(config, batch, a.points_per_scan, a.steps, a.warmup, a.seed)
        runs.append(r)
    result = dict(card, what=" ".join(__doc__.strip().split("\n\n")[0].split()),
                  timing="CUDA events per step from pinned raw scans to host detections, L2 flushed before each, modes "
                         "interleaved", runs=runs)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    sys.exit(0 if all(r["detections_equal_all_modes"] and r["detections"] > 0 for r in runs) else 1)


if __name__ == "__main__":
    main()
