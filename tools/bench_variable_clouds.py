#!/usr/bin/env python
"""Clouds/s on frames of varying size: graph replay against eager launches.

Real LiDAR frames rarely repeat a point count.  Each config runs at bench.py's batch on seeded lidar-like clouds whose
point counts are drawn uniformly from [0.6 N, N] (N = bench.py's points per cloud), and every step is timed like
bench.py's: CUDA events around the step, L2 flushed before it, every batch shape warmed up first.  Modes:
  graph      forward_graphed: one CUDA graph per (batch, point-capacity bucket), device offsets
  eager      pack(forward_device(...)): every kernel launched from the host
  e2e_graph  infer_host(pinned clouds, graphed=True): H2D, graph replay, D2H of the detections
  e2e_eager  infer_host(pinned clouds)
The detections of every step must be identical across the four modes; the run fails otherwise.

    python tools/bench_variable_clouds.py --steps 40 --out profiles/h100_variable_clouds.json
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"gpu": None, "power_limit": None}


def run_config(name, steps, pool, seed):
    import numpy as np
    import torch
    import bench
    from det3d.torchie import Config
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import lidar_like_cloud

    wl = bench.WORKLOADS[name]
    args = argparse.Namespace(config=name, wl=wl, dist="lidar_like")
    cfg = Config.fromfile(os.path.join(ROOT, "configs", wl["cfg"]))
    pipe = InferencePipeline(cfg, model=bench.build_model(cfg, args), device="cuda")
    B, N, ND = wl["batch"], wl["n_points"], wl["ndim"]
    rng = np.random.default_rng(seed)
    sizes = rng.integers(int(0.6 * N), N + 1, (pool, B))
    batches = []
    for k in range(pool):
        clouds = [lidar_like_cloud(int(n), cfg.voxel_generator.range, ND, seed + 100 * k + j) for j, n in enumerate(sizes[k])]
        offsets = np.cumsum([0] + [c.shape[0] for c in clouds]).tolist()
        batches.append(dict(offsets=offsets, dev=torch.from_numpy(np.concatenate(clouds)).cuda(),
                            pinned=[torch.from_numpy(c).pin_memory() for c in clouds]))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    out_pinned = None

    def device_step(mode, b):
        if mode == "graph":
            return pipe.forward_graphed(b["dev"], b["offsets"])
        return pipe.pack(pipe.forward_device(b["dev"], b["offsets"]))

    def host_step(mode, b):
        return pipe.infer_host(b["pinned"], pinned_out=out_pinned, graphed=mode == "e2e_graph")

    def timed(mode):
        fn = host_step if mode.startswith("e2e") else device_step
        outs, ms = [], 0.0
        torch.cuda.synchronize()
        for s in range(steps):
            b = batches[s % pool]
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            packed = fn(mode, b)
            e1.record()
            e1.synchronize()
            ms += e0.elapsed_time(e1)
            outs.append(packed.cpu().clone())
        return ms, outs

    modes = ("graph", "eager", "e2e_graph", "e2e_eager")
    for mode in modes:                       # warm-up: every batch shape, every graph captured before the clock
        for b in batches:
            p = device_step(mode, b) if not mode.startswith("e2e") else host_step(mode, b)
            if mode.startswith("e2e") and out_pinned is None:
                out_pinned = p
    n_graphs = len(pipe._graphs)
    buckets = sorted({pipe.bucket_of(b["offsets"][-1]) for b in batches})
    res, outs = {}, {}
    for mode in modes:
        ms, outs[mode] = timed(mode)
        res[mode] = {"ms_per_step": ms / steps, "clouds_per_s": steps * B / (ms * 1e-3)}
    equal = all(torch.equal(outs["graph"][s], outs[m][s]) for m in modes[1:] for s in range(steps))
    dets = sum(int((o[..., -1] > 0.5).sum()) for o in outs["graph"])
    assert len(pipe._graphs) == n_graphs, "a timed step captured a graph"
    return {"config": name, "batch": B, "points_per_cloud": [int(0.6 * N), N], "distinct_batches": pool, "steps": steps,
            "total_points_range": [int(sizes.sum(1).min()), int(sizes.sum(1).max())], "buckets": buckets,
            "graphs_captured": n_graphs, "detections_equal_all_modes": equal, "detections": dets,
            "modes": res, "graph_speedup_device": res["eager"]["ms_per_step"] / res["graph"]["ms_per_step"],
            "graph_speedup_e2e": res["e2e_eager"]["ms_per_step"] / res["e2e_graph"]["ms_per_step"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="second,pillars,cbgs")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--pool", type=int, default=8, help="distinct seeded batches cycled through the steps")
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_variable_clouds.py needs a CUDA device: det3d_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    result = dict(card(), what=__doc__.strip().splitlines()[0], timing="CUDA events per step, L2 flushed before each",
                  configs=[run_config(c, a.steps, a.pool, a.seed) for c in a.configs.split(",")])
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    ok = all(c["detections_equal_all_modes"] and c["detections"] > 0 for c in result["configs"])
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
