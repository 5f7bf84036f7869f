#!/usr/bin/env python
"""Clouds/s from raw nuScenes-style sweeps to host detections: batched device-table ingest against one ingest per sample.

CBGS (configs/cbgs_nusc.py) at B = 4.  Each sample is a key frame and 9 sweeps of about N = 34k raw records of 5 floats
(a nuScenes LIDAR_TOP sweep): seeded lidar_like_clouds under seeded small rigid motions (yaw <= 0.1 rad, translation
<= 5 m), time lags 0.05 s apart, held in pinned host memory.  The sweep sizes of every step are drawn from [0.9 N, N],
so no two steps share a sweep table.  Modes, all from the pinned raw sweeps to the detections in host memory:
  a  per_sample   B x ingest_sweeps (one host round trip each) + concatenation + forward_graphed
  b  eager        infer_sweeps(graphed=False): one batched ingest, device cloud offsets, eager forward
  c  graphed      infer_sweeps(graphed=True): ingest, voxelize and forward replayed from one CUDA graph
Steps are timed with CUDA events, the L2 flushed before each, the three modes interleaved step by step after a warm-up
that captures every graph.  The detections of every step must be identical in the three modes; the run fails otherwise.

    python tools/bench_sweeps.py --steps 20 --out profiles/h100_sweeps.json
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

MODES = ("per_sample", "eager", "graphed")


def run(steps, batch, n_sweep, n_sweeps, warmup, seed):
    import numpy as np
    import torch
    import bench
    from bench_variable_clouds import card
    from det3d.torchie import Config
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.datasets.pipelines.loading import ingest_sweeps
    from det3d_b200.utils.synthetic import lidar_like_sweeps

    wl = bench.WORKLOADS["cbgs"]
    args = argparse.Namespace(config="cbgs", wl=wl, dist="lidar_like")
    cfg = Config.fromfile(os.path.join(ROOT, "configs", wl["cfg"]))
    pipe = InferencePipeline(cfg, model=bench.build_model(cfg, args), device="cuda")
    base = []
    for b in range(batch):
        raws, tms, lags = lidar_like_sweeps([n_sweep] * n_sweeps, cfg.voxel_generator.range, seed + b)
        base.append(([torch.from_numpy(r).pin_memory() for r in raws], tms, lags))
    rng = np.random.default_rng(seed)
    n_steps = warmup + steps
    sizes = rng.integers(int(0.9 * n_sweep), n_sweep + 1, (n_steps, batch, n_sweeps))
    # a step's sweeps are leading rows of the pinned base sweeps (slices of pinned memory are pinned)
    batches = [[([r[:int(n)] for r, n in zip(raws, sizes[s, b])], tms, lags) for b, (raws, tms, lags) in enumerate(base)]
               for s in range(n_steps)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    pinned_out = {m: None for m in MODES}

    def step(mode, samples):
        if mode == "per_sample":
            clouds = [ingest_sweeps(*s) for s in samples]              # one sync per sample
            offsets = np.cumsum([0] + [c.shape[0] for c in clouds]).tolist()
            packed = pipe.forward_graphed(torch.cat(clouds), offsets)
            if pinned_out[mode] is None:
                pinned_out[mode] = torch.empty(packed.shape, dtype=torch.float32, pin_memory=True)
            pinned_out[mode].copy_(packed, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            return pinned_out[mode]
        out = pipe.infer_sweeps(samples, pinned_out=pinned_out[mode], graphed=mode == "graphed")
        pinned_out[mode] = out
        return out

    for s in range(warmup):
        for mode in MODES:
            step(mode, batches[s])
    n_graphs = len(pipe._graphs)
    ms = {m: 0.0 for m in MODES}
    wall = {m: 0.0 for m in MODES}
    equal, dets = True, 0
    torch.cuda.synchronize()
    for s in range(warmup, n_steps):
        outs = {}
        for k in range(len(MODES)):
            mode = MODES[(s + k) % len(MODES)]                  # rotate the order step by step
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            e0.record()
            out = step(mode, batches[s])
            e1.record()
            e1.synchronize()
            wall[mode] += time.perf_counter() - t0
            ms[mode] += e0.elapsed_time(e1)
            outs[mode] = out.clone()
        equal &= all(torch.equal(outs["per_sample"], outs[m]) for m in MODES[1:])
        dets += int((outs["graphed"][..., -1] > 0.5).sum())
    assert len(pipe._graphs) == n_graphs, "a timed step captured a graph"
    totals = sizes[warmup:].sum(axis=(1, 2))
    tables = {tuple(x.ravel()) for x in sizes}
    res = {m: {"ms_per_step": ms[m] / steps, "clouds_per_s": steps * batch / (ms[m] * 1e-3),
               "wall_ms_per_step": wall[m] * 1e3 / steps} for m in MODES}
    return dict(card(), what=__doc__.strip().splitlines()[0], config=wl["cfg"], batch=batch, sweeps_per_sample=n_sweeps,
                raw_points_per_sweep=[int(0.9 * n_sweep), n_sweep], raw_stride=5, steps=steps, warmup_steps=warmup,
                distinct_tables=len(tables), raw_total_range=[int(totals.min()), int(totals.max())],
                graphs_captured=n_graphs, graph_keys=[list(k) for k in pipe._graphs],
                timing="CUDA events per step from pinned raw sweeps to host detections, L2 flushed before each, modes "
                       "interleaved", detections_equal_all_modes=bool(equal), detections=dets, modes=res,
                speedup_eager_vs_per_sample=res["per_sample"]["ms_per_step"] / res["eager"]["ms_per_step"],
                speedup_graphed_vs_per_sample=res["per_sample"]["ms_per_step"] / res["graphed"]["ms_per_step"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--points-per-sweep", type=int, default=34000)
    ap.add_argument("--sweeps", type=int, default=10, help="per sample, key frame included")
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sweeps.py needs a CUDA device: det3d_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    result = run(a.steps, a.batch, a.points_per_sweep, a.sweeps, a.warmup, a.seed)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    sys.exit(0 if result["detections_equal_all_modes"] and result["detections"] > 0 else 1)


if __name__ == "__main__":
    main()
