#!/usr/bin/env python
"""Clouds/s of live LiDAR streams: device-resident sweep histories (SweepStream) against re-sending every sweep.

CBGS (configs/cbgs_nusc.py) at B = 1 and B = 4 streams.  Every step each stream receives one new sweep of 30.6k–34k raw
records of 5 floats (a nuScenes LIDAR_TOP sweep; seeded lidar_like_clouds, sizes redrawn every step) under a seeded
sensor pose (yaw <= 0.05 rad, <= 1.5 m per step) 0.05 s after the previous one; a frame is the new sweep as the key frame
and the stream's 9 previous sweeps.  Modes, from host sweeps to detections in host memory:
  a  infer_sweeps(graphed=True) given the frame's 10 sweeps (all of them copied H2D every step)
  b  SweepStream.push() of the new sweeps + SweepStream.infer(graphed=True) (only the new sweeps and the table go H2D)
each with the sweeps as pinned tensors and as plain numpy arrays.  Steps are timed with CUDA events, the L2 flushed
before each, the four modes interleaved step by step after a warm-up that fills the histories and captures every graph;
the timed loop runs --runs times.  The detections of every step must be identical in the four modes; the run fails
otherwise.

    python tools/bench_sweep_stream.py --steps 20 --out profiles/h100_sweep_stream.json
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

MODES = ("all_sweeps_pinned", "all_sweeps_numpy", "stream_pinned", "stream_numpy")


def run(batch, steps, runs, warmup, n_sweep, history, pool, seed, cfg, model):
    import numpy as np
    import torch
    from det3d_b200.apis import InferencePipeline, SweepStream
    from det3d_b200.datasets.pipelines.loading import stream_transforms
    from det3d_b200.utils.synthetic import lidar_like_cloud

    pcr = cfg.voxel_generator.range
    # one pipeline per stream (a captured graph holds its stream's buffers) and one for mode a; the model is shared
    pipes = {m: InferencePipeline(cfg, model=model, device="cuda") for m in ("all_sweeps", "stream_pinned",
                                                                           "stream_numpy")}
    streams = {m: SweepStream(pipes[m], batch, history, n_sweep) for m in ("stream_pinned", "stream_numpy")}
    rng = np.random.default_rng(seed)
    base = [[lidar_like_cloud(n_sweep, pcr, 5, seed * 1000 + b * 64 + k) for k in range(pool)] for b in range(batch)]
    base_pinned = [[torch.from_numpy(c).pin_memory() for c in row] for row in base]
    n_steps = warmup + runs * steps
    sizes = rng.integers(int(0.9 * n_sweep), n_sweep + 1, (n_steps, batch))
    poses, times = np.zeros((n_steps, batch, 4, 4)), np.zeros((n_steps, batch))
    for b in range(batch):
        pose, t = np.eye(4), 1.6e9 + b
        for s in range(n_steps):
            a = rng.uniform(-0.05, 0.05)
            m = np.eye(4)
            m[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
            m[:2, 3] = rng.uniform(-1.5, 1.5, 2)
            pose, t = pose @ m, t + 0.05
            poses[s, b], times[s, b] = pose, t

    def sweep(s, b, pinned):           # the sweep stream b received at step s (leading rows of a pooled cloud)
        src = base_pinned if pinned else base
        return src[b][s % pool][:int(sizes[s, b])]

    def frame(s, pinned):
        out = []
        for b in range(batch):
            steps_back = range(s, max(s - history, -1), -1)          # newest first
            tms, lags = stream_transforms([poses[j, b] for j in steps_back], [times[j, b] for j in steps_back])
            out.append(([sweep(j, b, pinned) for j in steps_back], tms, lags))
        return out

    pinned_out = {m: None for m in MODES}
    push_s = {m: 0.0 for m in MODES}
    h2d = {m: 0 for m in MODES}

    def step(mode, s):
        pinned = mode.endswith("pinned")
        if mode.startswith("all_sweeps"):
            samples = frame(s, pinned)
            out = pipes["all_sweeps"].infer_sweeps(samples, pinned_out=pinned_out[mode], graphed=True)
            entry = next(e for k, e in pipes["all_sweeps"]._graphs.items() if len(k) == 5)
            h2d[mode] = sum(r.shape[0] * r.shape[1] * 4 for smp in samples for r in smp[0]) + entry.ingest.table.numel()
        else:
            st = streams[mode]
            t0 = time.perf_counter()
            for b in range(batch):
                st.push(b, sweep(s, b, pinned), poses[s, b], float(times[s, b]))
            push_s[mode] += time.perf_counter() - t0
            out = st.infer(pinned_out=pinned_out[mode], graphed=True)
            h2d[mode] = st.last_h2d_bytes
        pinned_out[mode] = out
        return out

    for s in range(warmup):
        for mode in MODES:
            step(mode, s)
    n_graphs = {m: len(p._graphs) for m, p in pipes.items()}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    equal, dets, results = True, 0, []
    torch.cuda.synchronize()
    for r in range(runs):
        ms = {m: 0.0 for m in MODES}
        wall = {m: 0.0 for m in MODES}
        h2d_sum = {m: 0 for m in MODES}
        for m in MODES:
            push_s[m] = 0.0
        for s in range(warmup + r * steps, warmup + (r + 1) * steps):
            outs = {}
            for k in range(len(MODES)):
                mode = MODES[(s + k) % len(MODES)]                  # rotate the order step by step
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0.record()
                out = step(mode, s)
                e1.record()
                e1.synchronize()
                wall[mode] += time.perf_counter() - t0
                ms[mode] += e0.elapsed_time(e1)
                h2d_sum[mode] += h2d[mode]
                outs[mode] = out.clone()
            equal &= all(torch.equal(outs[MODES[0]], outs[m]) for m in MODES[1:])
            dets += int((outs[MODES[0]][..., -1] > 0.5).sum())
        results.append({m: {"ms_per_step": ms[m] / steps, "clouds_per_s": steps * batch / (ms[m] * 1e-3),
                            "host_wall_ms_per_step": wall[m] * 1e3 / steps,
                            "h2d_bytes_per_step": h2d_sum[m] / steps,
                            **({"push_wall_ms_per_step": push_s[m] * 1e3 / steps} if m.startswith("stream") else {})}
                        for m in MODES})
    assert {m: len(p._graphs) for m, p in pipes.items()} == n_graphs, "a timed step captured a graph"
    return dict(batch=batch, steps_per_run=steps, runs=runs, warmup_steps=warmup,
                graphs_captured=n_graphs, detections_equal_every_step=bool(equal), detections=dets,
                results=results,
                speedup_stream_vs_all_sweeps={kind: [res["all_sweeps_" + kind]["ms_per_step"]
                                                     / res["stream_" + kind]["ms_per_step"] for res in results]
                                              for kind in ("pinned", "numpy")})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=12, help=">= the history, so the timed frames have full histories")
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--points-per-sweep", type=int, default=34000)
    ap.add_argument("--history", type=int, default=10, help="sweeps per frame, key frame included")
    ap.add_argument("--pool", type=int, default=12, help="distinct base clouds per stream")
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sweep_stream.py needs a CUDA device: det3d_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    import bench
    from bench_variable_clouds import card
    from det3d.torchie import Config

    wl = bench.WORKLOADS["cbgs"]
    cfg = Config.fromfile(os.path.join(ROOT, "configs", wl["cfg"]))
    model = bench.build_model(cfg, argparse.Namespace(config="cbgs", wl=wl, dist="lidar_like"))
    per_batch = [run(b, a.steps, a.runs, a.warmup, a.points_per_sweep, a.history, a.pool, a.seed, cfg, model)
                 for b in a.batches]
    result = dict(card(), what=__doc__.strip().splitlines()[0], config=wl["cfg"], sweeps_per_frame=a.history,
                  raw_points_per_sweep=[int(0.9 * a.points_per_sweep), a.points_per_sweep], raw_stride=5,
                  timing="CUDA events per step from host sweeps to host detections, L2 flushed before each, modes "
                         "interleaved; host_wall_ms_per_step is perf_counter over the same call",
                  detections_equal_every_step=all(r["detections_equal_every_step"] for r in per_batch),
                  per_batch=per_batch)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    ok = result["detections_equal_every_step"] and all(r["detections"] > 0 for r in per_batch)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
