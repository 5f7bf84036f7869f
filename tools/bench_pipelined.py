#!/usr/bin/env python
"""Clouds/s of the serving entry points with frames in flight: blocking calls against block=False at max_in_flight 2
and 3, on the same frames, with every frame's output checked equal between the modes.

Workloads (calibrated demo weights as bench.py builds them; inputs in pinned host memory, a few input sets cycled, all
inside one capacity bucket so no timed frame captures a graph):
  host_second          infer_host(graphed=True), SECOND car, B = 1, 20k-point lidar-like clouds
  raw_kitti_second     infer_raw(graphed=True, kitti_results=True), SECOND car, B = 1, 110-125k-point raw scans
  raw_kitti_pillars    the same, PointPillars car, B = 8
  sweeps_nusc_cbgs     infer_sweeps(graphed=True, nusc_results=True), CBGS nuScenes, B = 4, 10 sweeps of 31-34k points
  stream_cbgs          SweepStream(history=10, in_flight=k).push per stream + infer(graphed=True), CBGS, B = 4, one
                       31-34k-point sweep per stream and frame (each mode replays the same pushes from a reset stream)
A run of a mode is `frames` frames, timed by host clock from the first submit to the last result() (L2 not flushed: a
steady stream).  The modes are interleaved round by round, after one untimed round that captures every graph.

    python tools/bench_pipelined.py --rounds 3 --out profiles/h100_pipelined.json
"""
import argparse
import collections
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DEPTHS = (1, 2, 3)                  # 1: blocking calls; k > 1: block=False at max_in_flight = k


def card():
    """The card's name, power limit and max SM clock, read in the same job as the numbers."""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"gpu": None, "power_limit": None, "max_sm_clock": None}


def same(a, b):
    """Equal outputs: packed tensors bit for bit; anno lists / dicts with equal keys, order, types and float bits."""
    import numpy as np
    import torch
    if type(a) is not type(b):
        return False
    if torch.is_tensor(a):
        return a.shape == b.shape and bool(torch.equal(a.view(torch.int32), b.view(torch.int32)))
    if isinstance(a, dict):
        return list(a) == list(b) and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    if isinstance(a, float):
        return np.float64(a).tobytes() == np.float64(b).tobytes()
    return a == b


def pipeline(config):
    import bench
    from det3d.torchie import Config
    from det3d_b200.apis import InferencePipeline
    wl = bench.WORKLOADS[config]
    cfg = Config.fromfile(os.path.join(ROOT, "configs", wl["cfg"]))
    model = bench.build_model(cfg, argparse.Namespace(config=config, wl=wl, dist="lidar_like"))
    return InferencePipeline(cfg, model=model, device="cuda")


def record(seed):
    from bench_nusc_results import record as nusc_record
    return nusc_record(seed)


def workloads(seed, n_sets=4):
    """name -> (pipe, batch, run(depth, frames) -> outputs), built lazily in order."""
    import numpy as np
    import torch
    from det3d_b200.apis import SweepStream
    from det3d_b200.utils.synthetic import (KITTI_IMAGE_SHAPES, kitti_like_calib, lidar_like_cloud, lidar_like_sweeps,
                                            raw_velodyne_scan)
    rng = np.random.default_rng(seed)
    pinned = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()          # noqa: E731

    def serve(pipe, submit):
        def run(depth, frames):
            if depth == 1:
                return [submit(f, True) for f in range(frames)]
            pipe.max_in_flight = depth
            handles = [submit(f, False) for f in range(frames)]
            out = [h.result() for h in handles]
            pipe.max_in_flight = 2
            return out
        return run

    def host_second():
        pipe = pipeline("second")
        pcr = pipe.cfg.voxel_generator.range
        sets = [[pinned(lidar_like_cloud(int(rng.integers(18000, 22000)), pcr, 4, seed + i))] for i in range(n_sets)]
        return pipe, 1, serve(pipe, lambda f, block: pipe.infer_host(sets[f % n_sets], graphed=True, block=block))

    def raw_kitti(config, batch):
        def make():
            pipe = pipeline(config)
            sets = []
            for i in range(n_sets):
                scans = [pinned(raw_velodyne_scan(int(rng.integers(110000, 125000)), 4, seed=seed + 50 * i + b))
                         for b in range(batch)]
                sets.append((scans, [kitti_like_calib(b % 3, KITTI_IMAGE_SHAPES[b % 4]) for b in range(batch)]))
            return pipe, batch, serve(pipe, lambda f, block: pipe.infer_raw(*sets[f % n_sets], graphed=True,
                                                                             kitti_results=True, block=block))
        return make

    cbgs = []

    def cbgs_pipe():
        if not cbgs:
            cbgs.append(pipeline("cbgs"))
        return cbgs[0]

    def sweeps_nusc_cbgs(batch=4):
        pipe = cbgs_pipe()
        records = [record(seed + b) for b in range(batch)]
        sets = []
        for i in range(n_sets):
            samples = []
            for b in range(batch):
                raws, tms, lags = lidar_like_sweeps(rng.integers(31000, 34001, 10), pipe.cfg.voxel_generator.range,
                                                    seed + 100 * i + b)
                samples.append(([pinned(r) for r in raws], tms, lags))
            sets.append(samples)
        return pipe, batch, serve(pipe, lambda f, block: pipe.infer_sweeps(
            sets[f % n_sets], graphed=True, nusc_results=True, poses=records,
            tokens=["f%d_%d" % (f, b) for b in range(batch)], block=block))

    def stream_cbgs(batch=4, history=10):
        pipe = cbgs_pipe()
        pcr = pipe.cfg.voxel_generator.range
        sweeps = [[pinned(lidar_like_cloud(int(rng.integers(31000, 34001)), pcr, 5, seed + 1000 + 10 * i + b))
                   for b in range(batch)] for i in range(2 * n_sets + 1)]
        motions = []
        for i in range(len(sweeps)):
            a = 0.01 * (i % 5 - 2)
            m = np.eye(4)
            m[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
            m[:3, 3] = [0.5, 0.05 * (i % 3), 0.0]
            motions.append(m)
        streams = {k: SweepStream(pipe, batch, history, 40000, in_flight=k) for k in DEPTHS}

        def run(depth, frames):
            st = streams[depth]
            for b in range(batch):
                st.reset(b)
            pose = np.eye(4)
            pipe.max_in_flight = depth
            unfinished, handles = collections.deque(), []
            for f in range(frames):
                while len(unfinished) > depth - 1:             # the push needs the slot of the oldest unfinished frame
                    unfinished.popleft().result()
                pose = pose @ motions[f % len(motions)]
                for b in range(batch):
                    st.push(b, sweeps[f % len(sweeps)][b], pose, 0.05 * f)
                h = st.infer(graphed=True, block=depth == 1)
                handles.append(h)
                if depth > 1:
                    unfinished.append(h)
            out = handles if depth == 1 else [h.result() for h in handles]
            pipe.max_in_flight = 2
            return out
        return pipe, batch, run

    return collections.OrderedDict([
        ("host_second", host_second), ("raw_kitti_second", raw_kitti("second", 1)),
        ("raw_kitti_pillars", raw_kitti("pillars", 8)), ("sweeps_nusc_cbgs", sweeps_nusc_cbgs),
        ("stream_cbgs", stream_cbgs)])


def bench(name, make, frames, rounds):
    import torch
    pipe, batch, run = make()
    want = run(1, frames)                                      # untimed: captures every graph
    for depth in DEPTHS[1:]:
        run(depth, frames)
    n_graphs = len(pipe._graphs)
    wall = {d: [] for d in DEPTHS}
    equal = True
    for r in range(rounds):
        for k in range(len(DEPTHS)):
            depth = DEPTHS[(r + k) % len(DEPTHS)]              # rotate the order round by round
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = run(depth, frames)
            wall[depth].append(time.perf_counter() - t0)
            equal &= len(out) == len(want) and all(same(a, b) for a, b in zip(out, want))
    assert len(pipe._graphs) == n_graphs, "a timed frame captured a graph"
    modes = {}
    for d in DEPTHS:
        best, mean = min(wall[d]), sum(wall[d]) / rounds
        modes["blocking" if d == 1 else "max_in_flight_%d" % d] = {
            "clouds_per_s": frames * batch / mean, "ms_per_frame": mean * 1e3 / frames,
            "ms_per_frame_best": best * 1e3 / frames, "ms_per_frame_runs": [w * 1e3 / frames for w in wall[d]]}
    base = modes["blocking"]["ms_per_frame"]
    return dict(workload=name, batch=batch, frames=frames, rounds=rounds, graphs=n_graphs,
                outputs_equal_all_modes=bool(equal), modes=modes,
                speedup_vs_blocking={m: base / v["ms_per_frame"] for m, v in modes.items() if m != "blocking"})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=21)
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_pipelined.py needs a CUDA device: det3d_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    runs = []
    for name, make in workloads(a.seed).items():
        if a.only and name not in a.only.split(","):
            continue
        runs.append(bench(name, make, a.frames, a.rounds))
        print("[bench_pipelined] %s" % json.dumps(runs[-1]), file=sys.stderr)
    result = dict(card(), what=" ".join(__doc__.strip().split("\n\n")[0].split()),
                  timing="host clock from the first submit to the last result(), pinned inputs, L2 not flushed, modes "
                         "interleaved round by round; clouds_per_s from the mean over rounds",
                  runs=runs)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    sys.exit(0 if all(r["outputs_equal_all_modes"] for r in runs) else 1)


if __name__ == "__main__":
    main()
