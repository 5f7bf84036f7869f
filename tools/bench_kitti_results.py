#!/usr/bin/env python
"""Clouds/s from raw KITTI velodyne scans to KITTI result annos: the reference's conversion on the host after the replayed
graph against the conversion on the device inside it.

SECOND car (configs/second_kitti_car.py) at B = 1 and PointPillars KITTI (configs/pointpillars_kitti_car.py) at B = 8,
each run twice.  Scans are full 360° 64-beam scans (utils/synthetic.raw_velodyne_scan, about 111k points of 4 floats)
in pinned host memory, their size varying from step to step; each slot of the batch has its own synthetic KITTI
calibration, fixed over the run.  Modes, both from the pinned raw scans to one anno dict per scan in host memory:
  a  host_convert  infer_raw(graphed=True), then the reference's convert_detection_to_kitti_annos per scan on the host
                   (oracle.kitti_results.reference_annos: the reference's numpy calls, pinned to its functions bit for
                   bit by tests/golden/make_golden_kitti_results.py)
  b  device        infer_raw(kitti_results=True, graphed=True): crop, voxelize, forward and d3b_kitti_results_dev
                   replayed from one CUDA graph
Steps are timed with CUDA events (and the host clock, which is what a caller waits: mode a's host work follows its
last event), the L2 flushed before each, the modes interleaved step by step after a warm-up that captures every graph.
On every timed step both modes must report the same detections under the same names in the same order, with
rotation_y, dimensions and score bit-identical and bbox, alpha and location within oracle.kitti_results.error_bound
(sin / cos / atan2 differ between numpy and CUDA by ulps); the run fails otherwise.  A second pass replays the device
graph with timing events at its stage boundaries and reports the new kernel's time inside the graph.

    python tools/bench_kitti_results.py --steps 20 --out profiles/h100_kitti_results.json
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

MODES = ("host_convert", "device")
CONFIGS = (("second", 1), ("pillars", 8))


def compare(host, dev, packed, calibs):
    """(same within the bound, bit-identical) for one step's annos."""
    import numpy as np
    from det3d_b200.ops.point_cloud.kitti_results import calib_table
    from oracle import kitti_results as okr
    nd = packed.shape[-1] - 3
    ok, bits = True, True
    for b, (h, d) in enumerate(zip(host, dev)):
        if list(h) != list(d) or any(h[k].dtype != d[k].dtype or h[k].shape != d[k].shape for k in h):
            return False, False
        if list(h["name"]) != list(d["name"]):
            return False, False
        ok &= all(np.array_equal(h[k], d[k]) for k in ("rotation_y", "dimensions", "score"))
        table = calib_table(calibs[b])
        _rows, keep, _a = okr.kernel_order(packed[b], nd, table)
        bound = okr.error_bound(packed[b], nd, table)[0][keep]
        for k, cols in (("bbox", slice(0, 4)), ("alpha", 4), ("location", slice(8, 11))):
            ok &= bool(np.all(np.abs(h[k] - d[k]) <= bound[:, cols]))
            bits &= np.array_equal(h[k].view(np.uint64), d[k].view(np.uint64))
    return bool(ok), bool(ok and bits)


def run(config, batch, n_scan, steps, warmup, seed):
    import numpy as np
    import torch
    import bench
    from bench_variable_clouds import card
    from det3d.torchie import Config
    from det3d_b200 import _lib
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import KITTI_IMAGE_SHAPES, kitti_like_calib, raw_velodyne_scan
    from oracle.kitti_results import reference_annos

    wl = bench.WORKLOADS[config]
    args = argparse.Namespace(config=config, wl=wl, dist="lidar_like")
    cfg = Config.fromfile(os.path.join(ROOT, "configs", wl["cfg"]))
    pipe = InferencePipeline(cfg, model=bench.build_model(cfg, args), device="cuda")
    names = pipe.class_names()
    calibs = [kitti_like_calib(seed + b, KITTI_IMAGE_SHAPES[b % 4]) for b in range(batch)]
    pool = [torch.from_numpy(raw_velodyne_scan(n_scan, 4, seed=seed * 100 + i)).pin_memory() for i in range(2 * batch)]
    rng = np.random.default_rng(seed)
    n_steps = warmup + steps
    frames = [[pool[int(rng.integers(len(pool)))][:int(rng.integers(int(0.9 * n_scan), n_scan))] for _ in range(batch)]
              for _ in range(n_steps)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    pinned_out = [None]
    packed_of = {}

    def step(mode, s):
        if mode == "host_convert":
            packed = pinned_out[0] = pipe.infer_raw(frames[s], calibs, pinned_out=pinned_out[0], graphed=True)
            host = packed.numpy()
            packed_of[s] = host.copy()
            return [reference_annos(host[b], host.shape[-1] - 3, calibs[b], names) for b in range(batch)]
        return pipe.infer_raw(frames[s], calibs, graphed=True, kitti_results=True)

    for s in range(warmup):
        for mode in MODES:
            step(mode, s)
    n_graphs = len(pipe._graphs)
    ms = {m: 0.0 for m in MODES}
    wall = {m: 0.0 for m in MODES}
    within, identical, kept = True, 0, 0
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
            outs[mode] = step(mode, s)
            e1.record()
            e1.synchronize()
            wall[mode] += time.perf_counter() - t0
            ms[mode] += e0.elapsed_time(e1)
        ok, bits = compare(outs["host_convert"], outs["device"], packed_of.pop(s), calibs)
        within &= ok
        identical += bits
        kept += sum(a["name"].shape[0] for a in outs["device"])
    assert len(pipe._graphs) == n_graphs, "a timed step captured a graph"
    graph_keys = [list(k) for k in pipe._graphs]

    # in-graph stage times of the device graph (recaptured with timing events at its stage boundaries)
    graph_ms = {}
    pipe._graphs.clear()
    _lib.GRAPH_MARKS = marks = []
    try:
        n_rep = min(steps, 10) + 2
        for s in range(n_rep):
            flush.zero_()
            pipe.infer_raw(frames[warmup + s % steps], calibs, graphed=True, kitti_results=True)
            torch.cuda.synchronize()
            if s >= 2:
                for (tag, ev, _st), (_t1, ev1, _s1) in zip(marks[:-1], marks[1:]):
                    graph_ms[tag] = graph_ms.get(tag, 0.0) + ev.elapsed_time(ev1) / (n_rep - 2)
    except RuntimeError as ex:            # (timing of externally recorded events unsupported)
        print("[bench_kitti_results] in-graph stage pass unavailable: %s" % ex, file=sys.stderr)
    finally:
        _lib.GRAPH_MARKS = None
        pipe._graphs.clear()

    res = {m: {"ms_per_step": ms[m] / steps, "clouds_per_s": steps * batch / (wall[m]),
               "wall_ms_per_step": wall[m] * 1e3 / steps} for m in MODES}
    return dict(config=wl["cfg"], batch=batch, steps=steps, warmup_steps=warmup, graphs_captured=n_graphs,
                graph_keys=graph_keys, annos_within_bound_all_steps=bool(within), annos_bit_identical_steps=identical,
                kept_detections=kept, modes=res,
                host_conversion_ms_per_scan=(wall["host_convert"] - wall["device"]) * 1e3 / (steps * batch),
                speedup_device_vs_host_convert=wall["host_convert"] / wall["device"],
                in_graph_stage_ms=graph_ms, kitti_results_in_graph_ms=graph_ms.get("kitti_results")), card()


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
        raise SystemExit("bench_kitti_results.py needs a CUDA device: det3d_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    runs, card = [], None
    for _rep in range(2):
        for config, batch in CONFIGS:
            r, card = run(config, batch, a.points_per_scan, a.steps, a.warmup, a.seed)
            runs.append(r)
    result = dict(card, what=" ".join(__doc__.strip().split("\n\n")[0].split()),
                  timing="host clock (clouds/s) and CUDA events per step from pinned raw scans to host annos, L2 flushed "
                         "before each, modes interleaved, two runs", runs=runs)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    sys.exit(0 if all(r["annos_within_bound_all_steps"] and r["kept_detections"] > 0 for r in runs) else 1)


if __name__ == "__main__":
    main()
