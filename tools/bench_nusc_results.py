#!/usr/bin/env python
"""Clouds/s from raw nuScenes-style sweeps to nuScenes submission boxes: the reference's per-box conversion on the host
after the replayed graph against the conversion on the device inside it.

CBGS nuScenes (configs/cbgs_nusc.py) and PointPillars nuScenes (configs/pointpillars_nusc.py), both at B = 4, each run
twice.  Each sample is a key frame and 9 sweeps of about 34k raw records of 5 floats (utils/synthetic.lidar_like_sweeps)
in pinned host memory, the sweep sizes drawn per step; each slot of the batch has its own nuScenes-like pose record
(LIDAR_TOP about -90 deg about z, the ego 300-2500 m out), fixed over the run.  Modes, both from the pinned raw sweeps to
the nusc_annos dict in host memory:
  a  host_convert  infer_sweeps(graphed=True), then the reference's conversion per box on the host
                   (oracle.nusc_results.reference_annos: the reference's code path on stand-ins that restate pyquaternion
                   and the devkit's Box -- not pyquaternion itself, which is not installed)
  b  device        infer_sweeps(graphed=True, nusc_results=True): ingest, voxelize, forward and d3b_nusc_results_dev
                   replayed from one CUDA graph
Steps are timed with CUDA events and the host clock (what a caller waits: mode a's host work follows its last event),
the L2 flushed before each, the modes interleaved step by step after a warm-up that captures every graph.  On every
timed step both modes must give the same tokens, names, attributes, sizes and scores in the same order, with the
translation, rotation and velocity within oracle.nusc_results.error_bound; the run fails otherwise.  A second pass
replays the device graph with timing events at its stage boundaries and reports the new kernel's time inside the graph.

    python tools/bench_nusc_results.py --steps 20 --out profiles/h100_nusc_results.json
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
CONFIGS = ("cbgs", "pillars_nusc")


def record(seed):
    """A nuScenes-like key-frame record (as tests/test_nusc_results_gpu.py draws them)."""
    import numpy as np
    from oracle.nusc_results import _q_matrix

    def quat(axis, angle):
        axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
        return np.concatenate([[np.cos(angle / 2)], axis * np.sin(angle / 2)])
    rng = np.random.default_rng(seed)
    cs_q = _q_matrix(quat([0, 0, 1], -np.pi / 2 + rng.uniform(-0.02, 0.02))) @ quat([1, 0, 0], rng.uniform(-0.005, 0.005))
    ego_q = _q_matrix(quat([0, 0, 1], rng.uniform(-np.pi, np.pi))) @ quat([0, 1, 0], rng.uniform(-0.03, 0.03))
    r, a = rng.uniform(300, 2500), rng.uniform(-np.pi, np.pi)
    return {"calibrated_sensor": {"translation": [0.94, 0.0, 1.84], "rotation": [float(v) for v in cs_q]},
            "ego_pose": {"translation": [r * np.cos(a), r * np.sin(a), 0.1], "rotation": [float(v) for v in ego_q]}}


def compare(host, dev, packed, records, tokens):
    """(same within the bound, bit-identical) for one step's nusc_annos."""
    import numpy as np
    from det3d_b200.ops.point_cloud.nusc_results import pose_table
    from oracle import nusc_results as onr
    if list(host) != list(dev) or host["meta"] != dev["meta"] or list(host["results"]) != list(dev["results"]):
        return False, False
    ok, bits = True, True
    for b, t in enumerate(tokens):
        h, d = host["results"][t], dev["results"][t]
        if len(h) != len(d):
            return False, False
        bound = onr.error_bound(packed[b], pose_table(records[b]), records[b])[0][packed[b][:, 11] > 0.5]
        for i, (x, y) in enumerate(zip(h, d)):
            if list(x) != list(y):
                return False, False
            ok &= all(x[k] == y[k] for k in ("sample_token", "size", "detection_name", "detection_score",
                                                "attribute_name"))
            for k, cols in (("translation", slice(0, 3)), ("rotation", slice(6, 10)), ("velocity", slice(10, 12))):
                diff = np.abs(np.array(x[k]) - np.array(y[k]))
                ok &= bool(np.all(diff <= bound[i, cols]))
                bits &= bool(np.all(diff == 0))
    return bool(ok), bool(ok and bits)


def run(config, batch, n_sweep, n_sweeps, steps, warmup, seed):
    import numpy as np
    import torch
    import bench
    from bench_variable_clouds import card
    from det3d.torchie import Config
    from det3d_b200 import _lib
    from det3d_b200.apis import InferencePipeline
    from det3d_b200.utils.synthetic import lidar_like_sweeps
    from oracle.nusc_results import reference_annos

    if config == "cbgs":
        wl = bench.WORKLOADS["cbgs"]
        cfg = Config.fromfile(os.path.join(ROOT, "configs", wl["cfg"]))
        model = bench.build_model(cfg, argparse.Namespace(config="cbgs", wl=wl, dist="lidar_like"))
    else:
        from bench_pillars_nusc import build_model
        cfg = Config.fromfile(os.path.join(ROOT, "configs", "pointpillars_nusc.py"))
        model = build_model(cfg)
    pipe = InferencePipeline(cfg, model=model, device="cuda")
    names = pipe.class_names()
    records = [record(seed + b) for b in range(batch)]
    base = []
    for b in range(batch):
        raws, tms, lags = lidar_like_sweeps([n_sweep] * n_sweeps, cfg.voxel_generator.range, seed + b)
        base.append(([torch.from_numpy(r).pin_memory() for r in raws], tms, lags))
    rng = np.random.default_rng(seed)
    n_steps = warmup + steps
    sizes = rng.integers(int(0.9 * n_sweep), n_sweep + 1, (n_steps, batch, n_sweeps))
    batches = [[([r[:int(n)] for r, n in zip(raws, sizes[s, b])], tms, lags) for b, (raws, tms, lags) in enumerate(base)]
               for s in range(n_steps)]
    tokens = [["s%d_%d" % (s, b) for b in range(batch)] for s in range(n_steps)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    pinned_out = [None]
    packed_of = {}

    def step(mode, s):
        if mode == "host_convert":
            packed = pinned_out[0] = pipe.infer_sweeps(batches[s], pinned_out=pinned_out[0], graphed=True)
            host = packed.numpy()
            packed_of[s] = host.copy()
            return reference_annos(host, records, tokens[s], names)
        return pipe.infer_sweeps(batches[s], graphed=True, nusc_results=True, poses=records, tokens=tokens[s])

    for s in range(warmup):
        for mode in MODES:
            step(mode, s)
    n_graphs = len(pipe._graphs)
    ms = {m: 0.0 for m in MODES}
    wall = {m: 0.0 for m in MODES}
    within, identical, boxes = True, 0, 0
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
        ok, bits = compare(outs["host_convert"], outs["device"], packed_of.pop(s), records, tokens[s])
        within &= ok
        identical += bits
        boxes += sum(len(v) for v in outs["device"]["results"].values())
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
            k = warmup + s % steps
            pipe.infer_sweeps(batches[k], graphed=True, nusc_results=True, poses=records, tokens=tokens[k])
            torch.cuda.synchronize()
            if s >= 2:
                for (tag, ev, _st), (_t1, ev1, _s1) in zip(marks[:-1], marks[1:]):
                    graph_ms[tag] = graph_ms.get(tag, 0.0) + ev.elapsed_time(ev1) / (n_rep - 2)
    except RuntimeError as ex:            # (timing of externally recorded events unsupported)
        print("[bench_nusc_results] in-graph stage pass unavailable: %s" % ex, file=sys.stderr)
    finally:
        _lib.GRAPH_MARKS = None
        pipe._graphs.clear()

    res = {m: {"ms_per_step": ms[m] / steps, "clouds_per_s": steps * batch / (wall[m]),
               "wall_ms_per_step": wall[m] * 1e3 / steps} for m in MODES}
    return dict(config=config, batch=batch, steps=steps,
                warmup_steps=warmup, graphs_captured=n_graphs, graph_keys=graph_keys,
                annos_within_bound_all_steps=bool(within), annos_bit_identical_steps=identical, boxes=boxes, modes=res,
                host_conversion_ms_per_sample=(wall["host_convert"] - wall["device"]) * 1e3 / (steps * batch),
                speedup_device_vs_host_convert=wall["host_convert"] / wall["device"],
                in_graph_stage_ms=graph_ms, nusc_results_in_graph_ms=graph_ms.get("nusc_results")), card()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--points-per-sweep", type=int, default=34000)
    ap.add_argument("--sweeps", type=int, default=10)
    ap.add_argument("--seed", type=int, default=13)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_nusc_results.py needs a CUDA device: det3d_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    runs, card = [], None
    for _rep in range(2):
        for config in CONFIGS:
            r, card = run(config, a.batch, a.points_per_sweep, a.sweeps, a.steps, a.warmup, a.seed)
            runs.append(r)
    result = dict(card, what=" ".join(__doc__.strip().split("\n\n")[0].split()),
                  timing="host clock (clouds/s) and CUDA events per step from pinned raw sweeps to host nusc_annos, L2 "
                         "flushed before each, modes interleaved, two runs",
                  host_baseline="oracle.nusc_results.reference_annos: the reference's conversion on stand-ins restating "
                                "pyquaternion and the devkit's Box, not pyquaternion itself",
                  runs=runs)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")
    sys.exit(0 if all(r["annos_within_bound_all_steps"] and r["boxes"] > 0 for r in runs) else 1)


if __name__ == "__main__":
    main()
