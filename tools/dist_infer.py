#!/usr/bin/env python
"""Multi-GPU inference harness (the role of the reference's tools/dist_test.py:180-215): one process per GPU, clouds
sharded round-robin over the ranks (DistributedSampler order, det3d/datasets/loader/sampler.py:74-96), every rank runs
the whole hot path on its shard, ONE all-gather of the fixed-shape detections over NCCL at the end.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tools/dist_infer.py --config cbgs --clouds 32 --check --out gpurun_out/dist_cbgs.json

--check: rank 0 also runs ALL clouds by itself (same per-call batch size) and asserts that the gathered detections are
bit-identical to the single-rank result -- BASELINE configs[3] (CBGS, 35k points, 32 clouds over 8 GPUs) at its stated size.
--graphed: every batch replays the CUDA graph of its (batch, point-capacity bucket) (infer_host(graphed=True)).
--variable-sizes: per-cloud point counts drawn uniformly from [0.6 N, N] (seeded), as real frames have.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cbgs", choices=["second", "pillars", "cbgs"])
    ap.add_argument("--clouds", type=int, default=32)
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--graphed", action="store_true", help="replay one CUDA graph per (batch, point-capacity bucket)")
    ap.add_argument("--variable-sizes", action="store_true", help="per-cloud point counts uniform in [0.6 N, N] (seeded)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    import bench
    from det3d.torchie import Config
    from det3d_b200.apis import InferencePipeline, all_gather_detections, init_from_env, interleave_rank_major, shard_indices

    rank, world, local = init_from_env()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    args = argparse.Namespace(config=a.config, wl=bench.WORKLOADS[a.config], dist="lidar_like")
    cfg = Config.fromfile(os.path.join(ROOT, "configs", args.wl["cfg"]))
    pipe = InferencePipeline(cfg, model=bench.build_model(cfg, args), device=dev)
    assert a.clouds % world == 0, "--clouds must be a multiple of the world size"
    b_local = a.clouds // world
    clouds = bench.make_clouds(args, a.clouds, 4242, cfg.voxel_generator.range)      # same clouds on every rank
    if a.variable_sizes:
        import numpy as np
        n = args.wl["n_points"]
        sizes = np.random.default_rng(4243).integers(int(0.6 * n), n + 1, a.clouds)
        clouds = [c[:k] for c, k in zip(clouds, sizes)]

    def run(indices):
        out = []
        for i0 in range(0, len(indices), b_local):
            chunk = [torch.from_numpy(clouds[i]) for i in indices[i0:i0 + b_local]]
            out.append(pipe.infer_host(chunk, graphed=a.graphed).clone())
        return torch.cat(out)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mine = run(shard_indices(a.clouds, rank, world)).to(dev)
    gathered = all_gather_detections(mine)                                          # [world * b_local, D, F], rank-major
    ordered = interleave_rank_major(gathered, world).cpu() if world > 1 else gathered.cpu()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    result = {"config": a.config, "clouds": a.clouds, "world": world, "clouds_per_rank": b_local, "seconds": dt,
              "graphed": a.graphed, "variable_sizes": a.variable_sizes, "graphs_captured": len(pipe._graphs),
              "detections_per_cloud": [int((ordered[i, :, -1] > 0.5).sum()) for i in range(a.clouds)]}
    ok = True
    if a.check and rank == 0:
        single = run(list(range(a.clouds)))
        result["gathered_equals_single_rank"] = bool(torch.equal(single, ordered))
        result["max_abs_diff"] = float((single - ordered).abs().max())
        result["total_detections"] = int((single[..., -1] > 0.5).sum())
        ok = result["gathered_equals_single_rank"] and result["total_detections"] > 0
    if rank == 0:
        print(json.dumps(result))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as fh:
                json.dump(result, fh, indent=1)
    if world > 1:
        flag = torch.tensor([0 if ok else 1], device=dev)
        dist.all_reduce(flag)
        ok = int(flag.item()) == 0
        dist.barrier()
        dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
