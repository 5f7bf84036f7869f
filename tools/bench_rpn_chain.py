#!/usr/bin/env python
"""The RPN + heads stack (FusedBevStack.run) of each detector at its bench shape, whose 3x3 stride-1 layers are the
dense stage's bulk: SECOND 1x200x176x128, PointPillars 8x496x432x64, CBGS 4x128x128x256 (necks of configs/, BN
statistics and weights drawn from a seed).

    python tools/bench_rpn_chain.py [--reps 30] [--out FILE]

Each run is timed with CUDA events after a 256 MiB write that flushes L2 and a device-side sleep that keeps the host's
enqueue time out of the window; median, min and max over --reps runs in milliseconds.  It runs unchanged on any tree
with FusedBevStack.run, so two builds can be compared.  The card's name, power limit and maximum SM clock are read in
the same call.  Prints one JSON line (and writes it to --out).
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_pillars_nusc import gpu_info  # noqa: E402

STACKS = [
    ("second", dict(layer_nums=[5], ds_layer_strides=[1], ds_num_filters=[128], us_layer_strides=[1],
                    us_num_filters=[128], num_input_features=128), (1, 200, 176, 128), (14, 2, 4)),
    ("pillars", dict(layer_nums=[3, 5, 5], ds_layer_strides=[2, 2, 2], ds_num_filters=[64, 128, 256],
                     us_layer_strides=[1, 2, 4], us_num_filters=[128, 128, 128], num_input_features=64),
     (8, 496, 432, 64), (14, 2, 4)),
    ("cbgs", dict(layer_nums=[5, 5], ds_layer_strides=[1, 2], ds_num_filters=[128, 256], us_layer_strides=[1, 2],
                  us_num_filters=[256, 256], num_input_features=256), (4, 128, 128, 256), (20, 4, 0)),
]


def _stack(neck, head_widths, device):
    import torch
    from torch import nn
    from det3d_b200.models.necks.rpn import RPN
    from det3d_b200.ops.spconv import bev

    class Task(nn.Module):
        def __init__(self, c, box, cls, dirs):
            super().__init__()
            self.conv_box, self.conv_cls = nn.Conv2d(c, box, 1), nn.Conv2d(c, cls, 1)
            self.use_dir = dirs > 0
            if self.use_dir:
                self.conv_dir = nn.Conv2d(c, dirs, 1)

    class Head(nn.Module):
        def __init__(self, c):
            super().__init__()
            self.tasks = nn.ModuleList([Task(c, *head_widths)])

    torch.manual_seed(0)
    rpn = RPN(**neck).eval().to(device)
    for m in rpn.modules():
        if isinstance(m, nn.modules.batchnorm._BatchNorm):
            m.running_mean.uniform_(-0.1, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    return bev.FusedBevStack(rpn, Head(sum(neck["us_num_filters"])).to(device))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_rpn_chain.py needs a CUDA device")
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16

    gpu = gpu_info()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    results = {}
    with torch.no_grad():
        for name, neck, shape, head_widths in STACKS:
            stack = _stack(neck, head_widths, dev)
            x = conv16.Planes.from_f32(torch.randn(shape, device=dev, generator=torch.Generator(device=dev).manual_seed(1)))
            for _ in range(3):                              # warm-up: module load, buffers, tensor-map encoder
                stack.run(x)
            torch.cuda.synchronize()
            launches0 = _lib.launch_count()
            stack.run(x)
            launches = _lib.launch_count() - launches0
            times = []
            for _ in range(args.reps):
                flush.zero_()
                torch.cuda._sleep(100000)
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                stack.run(x)
                e.record()
                e.synchronize()
                times.append(a.elapsed_time(e))
            results[name] = {"input": list(shape), "ms_median": statistics.median(times), "ms_min": min(times),
                             "ms_max": max(times), "launches": launches}
    line = {"what": "RPN + heads stack (FusedBevStack.run) at each detector's bench shape",
            "method": "CUDA events around one run, L2 flushed (256 MiB write) and a device sleep before each, median of %d"
                      % args.reps, "results": results, "gpu": gpu}
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(json.dumps(line) + "\n")
    print(json.dumps(line))


if __name__ == "__main__":
    main()
