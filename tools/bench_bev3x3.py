#!/usr/bin/env python
"""The dense 3x3 stride-1 RPN layer alone, at the shapes the three detectors run it: the automatic schedule against the
pixel-stationary kernel (variant 0), and the automatic schedule in single-pass FP16 (one input / output plane,
`set_math("fp16")`), alternating in one process.

    python tools/bench_bev3x3.py [--reps 30] [--out FILE]

Shapes (batch x H x W x C_in -> C_out, NHWC f16 planes, 3x3, pad 1, bias + folded BN + ReLU, planes out):
SECOND 1x200x176x128 -> 128, CBGS 4x128x128x128 -> 128 and 4x64x64x256 -> 256, PointPillars 8x124x108x128 -> 128.
Each launch is timed alone with CUDA events after a 256 MiB write that flushes L2; a device-side sleep ahead of the
first event keeps the host's enqueue time out of the window.  Per shape and variant: the median over --reps launches
in microseconds, fp32-equivalent TFLOP/s (2 B H W 9 C_in C_out / time) and its share of 989 / 3 TFLOP/s -- the H100
SXM data-sheet dense f16 rate over the three products FP16x3 spends per fp32-equivalent multiply-add (single pass: the
f16-equivalent TFLOP/s and its share of 989, one product per multiply-add).  The card's
name, power limit and maximum SM clock are read in the same call.  Prints one JSON line (and writes it to --out).
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

SHAPES = [
    ("second", 1, 200, 176, 128, 128),
    ("cbgs", 4, 128, 128, 128, 128),
    ("cbgs_256", 4, 64, 64, 256, 256),
    ("pillars", 8, 124, 108, 128, 128),
]
F16X3_PEAK_TFLOPS = 989.0 / 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_bev3x3.py needs a CUDA device")
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import conv16

    gpu = gpu_info()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    lib = _lib.lib()
    prev = lib.d3b_get_bev_variant()
    results = {}
    try:
        for name, b, h, w, c_in, c_out in SHAPES:
            g = torch.Generator(device=dev).manual_seed(c_in + h)
            wt = torch.randn((9, c_in, c_out), device=dev, generator=g) / (9 * c_in * 0.3) ** 0.5
            layer = conv16.BevConv16(wt, 3, stride=1, pad=1, bias=torch.randn(c_out, device=dev, generator=g) * 0.1,
                                     scale=torch.rand(c_out, device=dev, generator=g) + 0.5,
                                     shift=torch.randn(c_out, device=dev, generator=g) * 0.1, relu=True, device=dev)
            xf = torch.randn((b, h, w, c_in), device=dev, generator=g)
            x, x1 = conv16.Planes.from_f32(xf), conv16.Planes.from_f32(xf, n_planes=1)
            out, out1 = conv16.Planes((b, h, w, c_out), dev), conv16.Planes((b, h, w, c_out), dev, n_planes=1)
            flops = layer.flops(b, h, w)
            # (bev variant, input, output): pixel-stationary FP16x3, automatic FP16x3, automatic single pass
            runs = {"pixel_stationary": (0, x, out), "automatic": (2, x, out), "automatic_fp16": (2, x1, out1)}
            times = {k: [] for k in runs}
            for variant, xi, oi in runs.values():              # warm-up: module load, tensor-map encoder
                lib.d3b_set_bev_variant(variant)
                for _ in range(3):
                    layer(xi, out=oi)
            torch.cuda.synchronize()
            for _ in range(args.reps):
                for key, (variant, xi, oi) in runs.items():
                    lib.d3b_set_bev_variant(variant)
                    flush.zero_()
                    torch.cuda._sleep(100000)
                    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    layer(xi, out=oi)
                    e.record()
                    e.synchronize()
                    times[key].append(a.elapsed_time(e) * 1e3)
            row = {"shape": [b, h, w, c_in, c_out], "fp32_equivalent_flops": flops}
            for key in runs:
                us = statistics.median(times[key])
                tflops = flops / (us * 1e-6) / 1e12
                row[key] = {"us_per_launch": us, "us_min": min(times[key]), "us_max": max(times[key])}
                if key == "automatic_fp16":
                    row[key].update(f16_tflops=tflops, share_of_989=tflops / (3 * F16X3_PEAK_TFLOPS))
                else:
                    row[key].update(fp32_equivalent_tflops=tflops, share_of_989_over_3=tflops / F16X3_PEAK_TFLOPS)
            row["speedup"] = row["pixel_stationary"]["us_per_launch"] / row["automatic"]["us_per_launch"]
            row["speedup_fp16_over_automatic"] = row["automatic"]["us_per_launch"] / row["automatic_fp16"]["us_per_launch"]
            results[name] = row
    finally:
        lib.d3b_set_bev_variant(prev)
    line = {"what": "dense 3x3 stride-1 layer alone, automatic schedule vs pixel-stationary (variant 0), and the "
                    "automatic schedule in single-pass FP16",
            "method": "CUDA events around one launch, L2 flushed (256 MiB write) and a device sleep before each, "
                      "variants alternating, median of %d" % args.reps,
            "results": results, "gpu": gpu}
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(json.dumps(line) + "\n")
    print(json.dumps(line))
    for name, row in results.items():
        print("%-9s %-22s variant 0 %7.1f us %6.1f TFLOP/s %5.1f%% | automatic %7.1f us %6.1f TFLOP/s %5.1f%% | %.2fx"
              " | fp16 %7.1f us %6.1f TFLOP/s %5.1f%% of 989 | %.2fx" % (
                  name, "x".join(map(str, row["shape"][:4])) + "->%d" % row["shape"][4],
                  row["pixel_stationary"]["us_per_launch"], row["pixel_stationary"]["fp32_equivalent_tflops"],
                  100 * row["pixel_stationary"]["share_of_989_over_3"], row["automatic"]["us_per_launch"],
                  row["automatic"]["fp32_equivalent_tflops"], 100 * row["automatic"]["share_of_989_over_3"], row["speedup"],
                  row["automatic_fp16"]["us_per_launch"], row["automatic_fp16"]["f16_tflops"],
                  100 * row["automatic_fp16"]["share_of_989"], row["speedup_fp16_over_automatic"]))


if __name__ == "__main__":
    main()
