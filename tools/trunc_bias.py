"""Measure the residual bias of the convolution kernels' accumulation on the GPU this runs on.

For each kernel and operand regime (A: all-positive operands; B: ReLU-like activations, half zeros, with zero-mean
weights -- what the network feeds the kernels; C: zero-mean both) one large seeded launch is compared with its float64
reference, and the residual slope

    beta = sum (got - ref) ref / sum ref^2

is printed with its standard error, in units of eps = 2^-26 (kTruncLossPerMma in csrc/gmma.cuh).  The FP16x3 kernels
(sparse output-stationary, dense pixel-stationary and pipelined) are measured against the split-exact result yh of the
operands they see (tests/test_conv_error_model_gpu.py): each full slot chains n = 12 truncating MMAs and the epilogue
adds 12 eps (kTruncLossPerMma per MMA) to the sums, so the true mean loss per MMA is about (12 eps - beta) / 12.  The tf32x3
fallback kernels (simt, tc; tc over a dense rulebook) are measured against the exact y at features ~3e5.  The
single-pass FP16 kernels (math "fp16") are measured against yh1 = sum a_hi w_hi (tests/test_fp16_single_gpu.py): a full
slot chains n = 4 MMAs and the epilogue adds 4 eps.

    python tools/trunc_bias.py [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import test_conv_error_model_gpu as em  # noqa: E402
import test_fp16_single_gpu as f1  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable (%s)" % e


def tf32_case(algo, regime):
    from det3d_b200 import _lib
    from det3d_b200.ops.spconv import bev, core
    gen = torch.Generator(device="cuda").manual_seed(7)
    if algo == "tc_dense":
        b, h, w, c = 1, 96, 88, 128
        x, wt = em.operands((b, h, w, c), (9, c, c), regime, gen, a_scale=3.0e5)
        grid = bev.BevGrid(b, h, w, "cuda")
        out = torch.empty((b * h * w, c), device="cuda")
        core.sparse_conv(x.reshape(-1, c), grid.rulebook(3, 3, 1, 1), core.ConvWeights(wt, algo=_lib.ALGO_TC), out)
        w4 = wt.double().reshape(3, 3, c, c).permute(3, 2, 0, 1)
        y = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), w4, padding=1).permute(0, 2, 3, 1).reshape(-1, c)
        return out, y
    n, c = 20000, 64
    lvl = em._level(n, (20, 100, 100), 2, 11)
    rb = core.build_subm_rulebook(core.alloc_subm_rulebook(lvl, 3))
    x, w = em.operands((n, c), (27, c, c), regime, gen, a_scale=3.0e5)
    out = torch.empty((n, c), device="cuda")
    core.sparse_conv(x, rb, core.ConvWeights(w, algo=_lib.ALGO_SIMT if algo == "simt" else _lib.ALGO_TC), out)
    idx = rb.nbr[:, :n].long()
    y = torch.zeros((n, c), dtype=torch.float64, device="cuda")
    for k in range(27):
        ok = idx[k] >= 0
        y[ok] += x.double()[idx[k][ok]] @ w.double()[k]
    return out, y


def fp16_case(kernel, regime):
    """The shapes of em.bias_case on the single-pass kernels -> (got, Ref1)."""
    from det3d_b200 import _lib
    if kernel == "sparse":
        out, ref, *_ = f1.run_sparse1(64, 64, 27, 20000, 11, regime=regime, spatial=(20, 100, 100))
        return out[:20000], ref
    prev = _lib.lib().d3b_get_bev_variant()
    try:
        _lib.lib().d3b_set_bev_variant(2 if kernel == "dense_pl" else 0)
        got, ref, *_ = f1.run_dense1(1, 96, 88, 128, 128, 3, 1, 1, 1, 23, regime=regime)
    finally:
        _lib.lib().d3b_set_bev_variant(prev)
    return got, ref


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", default=None, help="also write the results as JSON lines to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU: the bias is a property of its tensor cores"
    import __graft_entry__
    __graft_entry__.build()
    info = gpu_info()
    print("gpu: %s" % info)
    rows = []
    eps = em.EPS
    for kernel in ("sparse", "dense_ps", "dense_pl"):
        for regime in ("A", "B", "C"):
            got, ref = em.bias_case(kernel, regime)
            beta, se = em.residual_slope(got, ref.yh)
            applied = 12 * eps
            rows.append(dict(kernel=kernel, math="fp16x3", regime=regime, outputs=got.numel(), beta_eps=beta / eps,
                             se_eps=se / eps, applied_eps=applied / eps, loss_per_mma_eps=(applied - beta) / 12 / eps))
    for kernel in ("sparse", "dense_ps", "dense_pl"):
        for regime in ("A", "B", "C"):
            got, ref = fp16_case(kernel, regime)
            beta, se = em.residual_slope(got, ref.yh)
            applied = 4 * eps
            rows.append(dict(kernel=kernel, math="fp16", regime=regime, outputs=got.numel(), beta_eps=beta / eps,
                             se_eps=se / eps, applied_eps=applied / eps, loss_per_mma_eps=(applied - beta) / 4 / eps))
    for algo in ("simt", "tc", "tc_dense"):
        for regime in ("A", "B", "C"):
            got, y = tf32_case(algo, regime)
            beta, se = em.residual_slope(got, y)
            rows.append(dict(kernel=algo, math="tf32x3", regime=regime, outputs=got.numel(), beta_eps=beta / eps,
                             se_eps=se / eps, beta_rel=beta))
    for r in rows:
        extra = (" (applied %+.0f eps/slot: loss/MMA %.2f eps)" % (r["applied_eps"], r["loss_per_mma_eps"])
                 if r["math"] in ("fp16x3", "fp16") else " (%.2e relative)" % r["beta_rel"])
        print("%-8s %-7s regime %s  n=%8d  beta = %+8.3f eps  se %.3f eps%s" % (
            r["kernel"], r["math"], r["regime"], r["outputs"], r["beta_eps"], r["se_eps"], extra))
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(json.dumps(dict(gpu=info, torch=torch.__version__)) + "\n")
            for r in rows:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
