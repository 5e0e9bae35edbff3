#!/usr/bin/env python
"""Kernel time of the fp8 block-sparse fprop / bprop (bsmm_xprop_fp8) against the shipped bf16 kernels, with the
cost of quantisation and of BlocksparseMatMul.matmul_fp8 against bsmm(I, W). Needs a CUDA device.

  python scripts/fp8_xprop.py [--reps R] [--out FILE]

Shape: the bench's 4096 x 4096 layer, block size 32, feature axis 1, N = 4096, Bernoulli layouts (diagonal on) at
5 / 10 / 25 / 50 / 100 % density; 25 % is the bench's headline density.
- xprop lines: per density, the default bf16 route of bsmm.fprop / bsmm.bprop (whichever of the one-block and grouped
  kernels it picks) and the fp8 kernel on operands quantised beforehand (fprop e4m3 x e4m3, bprop e5m2 x e4m3), each
  call captured in a CUDA graph; windows alternate between them. TFLOP/s counts 2 N blocks bs^2 per call; `fp8_share`
  is that rate over the 1,979 TFLOP/s dense fp8 figure of the H100 SXM data sheet, `bf16_share` over 989.
- quantise lines (25 %): quantize_fp8 of x (N x C) and quantize_fp8_weights, graphed.
- train_step lines (25 %): bsmm.matmul_fp8(I, W) against bsmm(I, W), forward + backward through autograd, eager (so
  the times include the host's launch overhead, the same for both).
- scaled_mm line: a dense 4096^3 torch._scaled_mm in e4m3 with bf16 output beside a dense bf16 torch.matmul.
Times are medians over R windows (CUDA events, after warm-up) with the spread (max - min). The first line names the
device and its power limit.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from conv_bias import graphed, timed  # noqa: E402
from dense_softmax import device_label  # noqa: E402

C = K = 4096
BS, N = 32, 4096
DENSITIES = [0.05, 0.10, 0.25, 0.50, 1.00]
FP8_TFLOPS, BF16_TFLOPS = 1979.0, 989.0


def layout(np, density, seed=0):
    rng = np.random.default_rng(seed)
    lay = (rng.random((C // BS, K // BS)) < density).astype(np.int32)
    np.fill_diagonal(lay, 1)
    return lay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out")
    args = ap.parse_args()
    import numpy as np
    import torch
    from blocksparse_b200 import BlocksparseMatMul, quantize_fp8
    from blocksparse_b200.fp8 import quantize_fp8_weights, xprop_fp8
    if not torch.cuda.is_available():
        raise SystemExit("scripts/fp8_xprop.py needs a CUDA device")
    name, power = device_label(torch)
    lines = [{"device": name, "power_limit": power}]
    print(json.dumps(lines[0]), flush=True)

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((N, C), generator=g, device="cuda").bfloat16()
    dy = torch.randn((N, K), generator=g, device="cuda").bfloat16()
    for density in DENSITIES:
        bsmm = BlocksparseMatMul(layout(np, density), block_size=BS, feature_axis=1)
        w = (torch.randn(bsmm.w_shape, generator=g, device="cuda") * 0.05).bfloat16()
        xq, xs = quantize_fp8(x, torch.float8_e4m3fn)
        dq, ds = quantize_fp8(dy, torch.float8_e5m2)
        wq, wq_t, ws = quantize_fp8_weights(bsmm, w, torch.float8_e4m3fn)
        flops = 2.0 * N * bsmm.blocks * BS * BS
        fns = {
            "bf16_fprop": lambda: bsmm.fprop(x, w),
            "fp8_fprop": lambda: xprop_fp8(bsmm, xq, wq_t, xs, ws, out_dtype=torch.bfloat16),
            "bf16_bprop": lambda: bsmm.bprop(dy, w),
            "fp8_bprop": lambda: xprop_fp8(bsmm, dq, wq, ds, ws, bprop=True, out_dtype=torch.bfloat16),
        }
        # the fp8 results against the bf16 ones, so that the times compare the same product
        agree = {}
        for op in ("fprop", "bprop"):
            a, b = fns["bf16_" + op]().float(), fns["fp8_" + op]().float()
            agree[op] = float((a - b).norm() / a.norm())
        runs = [graphed(torch, f) for f in fns.values()]
        res = timed(torch, [r[0] for r in runs], args.calls, args.reps)
        d = {"kind": "xprop", "density": density, "blocks": bsmm.blocks, "graph": all(r[1] for r in runs),
             "fp8_vs_bf16_l2": agree}
        for (key, _), (ms, spread) in zip(fns.items(), res):
            tf = flops / (ms * 1e-3) / 1e12
            d[key] = {"ms": round(ms, 4), "spread_ms": round(spread, 4), "tflops": round(tf, 1),
                      "share": round(tf / (FP8_TFLOPS if key.startswith("fp8") else BF16_TFLOPS), 3)}
        for op in ("fprop", "bprop"):
            d[op + "_speedup"] = round(d["bf16_" + op]["ms"] / d["fp8_" + op]["ms"], 3)
        emit(d)
        if density == 0.25:
            q = {"quantize_x": lambda: quantize_fp8(x, torch.float8_e4m3fn),
                 "quantize_w": lambda: quantize_fp8_weights(bsmm, w, torch.float8_e4m3fn)}
            runs = [graphed(torch, f) for f in q.values()]
            res = timed(torch, [r[0] for r in runs], args.calls, args.reps)
            emit({"kind": "quantise", "density": density, **{k: {"ms": round(ms, 4), "spread_ms": round(sp, 4)}
                                                             for k, (ms, sp) in zip(q, res)}})
            I = x.clone().requires_grad_()
            W = w.clone().requires_grad_()

            def step(op):
                def run():
                    I.grad = W.grad = None
                    op(I, W).backward(dy)
                return run
            res = timed(torch, [step(bsmm), step(bsmm.matmul_fp8)], 10, args.reps)
            emit({"kind": "train_step", "density": density, "eager": True,
                  "bsmm": {"ms": round(res[0][0], 4), "spread_ms": round(res[0][1], 4)},
                  "matmul_fp8": {"ms": round(res[1][0], 4), "spread_ms": round(res[1][1], 4)},
                  "speedup": round(res[0][0] / res[1][0], 3)})
    # dense scale: torch._scaled_mm in e4m3 against a dense bf16 matmul
    a = torch.randn((N, C), generator=g, device="cuda").to(torch.float8_e4m3fn)
    b = torch.randn((K, C), generator=g, device="cuda").to(torch.float8_e4m3fn)
    one = torch.ones((), device="cuda")
    ab, bb = a.bfloat16(), b.bfloat16()
    fns = [lambda: torch._scaled_mm(a, b.t(), scale_a=one, scale_b=one, out_dtype=torch.bfloat16),
           lambda: torch.matmul(ab, bb.t())]
    runs = [graphed(torch, f) for f in fns]
    res = timed(torch, [r[0] for r in runs], args.calls, args.reps)
    flops = 2.0 * N * C * K
    emit({"kind": "dense", "shape": [N, C, K],
          "scaled_mm_e4m3": {"ms": round(res[0][0], 4), "spread_ms": round(res[0][1], 4),
                             "tflops": round(flops / res[0][0] / 1e9, 1), "share": round(flops / res[0][0] / 1e9 / FP8_TFLOPS, 3)},
          "matmul_bf16": {"ms": round(res[1][0], 4), "spread_ms": round(res[1][1], 4),
                          "tflops": round(flops / res[1][0] / 1e9, 1), "share": round(flops / res[1][0] / 1e9 / BF16_TFLOPS, 3)}})
    if args.out:
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
