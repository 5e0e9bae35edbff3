#!/usr/bin/env python
"""Kernel time of the fp8 weight gradient (updat_fp8) against the bf16 updat, with the cost of the transposing
quantiser and of BlocksparseMatMul.matmul_fp8(fp8_dw=True) against fp8_dw=False. Needs a CUDA device.

  python scripts/fp8_updat.py [--reps R] [--out FILE]

Shape: the bench's 4096 x 4096 layer, N = 4096, feature axis 1, block sizes 32 and 64, Bernoulli layouts (diagonal
on) at 5 / 10 / 25 / 50 / 100 % density; 25 % is the bench's headline density.
- updat lines: per (block size, density), bsmm.updat of bf16 x and dy (fp32 dw) and updat_fp8 of their e4m3 / e5m2
  transposed copies, quantised beforehand (fp32 dw); each call captured in a CUDA graph, windows alternating between
  them. TFLOP/s counts 2 N blocks bs^2 per call; `share` is that rate over the H100 SXM data sheet's dense 989 (bf16)
  or 1,979 (fp8) TFLOP/s.
- quantise lines (25 %): quantize_fp8 of x (N x C) against quantize_fp8_t of x with and without the row-major copy,
  graphed.
- train_step lines (25 %): bsmm.matmul_fp8(I, W) forward + backward with fp8_dw False and True, eager, with the
  memory held between forward and backward: `new_mib` is what the forward allocates and keeps (y and the copies it
  saves), `saved_mib` the storage behind the tensors autograd saves, I itself included when it is saved.
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
N = 4096
DENSITIES = [0.05, 0.10, 0.25, 0.50, 1.00]
FP8_TFLOPS, BF16_TFLOPS = 1979.0, 989.0
MIB = 2.0 ** 20


def layout(np, bs, density, seed=0):
    rng = np.random.default_rng(seed)
    lay = (rng.random((C // bs, K // bs)) < density).astype(np.int32)
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
    from blocksparse_b200.fp8 import quantize_fp8_t, updat_fp8
    if not torch.cuda.is_available():
        raise SystemExit("scripts/fp8_updat.py needs a CUDA device")
    name, power = device_label(torch)
    lines = [{"device": name, "power_limit": power}]
    print(json.dumps(lines[0]), flush=True)

    def emit(d):
        lines.append(d)
        print(json.dumps(d), flush=True)

    def ms(r):
        return {"ms": round(r[0], 4), "spread_ms": round(r[1], 4)}

    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((N, C), generator=g, device="cuda").bfloat16()
    dy = torch.randn((N, K), generator=g, device="cuda").bfloat16()
    _, xt, xs = quantize_fp8_t(x, torch.float8_e4m3fn, with_rows=False)
    _, dyt, ds = quantize_fp8_t(dy, torch.float8_e5m2, with_rows=False)
    for bs in (32, 64):
        for density in DENSITIES:
            bsmm = BlocksparseMatMul(layout(np, bs, density), block_size=bs, feature_axis=1)
            flops = 2.0 * N * bsmm.blocks * bs * bs
            fns = {"bf16_updat": lambda: bsmm.updat([x], [dy], dw_dtype=torch.float32),
                   "fp8_updat": lambda: updat_fp8(bsmm, xt, dyt, xs, ds, N, dw_dtype=torch.float32)}
            a, b = fns["bf16_updat"](), fns["fp8_updat"]()      # the same product, so the times compare like for like
            agree = float((a - b).norm() / a.norm())
            runs = [graphed(torch, f) for f in fns.values()]
            res = timed(torch, [r[0] for r in runs], args.calls, args.reps)
            d = {"kind": "updat", "bs": bs, "density": density, "blocks": bsmm.blocks, "graph": all(r[1] for r in runs),
                 "fp8_vs_bf16_l2": agree}
            for key, r in zip(fns, res):
                tf = flops / (r[0] * 1e-3) / 1e12
                d[key] = dict(ms(r), tflops=round(tf, 1),
                              share=round(tf / (FP8_TFLOPS if key.startswith("fp8") else BF16_TFLOPS), 3))
            d["speedup"] = round(d["bf16_updat"]["ms"] / d["fp8_updat"]["ms"], 3)
            emit(d)
            if density != 0.25:
                continue
            q = {"quantize_fp8": lambda: quantize_fp8(x, torch.float8_e4m3fn),
                 "quantize_fp8_t": lambda: quantize_fp8_t(x, torch.float8_e4m3fn),
                 "quantize_fp8_t_no_rows": lambda: quantize_fp8_t(x, torch.float8_e4m3fn, with_rows=False)}
            runs = [graphed(torch, f) for f in q.values()]
            res = timed(torch, [r[0] for r in runs], args.calls, args.reps)
            emit({"kind": "quantise", "bs": bs, "density": density, **{k: ms(r) for k, r in zip(q, res)}})
            I = x.clone().requires_grad_()
            W = (torch.randn(bsmm.w_shape, generator=g, device="cuda") * 0.05).bfloat16().requires_grad_()

            def step(fp8_dw):
                def run():
                    I.grad = W.grad = None
                    bsmm.matmul_fp8(I, W, fp8_dw=fp8_dw).backward(dy)
                return run
            res = timed(torch, [step(False), step(True)], 10, args.reps)
            held = {}
            for fp8_dw in (False, True):
                I.grad = W.grad = None
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                y = bsmm.matmul_fp8(I, W, fp8_dw=fp8_dw)
                saved = {t.untyped_storage().data_ptr(): t.untyped_storage().nbytes() for t in y.grad_fn.saved_tensors}
                held[fp8_dw] = {"new_mib": round((torch.cuda.memory_allocated() - base) / MIB, 2),
                                "saved_mib": round(sum(saved.values()) / MIB, 2)}
                y.backward(dy)
                del y
            emit({"kind": "train_step", "bs": bs, "density": density, "eager": True,
                  "fp8_dw_false": dict(ms(res[0]), held=held[False]),
                  "fp8_dw_true": dict(ms(res[1]), held=held[True]),
                  "speedup": round(res[0][0] / res[1][0], 3)})
    if args.out:
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
