"""Achieved rates of BlocksparseConv fprop / bprop / updat on the GPU, with CUDA events after warm-up, on each route:
bf16 on the wgmma kernels, fp32 on the FMA kernels and bf16 forced onto the FMA kernels. Block-diagonal layouts are
also timed as torch.nn.functional.conv2d(groups=blocks) at the same shape (cuDNN) for comparison. Rates are
2 * sizeF * MPQ * N flops (the reference's `flops`) per op over its time. Prints the card and its power limit.

    python scripts/conv_rate.py [--iters 20] [--out conv_rate.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from blocksparse_b200 import _lib  # noqa: E402
from blocksparse_b200.conv import BlocksparseConv  # noqa: E402


def timed(fn, iters):
    for _ in range(3):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters * 1e-3


def cases():
    diag = [[list(range(b * 64, b * 64 + 64)), list(range(b * 64, b * 64 + 64))] for b in range(8)]
    over = [[list(range(b * 32, b * 32 + 64)), list(range(b * 32, b * 32 + 64))] for b in range(15)]
    return [("diag8x64 3x3 32x32 N32", diag, (32, 32), (1, 1), 32, True),
            ("diag8x64 3x3 56x56 N32", diag, (56, 56), (1, 1), 32, True),
            ("diag8x64 3x3 56x56 stride2 N32", diag, (56, 56), (2, 2), 32, True),
            ("overlap15x64 3x3 32x32 N32", over, (32, 32), (1, 1), 32, False)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("conv_rate.py needs a GPU")
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                                         "-i", "0"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    print("card: %s; power limit, max SM clock: %s" % (card, power))
    rows = []
    for label, BCK, DHW, strides, N, diag in cases():
        op = BlocksparseConv(BCK, (3, 3), DHW, strides=strides)
        flops = op.flops * N
        for route, dt, flags in (("wgmma bf16", torch.bfloat16, 0), ("fma fp32", torch.float32, 0),
                                 ("fma bf16", torch.bfloat16, _lib.FLAG_FORCE_GENERIC)):
            f = (torch.randn(op.sizeF, device="cuda") * 0.05).to(dt)
            x = torch.randn(op.i_shape(N), device="cuda").to(dt).view(N, op.C, -1)
            e = torch.randn(op.o_shape(N), device="cuda").to(dt).view(N, op.K, -1)
            t = {"fprop": timed(lambda: op._xprop(f, x, False, flags), args.iters),
                 "bprop": timed(lambda: op._xprop(f, e, True, flags), args.iters),
                 "updat": timed(lambda: op._updat(e, x, dt, flags), args.iters)}
            row = dict(case=label, route=route, **{k + "_ms": v * 1e3 for k, v in t.items()},
                       **{k + "_tflops": flops / v * 1e-12 for k, v in t.items()})
            rows.append(row)
            print("%-32s %-10s " % (label, route) + "  ".join("%s %.3f ms %.1f TFLOP/s" % (k, v * 1e3, flops / v * 1e-12)
                                                            for k, v in t.items()))
        if diag:
            w = torch.randn(op.K, 64, 3, 3, device="cuda", dtype=torch.bfloat16) * 0.05
            xi = torch.randn([N, op.C] + list(DHW), device="cuda", dtype=torch.bfloat16)
            tc = timed(lambda: torch.nn.functional.conv2d(xi, w, stride=strides, padding=1, groups=len(BCK)), args.iters)
            rows.append(dict(case=label, route="cudnn conv2d groups bf16", fprop_ms=tc * 1e3, fprop_tflops=flops / tc * 1e-12))
            print("%-32s %-10s fprop %.3f ms %.1f TFLOP/s" % (label, "cudnn bf16", tc * 1e3, flops / tc * 1e-12))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(dict(card=card, power=power, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
