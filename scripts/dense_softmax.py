#!/usr/bin/env python
"""Kernel time and bandwidth of the dense softmax ops against the torch composition of the same math. Needs a CUDA
device.

  python scripts/dense_softmax.py [--reps R] [--out FILE]

Shapes: batch 4, heads 16, ctx 1024 and 4096, fp16 and bf16, no mask and a causal (1, 1, ctx, ctx) fp32 mask; for each,
masked_softmax forward and its gradient. Then masked_top_k_softmax (causal mask) and top_k at D3 = 1024 with k = 32
and 256. Per case one JSON line with:
  * ms: median over R windows of N launches of the op's kernel (CUDA events around the window, after warm-up);
  * torch_ms: the same for the torch composition (x.float() * mask * scale, masked_fill, torch.softmax, cast back; the
    gradient formula; torch.topk), timed in windows alternating with ours;
  * GB/s and the share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s), from the algorithmic bytes: x, y and dy
    as the op reads or writes them, plus the mask counted once.
The first line names the device and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH, HEADS = 4, 16
HBM_TBS = 3.35
FLT_MAX = 3.4028234663852886e38


def device_label(torch):
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        out = ""
    return name, out or "unknown"


def window(torch, fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def compare(torch, ours, ref, n, reps):
    for fn in (ours, ref):
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    t_ours, t_ref = [], []
    for _ in range(reps):
        t_ours.append(window(torch, ours, n))
        t_ref.append(window(torch, ref, n))
    return sorted(t_ours)[reps // 2], sorted(t_ref)[reps // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from blocksparse_b200 import masked_softmax, masked_top_k_softmax, top_k
    from blocksparse_b200 import transformer as tr

    if not torch.cuda.is_available():
        sys.exit("scripts/dense_softmax.py needs a CUDA device")
    torch.cuda.set_device(0)
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power})]
    print(lines[-1], flush=True)
    scale = 0.125

    def emit(rec, nbytes, ms, torch_ms):
        rec.update(ms=round(ms, 4), torch_ms=round(torch_ms, 4), speedup=round(torch_ms / ms, 2),
                   GBps=round(nbytes / (ms * 1e6), 1), hbm_share=round(nbytes / (ms * 1e-3) / (HBM_TBS * 1e12), 3))
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)

    gen = torch.Generator(device="cuda").manual_seed(0)
    for ctx in (1024, 4096):
        n = 200 if ctx == 1024 else 40
        causal = torch.tril(torch.ones(ctx, ctx, device="cuda")).view(1, 1, ctx, ctx)
        for dtype in (torch.float16, torch.bfloat16):
            x = torch.randn(BATCH, HEADS, ctx, ctx, device="cuda", generator=gen).to(dtype)
            dy = torch.randn(BATCH, HEADS, ctx, ctx, device="cuda", generator=gen).to(dtype)
            esize = x.element_size()
            for mask in (None, causal):
                m, M1, M2 = tr._dense_mask(x, mask, "bench")
                mbytes = 0 if mask is None else mask.numel() * 4
                zero = None if mask is None else mask == 0

                def ref_fwd():
                    v = x.float() * scale if mask is None else (x.float() * mask * scale).masked_fill(zero, -FLT_MAX)
                    return torch.softmax(v, -1).to(dtype)
                y = masked_softmax(x, mask, scale)
                # the two compute the same probabilities; a gross mismatch would make the timing meaningless
                assert (y.float() - ref_fwd().float()).abs().max().item() < 1e-2
                ms, tms = compare(torch, lambda: tr._dense_softmax_fwd(x, m, M1, M2, scale), ref_fwd, n, args.reps)
                rec = dict(op="masked_softmax", shape=[BATCH, HEADS, ctx, ctx], dtype=str(dtype)[6:],
                           mask=None if mask is None else "causal (1, 1, ctx, ctx) fp32")
                emit(rec, 2 * x.numel() * esize + mbytes, ms, tms)

                def ref_grad():
                    yf, dyf = y.float(), dy.float()
                    g = (dyf - (dyf * yf).sum(-1, keepdim=True)) * yf
                    return (g * scale if mask is None else g * mask * scale).to(dtype)
                ms, tms = compare(torch, lambda: tr._dense_softmax_bwd(y, dy, m, M1, M2, scale), ref_grad, n, args.reps)
                emit(dict(rec, op="masked_softmax_grad"), 3 * x.numel() * esize + mbytes, ms, tms)
                del y
            del x, dy
            torch.cuda.empty_cache()

    ctx = 1024
    causal = torch.tril(torch.ones(ctx, ctx, device="cuda")).view(1, 1, ctx, ctx)
    zero = causal == 0
    for dtype in (torch.float16, torch.bfloat16):
        x = torch.randn(BATCH, HEADS, ctx, ctx, device="cuda", generator=gen).to(dtype)
        esize = x.element_size()
        m, M1, M2 = tr._dense_mask(x, causal, "bench")
        for k in (32, 256):
            def ref_tks():
                v = (x.float() * causal * scale).masked_fill(zero, -FLT_MAX)
                val, idx = torch.topk(v, k, dim=-1)
                return torch.zeros_like(v).scatter_(-1, idx, torch.softmax(val, -1)).to(dtype)
            ms, tms = compare(torch, lambda: tr._topk_softmax_fwd(x, m, M1, M2, k, scale), ref_tks, 20, args.reps)
            emit(dict(op="masked_top_k_softmax", shape=[BATCH, HEADS, ctx, ctx], dtype=str(dtype)[6:], k=k,
                      mask="causal (1, 1, ctx, ctx) fp32"), 2 * x.numel() * esize + causal.numel() * 4, ms, tms)
            ms, tms = compare(torch, lambda: tr._topk_fwd(x, k, tr._TOPK_VALUES), lambda: torch.topk(x, k, dim=-1), 20, args.reps)
            rows = x.numel() // ctx
            emit(dict(op="top_k", shape=[BATCH, HEADS, ctx, ctx], dtype=str(dtype)[6:], k=k),
                 x.numel() * esize + rows * k * (esize + 4), ms, tms)
        del x
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
