#!/usr/bin/env python
"""Time of one optimizer step -- clip_by_global_norm + AdamOptimizer.step -- against torch's fused baseline
(torch.nn.utils.clip_grad_norm_(foreach=True) + torch.optim.Adam(fused=True)). Needs a CUDA device.

  python scripts/optimizer_step.py [--reps R] [--calls N] [--out FILE]

Workloads:
  * gpt2-small: the parameter list of GPT-2 small (148 tensors, 124.4 M parameters: embeddings, 12 blocks of
    ln / attention / MLP weights and biases, final ln), fp32 params with fp32 grads;
  * bsmm-gated: the bench layer's weight, 4096 x 4096 features in 32 x 32 blocks at 25 % density (4096 blocks, 4.2 M
    parameters), gated with about half of the gates 0 (AdamOptimizer(gated=True); torch has no gated step and moves all).
Per workload and optimizer one JSON line with:
  * ms: median over R windows of N steps (CUDA events around the window, after warm-up), ours and torch's windows
    alternating;
  * host_us: host wall time per step call, i.e. the enqueue time (median over the same windows, no synchronisation);
  * GB/s and hbm_share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s), from the algorithmic bytes: the grad read
    twice (norm and step), the param read and written, and both moments read and written (4 bytes each in fp32, 2 bytes
    each as 16-bit codes). Pruned blocks are counted as if they were touched, so the gated rate is a lower bound.
The first line names the device and its power limit.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from dense_softmax import HBM_TBS, device_label  # noqa: E402


def gpt2_small_shapes(vocab=50257, ctx=1024, d=768, layers=12):
    shapes = [(vocab, d), (ctx, d)]
    for _ in range(layers):
        shapes += [(d,), (d,), (d, 3 * d), (3 * d,), (d, d), (d,), (d,), (d,), (d, 4 * d), (4 * d,), (4 * d, d), (d,)]
    return shapes + [(d,), (d,)]


def window(torch, fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    host = (time.perf_counter() - t0) / n
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n, host * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    import numpy as np
    import torch
    from blocksparse_b200 import AdamOptimizer, BlocksparseMatMul, clip_by_global_norm
    if not torch.cuda.is_available():
        raise SystemExit("scripts/optimizer_step.py needs a CUDA device")
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power})]
    print(lines[0], flush=True)
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    lay = (rng.random((128, 128)) < 0.25).astype(np.int32)
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=1)
    workloads = [("gpt2-small", gpt2_small_shapes(), False), ("bsmm-gated", [bsmm.w_shape], True)]
    for wl, shapes, gated in workloads:
        for fp16 in (False, True):
            ps = [(torch.randn(s, device="cuda") * 0.02) for s in shapes]
            gs = [torch.randn_like(p) * 1e-3 for p in ps]
            if gated:
                ps[0].gate = (torch.rand(ps[0].shape[0], device="cuda") < 0.5).float()
            tps = [p.clone().requires_grad_() for p in ps]
            for tp, g in zip(tps, gs):
                tp.grad = g.clone()
            ours = AdamOptimizer(ps, learning_rate=1e-4, gated=gated, fp16=fp16)
            theirs = torch.optim.Adam(tps, lr=1e-4, fused=True)

            def ours_step():
                _, scale = clip_by_global_norm(gs, clip_norm=1.0)
                ours.step(grads=gs, norm_scale=scale)

            def torch_step():
                torch.nn.utils.clip_grad_norm_(tps, 1.0, foreach=True)
                theirs.step()

            for fn in (ours_step, torch_step):
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            t = {"ours": [], "torch": []}
            for _ in range(args.reps):
                t["ours"].append(window(torch, ours_step, args.calls))
                t["torch"].append(window(torch, torch_step, args.calls))
            n = sum(p.numel() for p in ps)
            mom = 2 if fp16 else 4
            coded = sum(p.numel() for p in ps if p.numel() >= 8192) if fp16 else 0
            ours_bytes = n * (4 * 2 + 4 * 2) + 2 * 2 * (mom * coded + 4 * (n - coded))
            torch_bytes = n * (4 * 2 + 4 * 2 + 4 * 2 * 2)
            for who, nbytes in (("ours", ours_bytes), ("torch", torch_bytes)):
                if who == "torch" and fp16:
                    continue                                  # the torch baseline is the same for both moment formats
                ms = sorted(x[0] for x in t[who])[args.reps // 2]
                host = sorted(x[1] for x in t[who])[args.reps // 2]
                gbs = nbytes / (ms * 1e6)
                rec = {"op": "clip+adam", "workload": wl, "impl": who, "tensors": len(ps), "params": n,
                       "moments": ("16-bit" if fp16 else "fp32") if who == "ours" else "fp32", "ms": round(ms, 4),
                       "host_us": round(host, 1), "GB/s": round(gbs), "hbm_share": round(gbs / (HBM_TBS * 1e3), 3)}
                if who == "ours":
                    rec["torch_ms"] = round(sorted(x[0] for x in t["torch"])[args.reps // 2], 4)
                lines.append(json.dumps(rec))
                print(lines[-1], flush=True)
            del ps, gs, tps, ours, theirs
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
