#!/usr/bin/env python
"""Kernel time and bandwidth of bias_relu, dropout and embedding_lookup, forward and backward, against the torch code a
user would write for the same math. Needs a CUDA device.

  python scripts/ewops.py [--reps R] [--calls N] [--out FILE]

Cases, bf16 activations with fp32 biases:
  * bias_relu at (N, K) = (16384, 1024) and (16384, 4096) on the last axis and at (K, N) on axis 0, with fast_gelu:
    ours (ew._br_fwd / ew._br_bwd, db reduction included) against x + b followed by z * sigmoid(1.702 z) (axis 0:
    b[:, None]) and its torch.autograd.grad for dx and db; relu at (16384, 4096) against torch.relu(x + b);
  * dropout at keep_prob 0.9 on the same tensors, with a full mask and a (1, T, 1)-style broadcast mask on the tensor
    viewed as (16, 1024, K / 16): ours (mask drawn and applied; the backward applies it to dy) against F.dropout and
    its gradient;
  * embedding_lookup at an enwik8-like (C, K, nIdx) = (256, 512, 16384) and a GPT-2-like (50257, 768, 8192), int64
    indices: ours against F.embedding and its gradient.
Per case and direction one JSON line with ms (the median over R windows of N calls, CUDA events around each window,
after warm-up, alternating with torch), torch_ms, and GB/s and the share of the H100 SXM data-sheet HBM bandwidth
(3.35 TB/s) from the algorithmic bytes: bias_relu and dropout read x and write y (forward), read dy (and y or x) and
write dx (backward); embedding reads the indexed rows and writes y (forward), reads dy and writes dw (backward). Masks,
biases and indices are left out. The first line names the device and its power limit.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from dense_softmax import HBM_TBS, compare, device_label  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F
    from blocksparse_b200 import embed as em
    from blocksparse_b200 import ewops as ew
    if not torch.cuda.is_available():
        raise SystemExit("scripts/ewops.py needs a CUDA device")
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power})]
    print(lines[0], flush=True)

    def emit(rec, ours, ref, nbytes):
        ms, tms = compare(torch, ours, ref, args.calls, args.reps)
        gbs = nbytes / (ms * 1e6)
        rec.update({"ms": round(ms, 4), "torch_ms": round(tms, 4), "GB/s": round(gbs),
                    "hbm_share": round(gbs / (HBM_TBS * 1e3), 3), "speedup": round(tms / ms, 2)})
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)

    dt = torch.bfloat16
    for N, K in ((16384, 1024), (16384, 4096)):
        for axis in (-1, 0):
            shape = (N, K) if axis == -1 else (K, N)
            x = torch.randn(shape, device="cuda", dtype=dt)
            dy = torch.randn_like(x)
            b = torch.randn(K, device="cuda")
            ax = 1 if axis == -1 else 0
            acts = [("fast_gelu", ew.ACT_FAST_GELU)] + ([("relu", ew.ACT_RELU)] if K == 4096 and axis == -1 else [])
            for act_name, act in acts:
                a = (ax, N, K, act)
                y = ew._br_fwd(x, b, *a)
                src = y if act == ew.ACT_RELU else x

                def torch_fwd(xr, br):
                    z = xr + (br.to(dt) if axis == -1 else br.to(dt)[:, None])
                    return torch.relu(z) if act == ew.ACT_RELU else z * torch.sigmoid(1.702 * z)
                xr, br = x.detach().clone().requires_grad_(), b.detach().clone().requires_grad_()
                yr = torch_fwd(xr, br)
                rec = dict(op="bias_relu", act=act_name, axis=axis, shape=list(shape), dtype="bfloat16")
                nb = x.numel() * x.element_size()
                emit(dict(rec, dir="forward"), lambda: ew._br_fwd(x, b, *a), lambda: torch_fwd(x, b), 2 * nb)
                emit(dict(rec, dir="backward"), lambda: ew._br_bwd(dy, src, b, *a),
                     lambda: torch.autograd.grad(yr, (xr, br), dy, retain_graph=True), 3 * nb)
                del y, xr, yr
            del x, dy

    for N, K in ((16384, 1024), (16384, 4096)):
        x = torch.randn(N, K, device="cuda", dtype=dt)
        dy = torch.randn_like(x)
        nb = x.numel() * x.element_size()
        for bcast in (False, True):
            xs = x.view(16, N // 16, K) if bcast else x
            ms = (1, N // 16, 1) if bcast else None
            M = N // 16 if bcast else x.numel()
            shape, strides = tuple(xs.shape), ew._mask_strides(xs, ms or tuple(xs.shape))
            mask = ew._gen_mask(xs, M, 0.9)
            xr = xs.detach().clone().requires_grad_()
            yr = F.dropout(xr, 0.1)
            rec = dict(op="dropout", keep_prob=0.9, shape=list(xs.shape), mask_shape=list(ms) if ms else None,
                       dtype="bfloat16")
            emit(dict(rec, dir="forward"), lambda: ew._apply_mask(xs, ew._gen_mask(xs, M, 0.9), shape, strides, 0.9),
                 lambda: F.dropout(xs, 0.1), 2 * nb)
            emit(dict(rec, dir="backward"), lambda: ew._apply_mask(dy.view(shape), mask, shape, strides, 0.9),
                 lambda: torch.autograd.grad(yr, xr, dy.view(shape), retain_graph=True), 2 * nb)
            del xr, yr

    for C, K, n in ((256, 512, 16384), (50257, 768, 8192)):
        emb = torch.randn(C, K, device="cuda", dtype=dt)
        idx = torch.randint(0, C, (n,), device="cuda")
        dy = torch.randn(n, K, device="cuda", dtype=dt)
        er = emb.detach().clone().requires_grad_()
        yr = F.embedding(idx, er)
        rec = dict(op="embedding_lookup", C=C, K=K, nIdx=n, dtype="bfloat16")
        nb = n * K * emb.element_size()
        emit(dict(rec, dir="forward"), lambda: em._emb_fwd(emb, idx), lambda: F.embedding(idx, emb), 2 * nb)
        emit(dict(rec, dir="backward"), lambda: em._emb_bwd(dy, idx, C, K),
             lambda: torch.autograd.grad(yr, er, dy, retain_graph=True), nb + C * K * emb.element_size())
        del emb, dy, er, yr
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
