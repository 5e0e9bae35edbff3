#!/usr/bin/env python
"""Block-sparse attention training step, default backward against fused_backward=True, at BASELINE configs[2] (batch 4,
heads 16, ctx 4096, block 64, the local + strided causal layout with 453 blocks, fp16) for head_state 64 and 128.
Needs a CUDA device.

  python scripts/attention_backward.py [--reps R]

Per head_state it prints one JSON line with:
  * forward + backward and backward-only times (ms, median of R; CUDA events), the two modes alternating in one run;
  * the device time of each fused kernel (torch.profiler, median over R calls);
  * the peak memory the backward allocates on top of what the forward left (torch.cuda.max_memory_allocated);
  * the device name and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH, HEADS, BS, NB = 4, 16, 64, 64


def device_label():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        out = ""
    return "%s, power limit %s" % (name, out or "unknown")


def causal(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    m = np.ones(blk_shape, dtype=bool)
    return np.tril(m) if qry_idx == key_idx else m


def measure(torch, bst, hs, reps):
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(0)
    q, k, v, dy = ((torch.rand((BATCH, NB * BS, HEADS * hs), generator=gen, device=dev) * 2 - 1).half() for _ in range(4))
    scale = 1.0 / np.sqrt(hs)
    ins = [t.clone().requires_grad_() for t in (q, k, v)]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def step(fused):
        for t in ins:
            t.grad = None
        ev[0].record()
        y = bst.attention(*ins, scale=scale, fused_backward=fused)
        ev[1].record()
        y.backward(dy)
        ev[2].record()
        ev[2].synchronize()
        return ev[0].elapsed_time(ev[2]), ev[1].elapsed_time(ev[2])

    for fused in (False, True):          # warm-up: LUT upload, tensor maps, allocator
        for _ in range(3):
            step(fused)
    times = {False: [], True: []}
    for _ in range(reps):
        for fused in (False, True):
            times[fused].append(step(fused))

    mem = {}
    for fused in (False, True):
        for t in ins:
            t.grad = None
        y = bst.attention(*ins, scale=scale, fused_backward=fused)
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        y.backward(dy)
        torch.cuda.synchronize()
        mem[fused] = (torch.cuda.max_memory_allocated() - before) / 2 ** 20
        del y

    from torch.profiler import ProfilerActivity, profile
    o, m, l = bst._attention_train(q, k, v, scale, None)
    kern = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            bst._attention_train(q, k, v, scale, None)
            bst._attention_grad(q, k, v, o, dy, m, l, scale, None)
        torch.cuda.synchronize()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "wgmma_bst_attention" in e.name:
            name = e.name.split("<")[0].split("(")[0].replace("void ", "").replace("bsmm::", "")
            name += "_train" if name == "wgmma_bst_attention" else ""
            kern.setdefault(name, []).append(e.device_time_total / 1000.0)

    med = lambda xs: float(np.median(xs))
    return {
        "head_state": hs, "reps": reps,
        "default_ms": {"fwd_bwd": med([t[0] for t in times[False]]), "bwd": med([t[1] for t in times[False]])},
        "fused_ms": {"fwd_bwd": med([t[0] for t in times[True]]), "bwd": med([t[1] for t in times[True]])},
        "kernel_ms": {n: med(v) for n, v in sorted(kern.items())},
        "bwd_peak_extra_mib": {"default": mem[False], "fused": mem[True]},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("attention_backward.py needs a CUDA device")
    from blocksparse_b200 import BlocksparseTransformer
    from blocksparse_b200.layouts import local_strided_layout

    torch.cuda.set_device(0)
    bst = BlocksparseTransformer(local_strided_layout(NB), BS, heads=HEADS, mask_callback=causal)
    print("# %s; batch %d, heads %d, ctx %d, %d blocks, fp16" % (device_label(), BATCH, HEADS, NB * BS, bst.blocks))
    for hs in (64, 128):
        rec = measure(torch, bst, hs, args.reps)
        rec["device"] = device_label()
        print(json.dumps(rec))


if __name__ == "__main__":
    main()
