#!/usr/bin/env python
"""What attention dropout costs in the fused kernels, at BASELINE configs[2] (batch 4, heads 16, ctx 4096, block 64, the
local + strided causal layout with 453 blocks, fp16) for head_state 64 and 128. Needs a CUDA device.

  python scripts/attention_dropout.py [--reps R]

Three modes alternate in one run, R steps each:
  fused_kp1    attention(..., fused_backward=True), keep_prob 1.0;
  fused_kp09   the same with keep_prob 0.9 (the dropout instantiations of the three fused kernels);
  chain_kp09   query_key_op -> masked_softmax -> ewops.dropout(keep_prob 0.9) -> weight_value_op and its backward.
Per head_state it prints one JSON line with, per mode, the forward + backward and backward-only times (ms, median of R;
CUDA events), the peak memory the backward allocates on top of what the forward left, and for the fused modes each
fused kernel's device time (torch.profiler, median over R calls); and the device name and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BATCH, HEADS, BS, NB, KP = 4, 16, 64, 64, 0.9
MODES = ("fused_kp1", "fused_kp09", "chain_kp09")


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
    from blocksparse_b200 import ewops
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(0)
    q, k, v, dy = ((torch.rand((BATCH, NB * BS, HEADS * hs), generator=gen, device=dev) * 2 - 1).half() for _ in range(4))
    scale = 1.0 / np.sqrt(hs)
    ins = [t.clone().requires_grad_() for t in (q, k, v)]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def forward(mode):
        if mode == "chain_kp09":
            p = bst.masked_softmax(bst.query_key_op(ins[0], ins[1]), scale)
            return bst.weight_value_op(ewops.dropout(p, KP)[0], ins[2])
        return bst.attention(*ins, scale=scale, fused_backward=True, keep_prob=1.0 if mode == "fused_kp1" else KP)

    def step(mode):
        for t in ins:
            t.grad = None
        ev[0].record()
        y = forward(mode)
        ev[1].record()
        y.backward(dy)
        ev[2].record()
        ev[2].synchronize()
        return ev[0].elapsed_time(ev[2]), ev[1].elapsed_time(ev[2])

    for mode in MODES:                   # warm-up: LUT upload, tensor maps, allocator
        for _ in range(3):
            step(mode)
    times = {m: [] for m in MODES}
    for _ in range(reps):
        for mode in MODES:
            times[mode].append(step(mode))

    mem = {}
    for mode in MODES:
        for t in ins:
            t.grad = None
        y = forward(mode)
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        y.backward(dy)
        torch.cuda.synchronize()
        mem[mode] = (torch.cuda.max_memory_allocated() - before) / 2 ** 20
        del y

    from torch.profiler import ProfilerActivity, profile
    state = torch.tensor([1234, 0], dtype=torch.int64, device=dev)
    kern = {}
    for mode, kp in (("fused_kp1", 1.0), ("fused_kp09", KP)):
        o, m, l = bst._attention_train(q, k, v, scale, None, kp, state)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                bst._attention_train(q, k, v, scale, None, kp, state)
                bst._attention_grad(q, k, v, o, dy, m, l, scale, None, kp, state)
            torch.cuda.synchronize()
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and "wgmma_bst_attention" in e.name:
                name = e.name.split("<")[0].split("(")[0].replace("void ", "").replace("bsmm::", "")
                name += "_train" if name == "wgmma_bst_attention" else ""
                kern.setdefault(mode, {}).setdefault(name, []).append(e.device_time_total / 1000.0)

    med = lambda xs: float(np.median(xs))
    return {
        "head_state": hs, "reps": reps, "keep_prob": KP,
        "ms": {m: {"fwd_bwd": med([t[0] for t in times[m]]), "bwd": med([t[1] for t in times[m]])} for m in MODES},
        "kernel_ms": {m: {n: med(v) for n, v in sorted(d.items())} for m, d in kern.items()},
        "bwd_peak_extra_mib": mem,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("attention_dropout.py needs a CUDA device")
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
