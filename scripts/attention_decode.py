#!/usr/bin/env python
"""Time BlocksparseTransformer.attention_decode steps, captured in a CUDA graph, on the card it runs on. Needs a CUDA
device.

  python scripts/attention_decode.py [--reps R] [--quick]

Layouts (heads 16, ctx 4096 rows, causal mask inside diagonal blocks):
  cfg3   local_strided_layout (local 4, stride 8), the layout of BASELINE configs[2];
  tril   dense causal tril, whose last query block holds ctx / bs key blocks.
Over head_state 64 / 128, fp16 / bf16, batch 1 / 8 / 64, n = 1 / 16 and block size 32 / 64, with the chunk's rows at
the end of the context. Per configuration one JSON line: the time per decode call (median over R graph replays of 20
calls each; CUDA events), the achieved bandwidth in algorithmic bytes (the K and V rows of every LUT entry of the
rows' query blocks, plus q and o) against 3.35 TB/s, and the time of today's alternative: attention() over the full
context (eager, median of R calls) from which the rows would be kept. The first line names the device and its power
limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HEADS, CTX, PEAK = 16, 4096, 3.35e12
CALLS = 20


def device_label():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        out = ""
    return name, out or "unknown"


def causal(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    m = np.ones(blk_shape, dtype=bool)
    return np.tril(m) if qry_idx == key_idx else m


def algorithmic_bytes(bst, batch, n, hs, positions):
    """K and V rows of every LUT entry of the query blocks the rows touch (per head, 2 bytes each), plus q and o."""
    bs, total = bst.blk_size, 0
    for p in positions:
        for qb in sorted({(p + i) // bs for i in range(n)}):
            for h in range(HEADS):
                total += 2 * len(bst.nn_list[h if bst.lut_heads > 1 else 0][qb]) * bs * hs * 2
    return total + 2 * batch * n * HEADS * hs * 2


def median_ms(torch, fn, reps):
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def measure(torch, bst, name, dtype, hs, batch, n, reps, full_cache):
    dev = torch.device("cuda", 0)
    S = HEADS * hs
    gen = torch.Generator(device=dev).manual_seed(0)
    k, v = ((torch.rand((batch, CTX, S), generator=gen, device=dev) * 2 - 1).to(dtype) for _ in range(2))
    q = (torch.rand((batch, n, S), generator=gen, device=dev) * 2 - 1).to(dtype)
    positions = [CTX - n - 3 * b % bst.blk_size for b in range(batch)]
    pos = torch.tensor(positions, dtype=torch.int32, device=dev)
    step = lambda: bst.attention_decode(q, k, v, pos, scale=0.125)
    step()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            for _ in range(CALLS):
                step()
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    ms = median_ms(torch, g.replay, reps) / CALLS
    nbytes = algorithmic_bytes(bst, batch, n, hs, positions)
    row = {"layout": name, "bs": bst.blk_size, "dtype": str(dtype).replace("torch.", ""), "head_state": hs,
           "batch": batch, "n": n, "decode_ms": round(ms, 5), "algorithmic_MB": round(nbytes / 1e6, 3),
           "GB_per_s": round(nbytes / ms / 1e6, 1), "share_of_3.35TB_per_s": round(nbytes / ms / 1e-3 / PEAK, 3)}
    if full_cache:
        qf = (torch.rand((batch, CTX, S), generator=gen, device=dev) * 2 - 1).to(dtype)
        att = lambda: bst.attention(qf, k, v, scale=0.125)
        att()
        row["attention_full_ms"] = round(median_ms(torch, att, reps), 4)
    del k, v, q
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="fp16 only, batch 1 / 64, head_state 64")
    args = ap.parse_args()
    import torch
    from blocksparse_b200 import BlocksparseTransformer
    from blocksparse_b200.layouts import local_strided_layout
    if not torch.cuda.is_available():
        sys.exit("attention_decode.py needs a CUDA device")
    name, power = device_label()
    print(json.dumps({"device": name, "power_limit": power}), flush=True)
    dtypes = (torch.float16,) if args.quick else (torch.float16, torch.bfloat16)
    batches = (1, 64) if args.quick else (1, 8, 64)
    states = (64,) if args.quick else (64, 128)
    for bs in (64, 32):
        nb = CTX // bs
        for lname, lay in (("cfg3", local_strided_layout(nb)), ("tril", np.tril(np.ones((nb, nb), np.int32)))):
            bst = BlocksparseTransformer(lay, bs, heads=HEADS, mask_callback=causal)
            for dtype in dtypes:
                for hs in states:
                    for batch in batches:
                        for n in (1, 16):
                            full = n == 1 and dtype == dtypes[0] and batch != 64
                            print(json.dumps(measure(torch, bst, lname, dtype, hs, batch, n, args.reps, full)),
                                  flush=True)


if __name__ == "__main__":
    main()
