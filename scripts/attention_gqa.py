#!/usr/bin/env python
"""Time grouped-query attention (kv_heads < heads) against the same op on k and v expanded to heads heads, on the card
it runs on. Needs a CUDA device.

  python scripts/attention_gqa.py [--reps R] [--quick]

Layouts (heads 16, ctx 4096 rows, block size 64, causal mask inside diagonal blocks): cfg3 (local_strided_layout,
local 4, stride 8) and tril. Over head_state 64 / 128 and kv_heads 16 / 4 / 1, fp16:
  decode     attention_decode of n = 1 row at the end of the context, batch 1 / 8 / 64, captured in a CUDA graph of 20
             calls: ms per call (median of R replays, CUDA events) and GB/s of the bytes the kernels read (the K and V
             tiles each CTA stages, plus q and o);
  training   attention(fused_backward=True) forward + backward at batch 1: ms (median of R, CUDA events) and the
             backward's peak memory above what it started with.
Each GQA case alternates with the same op on k and v expanded to 16 heads (contiguous copies made beforehand, as a
user without kv_heads would pass them). One JSON line per case; the first names the device and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HEADS, CTX, BS = 16, 4096, 64
CALLS = 20
SLOTS = 64                     # row slots of one decode CTA (csrc/tc_bst_decode.cuh)


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


def decode_bytes(bst, kv, batch, hs, positions):
    """K and V tiles staged: once per LUT entry and CTA, a CTA serving min(g, 64 / n) query heads of a group (n = 1),
    plus q and o."""
    g = HEADS // kv
    ctas_per_group = -(-g // min(g, SLOTS))
    total = 0
    for p in positions:
        total += 2 * len(bst.nn_list[0][p // BS]) * BS * hs * 2 * kv * ctas_per_group
    return total + 2 * batch * HEADS * hs * 2


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


def expand(x, kv):
    B, C, S = x.shape
    hs = S // kv
    return x.reshape(B, C, kv, 1, hs).expand(B, C, kv, HEADS // kv, hs).reshape(B, C, HEADS * hs).contiguous()


def graph_of(torch, step):
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
    return g


def measure_decode(torch, bst, name, hs, kv, batch, reps):
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(0)
    dtype = torch.float16
    k, v = ((torch.rand((batch, CTX, kv * hs), generator=gen, device=dev) * 2 - 1).to(dtype) for _ in range(2))
    q = (torch.rand((batch, 1, HEADS * hs), generator=gen, device=dev) * 2 - 1).to(dtype)
    positions = [CTX - 1 - 3 * b % BS for b in range(batch)]
    pos = torch.tensor(positions, dtype=torch.int32, device=dev)
    kx, vx = expand(k, kv), expand(v, kv)
    g_gqa = graph_of(torch, lambda: bst.attention_decode(q, k, v, pos, scale=0.125, kv_heads=kv))
    g_mha = graph_of(torch, lambda: bst.attention_decode(q, kx, vx, pos, scale=0.125))
    t_gqa, t_mha = [], []
    for _ in range(reps):                              # alternate, so clocks and L2 state hit both alike
        t_gqa.append(median_ms(torch, g_gqa.replay, 1) / CALLS)
        t_mha.append(median_ms(torch, g_mha.replay, 1) / CALLS)
    ms, ms_x = float(np.median(t_gqa)), float(np.median(t_mha))
    nb, nb_x = decode_bytes(bst, kv, batch, hs, positions), decode_bytes(bst, HEADS, batch, hs, positions)
    row = {"op": "decode", "layout": name, "head_state": hs, "kv_heads": kv, "batch": batch, "n": 1,
           "gqa_ms": round(ms, 5), "gqa_MB": round(nb / 1e6, 3), "gqa_GB_per_s": round(nb / ms / 1e6, 1),
           "expanded_ms": round(ms_x, 5), "expanded_MB": round(nb_x / 1e6, 3),
           "expanded_GB_per_s": round(nb_x / ms_x / 1e6, 1), "speedup": round(ms_x / ms, 3)}
    del g_gqa, g_mha
    return row


def measure_train(torch, bst, name, hs, kv, reps):
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(1)
    dtype = torch.float16
    q, dy = ((torch.rand((1, CTX, HEADS * hs), generator=gen, device=dev) * 2 - 1).to(dtype) for _ in range(2))
    k, v = ((torch.rand((1, CTX, kv * hs), generator=gen, device=dev) * 2 - 1).to(dtype) for _ in range(2))
    kx, vx = expand(k, kv), expand(v, kv)

    def step(kk, vv, kv_heads):
        ins = [t.detach().requires_grad_() for t in (q, kk, vv)]
        y = bst.attention(*ins, scale=0.125, fused_backward=True, kv_heads=kv_heads)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        y.backward(dy)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    gqa = lambda: step(k, v, kv)
    mha = lambda: step(kx, vx, None)
    gqa(), mha()
    t_gqa, t_mha = [], []
    for _ in range(reps):
        t_gqa.append(median_ms(torch, gqa, 1))
        t_mha.append(median_ms(torch, mha, 1))
    return {"op": "fwd+bwd", "layout": name, "head_state": hs, "kv_heads": kv, "batch": 1,
            "gqa_ms": round(float(np.median(t_gqa)), 4), "expanded_ms": round(float(np.median(t_mha)), 4),
            "gqa_bwd_peak_extra_MB": round(gqa() / 2 ** 20, 2), "expanded_bwd_peak_extra_MB": round(mha() / 2 ** 20, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="head_state 64 and the cfg3 layout only")
    args = ap.parse_args()
    import torch
    from blocksparse_b200 import BlocksparseTransformer
    from blocksparse_b200.layouts import local_strided_layout
    if not torch.cuda.is_available():
        sys.exit("attention_gqa.py needs a CUDA device")
    name, power = device_label()
    print(json.dumps({"device": name, "power_limit": power}), flush=True)
    nb = CTX // BS
    layouts = [("cfg3", local_strided_layout(nb))]
    if not args.quick:
        layouts.append(("tril", np.tril(np.ones((nb, nb), np.int32))))
    for lname, lay in layouts:
        bst = BlocksparseTransformer(lay, BS, heads=HEADS, mask_callback=causal)
        for hs in ((64,) if args.quick else (64, 128)):
            for kv in (16, 4, 1):
                for batch in (1, 8, 64):
                    print(json.dumps(measure_decode(torch, bst, lname, hs, kv, batch, args.reps)), flush=True)
                print(json.dumps(measure_train(torch, bst, lname, hs, kv, args.reps)), flush=True)


if __name__ == "__main__":
    main()
