#!/usr/bin/env python
"""fprop / bprop of the default 32 x 32 wgmma route with the tile forced: one output block per CTA (csrc/tc.cuh) against
every grouped tile the library has (csrc/tc_xprop2.cuh: tc_xprop_grouped_kernel).  Needs a CUDA device.

  python scripts/xprop_tiles.py [--out DIR] [--rounds R] [--window S]

Workloads: bench.py's shape (4096 x 4096, block 32, N = 4096, bf16, feature axis 1) at 5 / 10 / 25 / 50 / 100 % density,
its Barabasi-Albert layout, feature axis 0, fp16, and N = 2048 (cfg4's 20 % layout) and 32768 (cfg5).  Inputs rotate over
sets larger than L2.  Every variant of a line is timed in the same process, alternating within each round: CUDA events
over a window of at least S seconds (default 0.2), median of R rounds (default 7) with min and max.

Per line it prints the bytes the kernel is modelled to stage from L2 into shared memory (lut.xprop_staged_bytes: an 8 KB
activation tile per LUT entry -- per merged entry for a grouped tile -- plus a 2 KB W block per LUT entry, per 128 rows)
and the rate that makes of the measured time, then which tile lut.pick_xprop_tile selects.  One JSON file goes to DIR.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import BS, C, K, N_PER_GPU, SEED, make_layout  # noqa: E402


def device_label():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=10).stdout.strip()
    return out or "unknown device"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "xprop_tiles"))
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--window", type=float, default=0.2)
    args = ap.parse_args()
    if args.rounds < 7 or args.window < 0.2:
        sys.exit("xprop_tiles.py: use at least 7 rounds and windows of 0.2 s")
    import torch
    if not torch.cuda.is_available():
        sys.exit("xprop_tiles.py needs a CUDA device")
    import blocksparse_b200.matmul as mm
    from blocksparse_b200 import BlocksparseMatMul, _lib
    from blocksparse_b200.layouts import barabasi_albert_layout
    from blocksparse_b200.lut import xprop_staged_bytes

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gen = torch.Generator(device=dev).manual_seed(SEED)
    tiles = [1] + sorted(mm._GROUPED_VARIANTS)
    label = device_label()
    print(label, flush=True)

    def inputs(N, dtype, axis, sets):
        shape = (lambda f: (N, f)) if axis else (lambda f: (f, N))
        return ([(torch.randn(shape(C), generator=gen, device=dev) * 0.1).to(dtype) for _ in range(sets)],
                [(torch.randn(shape(K), generator=gen, device=dev) * 0.1).to(dtype) for _ in range(sets)])

    def window(fn, reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(reps):
            fn(i)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / reps

    workloads = [("d%d" % round(d * 100), make_layout(d), 1, torch.bfloat16, N_PER_GPU) for d in (0.05, 0.10, 0.25, 0.50, 1.00)]
    workloads += [("barabasi_albert", barabasi_albert_layout(C // BS, 0.25, np.random.default_rng(SEED + 1)), 1, torch.bfloat16, N_PER_GPU),
                  ("axis0", make_layout(0.25), 0, torch.bfloat16, N_PER_GPU),
                  ("fp16", make_layout(0.25), 1, torch.float16, N_PER_GPU),
                  ("cfg4_N2048", make_layout(0.20, seed=1238), 1, torch.bfloat16, 2048),
                  ("cfg5_N32768", make_layout(0.25), 1, torch.bfloat16, 32768)]
    results = []
    cache = {}
    print("%-16s %-5s %4s %9s %9s %9s %10s %8s %5s" % ("workload", "op", "tile", "ms", "min", "max", "staged GB", "TB/s", "pick"))
    for name, lay, axis, dtype, N in workloads:
        key = (N, dtype, axis)
        if key not in cache:
            cache.clear()
            cache[key] = inputs(N, dtype, axis, 3 if N <= 4096 else 2)
        Xs, Es = cache[key]
        bsmm = BlocksparseMatMul(lay, block_size=BS, feature_axis=axis)
        W = (torch.randn(bsmm.w_shape, generator=gen, device=dev) * 0.01).to(dtype)
        for bprop, ins in ((False, Xs), (True, Es)):
            op = bsmm.bprop if bprop else bsmm.fprop
            fn = lambda i: op(ins[i % len(ins)], W)
            mm._XPROP_TILE = None
            pick = bsmm.xprop_tile(bprop, N, dev)
            ref, reps = None, {}
            for t in tiles:                                 # warm up, size the window, and compare the results
                mm._XPROP_TILE = t
                out = op(ins[0], W)
                assert _lib.last_kernel() == "wgmma_xprop_bs32", _lib.last_kernel()
                if ref is None:
                    ref = out
                elif not torch.equal(ref, out):
                    sys.exit("%s %s: tile %d differs from one block per CTA" % (name, "bprop" if bprop else "fprop", t))
                reps[t] = max(10, int(np.ceil(args.window / (window(fn, 10) * 1e-3))))
            times = {t: [] for t in tiles}
            for _ in range(args.rounds):
                for t in tiles:
                    mm._XPROP_TILE = t
                    times[t].append(window(fn, reps[t]))
            mm._XPROP_TILE = None
            for t in tiles:
                entries = bsmm.blocks if t == 1 else bsmm._wide_schedule(bsmm._device_luts(dev), dev, bprop, t)[3]
                nbytes = xprop_staged_bytes(bsmm.blocks, entries, N)[0 if t == 1 else 1]
                ms = float(np.median(times[t]))
                rec = {"workload": name, "op": "bprop" if bprop else "fprop", "tile": t, "ms": ms, "ms_min": min(times[t]),
                       "ms_max": max(times[t]), "staged_bytes": nbytes, "staged_tbs": nbytes / (ms * 1e-3) / 1e12,
                       "picked": pick, "nnz_blocks": bsmm.blocks, "N": N, "axis": axis, "dtype": str(dtype)}
                results.append(rec)
                print("%-16s %-5s %4d %9.4f %9.4f %9.4f %10.3f %8.2f %5s" % (name, rec["op"], t, ms, rec["ms_min"], rec["ms_max"],
                                                                        nbytes / 1e9, rec["staged_tbs"], pick if t == tiles[0] else ""),
                      flush=True)
    err = _lib.device_error()
    if err:
        sys.exit("device error %d after the xprop runs" % err)
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "xprop_tiles.json")
    with open(path, "w") as f:
        json.dump({"device": label, "rounds": args.rounds, "window_s": args.window, "results": results}, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
