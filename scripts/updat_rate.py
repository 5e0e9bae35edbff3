#!/usr/bin/env python
"""Updat kernel time and the rate at which it stages operand bytes from L2, at BASELINE configs[1] (4096 x 4096,
block 32, N = 4096, bf16, feature axis 1) for 5 / 10 / 25 / 50 / 100 % density.  Needs a CUDA device.

  python scripts/updat_rate.py [--reps R]

Staged bytes per call are counted from the updat schedule the op launches with (lut.py:build_updat_schedule): per
64 minibatch rows every tile stages its 128-feature activation group (16 KB) and its n_act kept output-gradient
blocks (bs x 64 x 2 bytes each).  Time: CUDA events over R back-to-back calls after a warm-up, inputs rotating over
three sets larger than L2 (as bench.py's per-op timings).  Rate = staged bytes / time.
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import BS, C, K, N_PER_GPU, SEED, make_layout  # noqa: E402

DENSITIES = (0.05, 0.10, 0.25, 0.50, 1.00)
KCHUNK = 64          # minibatch rows per pipeline stage of the updat kernel


def staged_bytes(sched, bsize, N, pcount=1):
    """Bytes the updat kernel stages per call: every tile, per KCHUNK rows, 128 x-features + n_act dy blocks (16-bit)."""
    n_tiles, rec_ints = int(sched[0]), int(sched[3])
    n_act = sched[4:4 + n_tiles * rec_ints].reshape(n_tiles, rec_ints)[:, 1].astype(np.int64)
    per_stage = 128 * KCHUNK * 2 + n_act * bsize * KCHUNK * 2
    return int(per_stage.sum()) * -(-N // KCHUNK) * pcount, n_tiles, float(n_act.mean())


def device_label():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        out = ""
    return "%s, power limit %s" % (name, out or "unknown")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    args = ap.parse_args()
    if args.reps < 50:
        sys.exit("updat_rate.py: use at least 50 repetitions")
    import torch
    if not torch.cuda.is_available():
        sys.exit("updat_rate.py needs a CUDA device")
    from blocksparse_b200 import BlocksparseMatMul, _lib

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gen = torch.Generator(device=dev).manual_seed(SEED)
    N = N_PER_GPU
    Xs = [(torch.randn((N, C), generator=gen, device=dev) * 0.1).bfloat16() for _ in range(3)]
    Es = [(torch.randn((N, K), generator=gen, device=dev) * 0.1).bfloat16() for _ in range(3)]
    print("updat, %dx%d block %d N %d bf16 axis 1, %s" % (C, K, BS, N, device_label()))
    print("%8s %6s %6s %8s %10s %12s %10s  %s" % ("density", "blocks", "tiles", "n_act", "ms", "staged GB", "TB/s", "kernel"))
    for d in DENSITIES:
        bsmm = BlocksparseMatMul(make_layout(d), block_size=BS, feature_axis=1)
        sched = bsmm._device_luts(dev)["updat_sched"].cpu().numpy()
        nbytes, n_tiles, mean_act = staged_bytes(sched, BS, N)
        for i in range(5):
            bsmm.updat([Xs[i % 3]], [Es[i % 3]])
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(args.reps):
            bsmm.updat([Xs[i % 3]], [Es[i % 3]])
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / args.reps
        print("%7d%% %6d %6d %8.2f %10.4f %12.3f %10.2f  %s" % (round(d * 100), bsmm.blocks, n_tiles, mean_act, ms,
                                                               nbytes / 1e9, nbytes / (ms * 1e-3) / 1e12, _lib.last_kernel()),
              flush=True)
    err = _lib.device_error()
    if err:
        sys.exit("device error %d after the updat runs" % err)


if __name__ == "__main__":
    main()
