#!/usr/bin/env python
"""Kernel time of dw_matmul_large_n (U = X^T E in fp32, fp16 inputs) beside what a user could run instead: cuBLAS
through torch.matmul(x.t(), e) (16-bit output), BlocksparseMatMul.updat with a fully dense layout (block size 32,
feature axis 1, fp32 dW in block format), and the reference's own Gemm_TN kernel (oracle/_ref/libbsref.so, when built).
Needs a CUDA device.

  python scripts/dw_matmul.py [--reps R] [--out FILE]

Shapes (N, C, K): the reference test's (1M, 32, 32), (128K, 128, 128), (32K, 512, 512); a dense layer's
(65536, 1024, 1024); (4096, 4096, 4096) and (65536, 4096, 4096).
Each implementation's calls for one shape are captured in one CUDA graph that walks copies of the inputs, enough that
they do not fit the 50 MB L2 together, so every call reads its operands from HBM. Times are the median over R windows
(CUDA events, after warm-up, implementations alternating) per call, with the spread (max - min window). TFLOP/s is
2 N C K over the time. The bound is the larger of 2 N C K over 989 TFLOP/s (dense 16-bit) and the bytes the op must
move -- N (C + K) 2 bytes read, C K 4 bytes written -- over 3.35 TB/s (the H100 SXM data sheet); `bound` names which
one applies and `share` is that least time over the measured one. The first line names the device and its power limit.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from conv_bias import graphed  # noqa: E402
from dense_softmax import HBM_TBS, device_label, window  # noqa: E402

SHAPES = [(1 << 20, 32, 32), (1 << 17, 128, 128), (1 << 15, 512, 512), (65536, 1024, 1024), (4096, 4096, 4096),
          (65536, 4096, 4096)]
TC_TFLOPS = 989.0
L2_BYTES = 50 << 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out")
    args = ap.parse_args()
    import numpy as np
    import torch
    from blocksparse_b200 import BlocksparseMatMul, dw_matmul_large_n
    if not torch.cuda.is_available():
        raise SystemExit("scripts/dw_matmul.py needs a CUDA device")
    ref = None
    try:
        from oracle import ref_matmul as ref
        if ref.missing():
            ref = None
    except Exception:
        ref = None
    name, power = device_label(torch)
    lines = [{"device": name, "power_limit": power, "reference_kernel": ref is not None}]
    print(json.dumps(lines[0]), flush=True)
    for N, C, K in SHAPES:
        pair = N * (C + K) * 2
        copies = max(2, min(8, -(-2 * L2_BYTES // pair)))
        g = torch.Generator(device="cuda").manual_seed(0)
        xs = [(torch.randn((N, C), generator=g, device="cuda") + 0.1).half() for _ in range(copies)]
        es = [(torch.randn((N, K), generator=g, device="cuda") + 0.2).half() for _ in range(copies)]
        bsmm = BlocksparseMatMul(np.ones((C // 32, K // 32), np.int32), block_size=32, feature_axis=1)
        impls = {
            "dw_matmul_large_n": lambda: [dw_matmul_large_n(x, e) for x, e in zip(xs, es)],
            "cublas_matmul": lambda: [torch.matmul(x.t(), e) for x, e in zip(xs, es)],
            "dense_updat": lambda: [bsmm.updat(x, e, dw_dtype=torch.float32) for x, e in zip(xs, es)],
        }
        if ref is not None:
            u = torch.empty((C, K), dtype=torch.float32, device="cuda")
            fn = ref._fn()

            def run_ref():
                st = torch.cuda.current_stream().cuda_stream
                for x, e in zip(xs, es):
                    rc = fn(1, u.data_ptr(), x.data_ptr(), e.data_ptr(), C, K, N, st)
                    if rc != 0:
                        raise RuntimeError("bsref_dw_matmul_large_n: CUDA error %d" % rc)
            impls["reference_gemm_tn"] = run_ref
        # agreement on the first copy, so that the times compare the same math
        u0 = dw_matmul_large_n(xs[0], es[0]).double()
        scale = u0.abs().mean().item()
        diffs = {"cublas_matmul": (torch.matmul(xs[0].t(), es[0]).double() - u0).abs().max().item() / scale}
        fns = {k: graphed(torch, f) for k, f in impls.items()}
        for f, _ in fns.values():
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        calls = max(1, int(round(2e-2 / max(1e-6, window(torch, fns["dw_matmul_large_n"][0], 1) * 1e-3))))
        t = {k: [] for k in fns}
        for _ in range(args.reps):
            for k, (f, _) in fns.items():
                t[k].append(window(torch, f, calls) / copies)
        flops = 2.0 * N * C * K
        nbytes = N * (C + K) * 2 + C * K * 4
        t_flop, t_mem = flops / (TC_TFLOPS * 1e12), nbytes / (HBM_TBS * 1e12)
        for k, v in t.items():
            ms = sorted(v)[len(v) // 2]
            rec = {"N": N, "C": C, "K": K, "impl": k, "graph": fns[k][1], "ms": round(ms, 5),
                   "spread_ms": round(max(v) - min(v), 5), "tflops": round(flops / (ms * 1e-3) / 1e12, 1),
                   "bound": "hbm" if t_mem > t_flop else "tensor", "share": round(max(t_flop, t_mem) / (ms * 1e-3), 3)}
            if k in diffs:
                rec["max_diff_vs_ours"] = float("%.3g" % diffs[k])
            lines.append(rec)
            print(json.dumps(rec), flush=True)
        del xs, es, fns, impls
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
