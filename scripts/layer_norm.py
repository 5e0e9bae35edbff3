#!/usr/bin/env python
"""Kernel time and bandwidth of layer_norm and its gradient against the torch code a user would write for the same
math. Needs a CUDA device.

  python scripts/layer_norm.py [--reps R] [--out FILE]

Shapes: 8192 rows at K = 1024, 4096 and 12288 on the last axis; K = 4096 with segments = 4; (K, N) = (4096, 4096) and
(4096, 256) on axis 0; fp16 and bf16, fp32 gain and bias. Per case and direction one JSON line with:
  * ms: median over R windows of N calls (CUDA events around the window, after warm-up) of our op: forward
    (nm._ln_fwd) or backward (nm._ln_bwd, dg / db reduction included);
  * torch_ms: the same for torch, timed in windows alternating with ours: F.layer_norm (axis -1; per segment through a
    view of (rows, segments, L) with the gain applied after, for segments) or x.t() -> F.layer_norm -> .t().contiguous()
    (axis 0), and the backward through torch.autograd.grad of that forward;
  * GB/s and the share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s), from the algorithmic bytes: x read and y
    written (forward); dy and x read and dx written (backward). Gains, biases and statistics are left out.
The first line names the device and its power limit.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from dense_softmax import HBM_TBS, compare, device_label  # noqa: E402

CASES = [(-1, 8192, 1024, 1), (-1, 8192, 4096, 1), (-1, 8192, 12288, 1), (-1, 8192, 4096, 4), (0, 4096, 4096, 1),
         (0, 256, 4096, 1)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F
    from blocksparse_b200 import norms as nm
    if not torch.cuda.is_available():
        raise SystemExit("scripts/layer_norm.py needs a CUDA device")
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power})]
    print(lines[0], flush=True)
    for dtype in (torch.bfloat16, torch.float16):
        for axis, N, K, S in CASES:
            shape = (N, K) if axis == -1 else (K, N)
            x = torch.randn(shape, device="cuda", dtype=dtype)
            dy = torch.randn_like(x)
            g = torch.rand(K, device="cuda") + 0.5
            b = torch.randn(K, device="cuda")
            ax = 1 if axis == -1 else 0
            a = (ax, N, K, S, 1e-6, False)
            y, mean, rstd = nm._ln_fwd(x, g, b, *a)
            L = K // S

            def torch_fwd(xr, gr, br):
                if axis == 0:
                    return F.layer_norm(xr.t(), (K,), gr.to(dtype), br.to(dtype), 1e-6).t().contiguous()
                if S == 1:
                    return F.layer_norm(xr, (K,), gr.to(dtype), br.to(dtype), 1e-6)
                return (F.layer_norm(xr.view(N, S, L), (L,), None, None, 1e-6).view(N, K) * gr.to(dtype) + br.to(dtype))

            xr, gr, br = (t.detach().clone().requires_grad_() for t in (x, g, b))
            yr = torch_fwd(xr, gr, br)

            def torch_bwd():
                torch.autograd.grad(yr, (xr, gr, br), dy, retain_graph=True)
            for direction, ours, ref, nbytes in (
                    ("forward", lambda: nm._ln_fwd(x, g, b, *a), lambda: torch_fwd(x, g, b), 2 * x.numel() * x.element_size()),
                    ("backward", lambda: nm._ln_bwd(x, dy, g, b, mean, rstd, *a), torch_bwd, 3 * x.numel() * x.element_size())):
                ms, tms = compare(torch, ours, ref, args.calls, args.reps)
                gbs = nbytes / (ms * 1e6)
                rec = {"op": "layer_norm", "dir": direction, "axis": axis, "shape": list(shape), "segments": S,
                       "dtype": str(dtype).replace("torch.", ""), "ms": round(ms, 4), "torch_ms": round(tms, 4),
                       "GB/s": round(gbs), "hbm_share": round(gbs / (HBM_TBS * 1e3), 3), "speedup": round(tms / ms, 2)}
                lines.append(json.dumps(rec))
                print(lines[-1], flush=True)
            del x, dy, y, xr, yr
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
