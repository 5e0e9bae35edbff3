#!/usr/bin/env python
"""Kernel time and bandwidth of softmax_cross_entropy and the transposes against torch. Needs a CUDA device.

  python scripts/cross_entropy.py [--reps R] [--out FILE]

Cross entropy: N = 8192 rows, K in {256, 32768, 50257, 65536, 131072}, fp16 and bf16, int64 labels. For each, the
forward, the backward and forward plus backward, against F.cross_entropy(logits, labels, reduction="none") on the same
dtype (its backward through autograd). Transposes: transpose_0213 of (16, 1024, 16, 64) and (16, 1024, 16, 4) and
transpose_2d of (8192, 8192), fp16, against permute().contiguous() / .t().contiguous() and against a copy_ of the same
size, the practical ceiling. Per case one JSON line with:
  * ms: median over R windows of launches (CUDA events around each window, after warm-up), alternating with torch;
  * GB/s and the share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s), from the algorithmic bytes: forward
    N*K*s plus the labels and 8N (loss and lse); backward 2*N*K*s plus the labels, lse and dy; transposes 2 * bytes;
  * extra_MB (backward): peak memory allocated during the backward beyond what was allocated before it.
The first line names the device and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35


def device_label(torch):
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        out = ""
    return name, out or "unknown"


def window(torch, fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def compare(torch, fns, n, reps):
    """median ms of each fn over reps windows of n calls, the fns alternating window by window"""
    for fn in fns:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(reps):
        for t, fn in zip(times, fns):
            t.append(window(torch, fn, n))
    return [sorted(t)[reps // 2] for t in times]


def peak_extra_mb(torch, fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    extra = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    del out
    return round(extra, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F
    from blocksparse_b200 import transformer as tr
    from blocksparse_b200 import transpose_0213, transpose_2d

    if not torch.cuda.is_available():
        sys.exit("scripts/cross_entropy.py needs a CUDA device")
    torch.cuda.set_device(0)
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power})]
    print(lines[-1], flush=True)

    def emit(rec, nbytes, ms, torch_ms, extra=None):
        rec.update(ms=round(ms, 4), torch_ms=round(torch_ms, 4), speedup=round(torch_ms / ms, 2),
                   GBps=round(nbytes / (ms * 1e6), 1), hbm_share=round(nbytes / (ms * 1e-3) / (HBM_TBS * 1e12), 3))
        rec.update(extra or {})
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)

    gen = torch.Generator(device="cuda").manual_seed(0)
    N = 8192
    for K in (256, 32768, 50257, 65536, 131072):
        n = 200 if K == 256 else 20
        for dtype in (torch.float16, torch.bfloat16):
            x = (3 * torch.randn(N, K, device="cuda", generator=gen)).to(dtype)
            labels = torch.randint(0, K, (N,), device="cuda", generator=gen)
            dy = torch.rand(N, device="cuda", generator=gen) + 0.5
            s = x.element_size()
            loss, lse = tr._xent_fwd(x, labels)
            ref = F.cross_entropy(x, labels, reduction="none")
            # the two compute the same loss; a gross mismatch would make the timing meaningless
            assert (loss - ref.float()).abs().max().item() < 0.05 * max(1.0, ref.float().abs().max().item())
            rec = dict(op="softmax_cross_entropy", N=N, K=K, dtype=str(dtype)[6:])
            fwd_bytes = N * K * s + N * 8 + N * 8
            ms, tms = compare(torch, [lambda: tr._xent_fwd(x, labels),
                                      lambda: F.cross_entropy(x, labels, reduction="none")], n, args.reps)
            emit(dict(rec, part="forward"), fwd_bytes, ms, tms)

            xr = x.detach().requires_grad_()
            ref_out = F.cross_entropy(xr, labels, reduction="none")
            bwd_bytes = 2 * N * K * s + N * (8 + 4 + 4)

            def torch_bwd():
                return torch.autograd.grad(ref_out, xr, dy, retain_graph=True)[0]
            ms, tms = compare(torch, [lambda: tr._xent_bwd(x, labels, lse, dy), torch_bwd], n, args.reps)
            extra = dict(extra_MB=peak_extra_mb(torch, lambda: tr._xent_bwd(x, labels, lse, dy)),
                         torch_extra_MB=peak_extra_mb(torch, torch_bwd))
            emit(dict(rec, part="backward"), bwd_bytes, ms, tms, extra)

            xo = x.detach().requires_grad_()

            def ours_both():
                from blocksparse_b200 import softmax_cross_entropy
                softmax_cross_entropy(xo, labels).backward(dy)
                xo.grad = None

            def torch_both():
                F.cross_entropy(xo, labels, reduction="none").backward(dy)
                xo.grad = None
            ms, tms = compare(torch, [ours_both, torch_both], n, args.reps)
            emit(dict(rec, part="forward+backward"), fwd_bytes + bwd_bytes, ms, tms)
            del x, xr, xo, ref_out, loss, lse, ref
            torch.cuda.empty_cache()

    for shape, what in (((16, 1024, 16, 64), "transpose_0213"), ((16, 1024, 16, 4), "transpose_0213"),
                        ((8192, 8192), "transpose_2d")):
        x = torch.randn(shape, device="cuda", generator=gen).half()
        if what == "transpose_0213":
            ours, ref = (lambda: tr._transpose_0213(x, *x.shape)), (lambda: x.permute(0, 2, 1, 3).contiguous())
        else:
            ours, ref = (lambda: transpose_2d(x)), (lambda: x.t().contiguous())
        assert torch.equal((transpose_0213(x) if x.dim() == 4 else transpose_2d(x)).view(torch.int16), ref().view(torch.int16))
        dst = torch.empty_like(x)
        ms, tms, cms = compare(torch, [ours, ref, lambda: dst.copy_(x)], 50, args.reps)
        emit(dict(op=what, shape=list(shape), dtype="float16", copy_ms=round(cms, 4),
                  copy_share=round(cms / ms, 3)), 2 * x.numel() * 2, ms, tms)
        del x, dst
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
