#!/usr/bin/env python
"""Kernel time and bandwidth of the elementwise ops against the torch expression a user would write and against the
reference's own kernels (oracle/_ref/libbsref.so, when it was built). Needs a CUDA device.

  python scripts/elementwise.py [--reps R] [--calls N] [--out FILE]

Cases, bf16 at (N, K) = (16384, 4096):
  * forward: add, subtract, multiply, divide, maximum, minimum (two operands), sigmoid, tanh, gelu (one), float_cast
    bf16 -> fp32 and fp32 -> bf16, add_n8 of 8 inputs, against torch.add / sub / mul / div / fmax / fmin, torch.sigmoid,
    torch.tanh, the tanh gelu expression, .to() and a chain of 7 torch.add;
  * backward of the bias-add and gain-mul broadcasts (fp32 vector of K): ours (dx = dz and the fixed-order db; dx = dz g
    and dg) against torch.autograd.grad of x + b and x * g.
Per case one JSON line with ms (the median over R windows of N calls, CUDA events around each window, after warm-up,
alternating with the other side), torch_ms, ref_ms (the reference's raw launcher, null without the library), and GB/s
and the share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s) from the algorithmic bytes: every operand read once
and every output written once (the vector and the db partials left out). The first line names the device and its power
limit.
"""
import argparse
import ctypes
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
    from blocksparse_b200 import elementwise as el
    from oracle import ref_elementwise as rew
    from oracle import ref_kernels as rk
    if not torch.cuda.is_available():
        raise SystemExit("scripts/elementwise.py needs a CUDA device")
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power, "reference": rew.missing() or "built"})]
    print(lines[0], flush=True)
    ref_lib = rk.load() if rew.available() else None

    def raw(fn_name, *a):
        """The reference entry called as it is, without the binding's checks and synchronisation."""
        fn = getattr(ref_lib, fn_name)
        fn.argtypes, fn.restype = rew.SIGNATURES[fn_name], ctypes.c_int
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        return lambda: fn(*a, s)

    def emit(rec, ours, tref, ref, nbytes):
        ms, tms = compare(torch, ours, tref, args.calls, args.reps)
        rms = compare(torch, ours, ref, args.calls, args.reps)[1] if ref is not None else None
        gbs = nbytes / (ms * 1e6)
        rec.update({"ms": round(ms, 4), "torch_ms": round(tms, 4), "ref_ms": None if rms is None else round(rms, 4),
                    "GB/s": round(gbs), "hbm_share": round(gbs / (HBM_TBS * 1e3), 3), "vs_torch": round(tms / ms, 2),
                    "vs_ref": None if rms is None else round(rms / ms, 2)})
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)

    dt, N, K = torch.bfloat16, 16384, 4096
    n = N * K
    x = torch.randn(N, K, device="cuda", dtype=dt)
    y = torch.randn(N, K, device="cuda", dtype=dt) + 3
    z = torch.empty_like(x)
    nb = n * x.element_size()
    binary = [("add", el.ADD_OP, torch.add), ("subtract", el.SUB_OP, torch.sub), ("multiply", el.MUL_OP, torch.mul),
              ("divide", el.DIV_OP, torch.div), ("maximum", el.MAXIMUM_OP, torch.fmax),
              ("minimum", el.MINIMUM_OP, torch.fmin)]
    for op, code, tfn in binary:
        ref = raw("bsref_ew_forward", 2, z.data_ptr(), x.data_ptr(), y.data_ptr(), None, 1.0, n, 0, code) \
            if ref_lib else None
        emit(dict(op=op, dir="forward", shape=[N, K], dtype="bfloat16"), lambda: el._fwd(x, code, y),
             lambda: tfn(x, y), ref, 3 * nb)
    c = 0.7978845608028654
    unary = [("sigmoid", el.SIG_OP, torch.sigmoid), ("tanh", el.TANH_OP, torch.tanh),
             ("gelu", el.GELU_OP, lambda v: 0.5 * v * (1 + torch.tanh(c * (v + 0.044715 * v ** 3))))]
    for op, code, tfn in unary:
        alpha = 0.044715 if op == "gelu" else 1.0
        ref = raw("bsref_ew_forward", 2, z.data_ptr(), x.data_ptr(), None, None, alpha, n, 0, code) if ref_lib else None
        emit(dict(op=op, dir="forward", shape=[N, K], dtype="bfloat16"), lambda: el._fwd(x, code, None, None, 0, alpha),
             lambda: tfn(x), ref, 2 * nb)
    xf = x.float()
    zf = torch.empty_like(xf)
    for src, dst, out in ((x, torch.float32, zf), (xf, torch.bfloat16, z)):
        ref = raw("bsref_float_cast", rk.DT[dst], rk.DT[src.dtype], out.data_ptr(), src.data_ptr(), n) \
            if ref_lib else None
        emit(dict(op="float_cast", dir="forward", src=str(src.dtype)[6:], dst=str(dst)[6:], shape=[N, K]),
             lambda: el._cast(src, dst), lambda: src.to(dst), ref, n * (src.element_size() + out.element_size()))
    del xf, zf
    xs = [torch.randn(N // 4, K, device="cuda", dtype=dt) for _ in range(8)]
    arr = (ctypes.c_void_p * 8)(*[t.data_ptr() for t in xs])
    z8 = torch.empty_like(xs[0])

    def torch_sum():
        s = xs[0] + xs[1]
        for t in xs[2:]:
            s = s + t
        return s
    ref = raw("bsref_add_n", 2, z8.data_ptr(), arr, 8, z8.numel()) if ref_lib else None
    emit(dict(op="add_n8", inputs=8, dir="forward", shape=[N // 4, K], dtype="bfloat16"), lambda: el._add_n(xs[0], xs),
         torch_sum, ref, 9 * z8.numel() * z8.element_size())
    del xs, z8
    g = torch.randn(K, device="cuda")
    dz = torch.randn_like(x)
    db = torch.empty(K, device="cuda")
    dx = torch.empty_like(x)
    xr, br = x.detach().clone().requires_grad_(), g.detach().clone().requires_grad_()
    yr = xr + br.to(dt)
    ref = raw("bsref_ew_backward", 2, None, None, db.data_ptr(), dz.data_ptr(), None, None, None, None, 1.0, K, N, 18) \
        if ref_lib else None
    emit(dict(op="bias_add", dir="backward", shape=[N, K], dtype="bfloat16"),
         lambda: el._br_bwd(dz, None, g, 1, N, K, el.ACT_NONE), lambda: torch.autograd.grad(yr, (xr, br), dz,
                                                                                           retain_graph=True),
         ref, nb)
    yr = xr * br.to(dt)
    ref = raw("bsref_ew_backward", 2, dx.data_ptr(), None, db.data_ptr(), dz.data_ptr(), x.data_ptr(), None, None,
              g.data_ptr(), 1.0, K, N, 19) if ref_lib else None
    emit(dict(op="gain_mul", dir="backward", shape=[N, K], dtype="bfloat16"),
         lambda: el._gain_mul_grad(dz, x, g, N, K), lambda: torch.autograd.grad(yr, (xr, br), dz, retain_graph=True),
         ref, 3 * nb)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
