#!/usr/bin/env python
"""Kernel time of fused_lstm_gates (both forms, forward and backward) and sparse_relu against the eager torch composition
of the same math and, when oracle/_ref/libbsref.so is there, against the reference's own kernels; and of one
block-sparse LSTM timestep with our gates against the same step with the torch gates. Needs a CUDA device.

  python scripts/lstm_step.py [--reps R] [--calls N] [--out FILE]

Shapes: (N, K) = (128, 2048), an LSTM step, latency-bound, reported in us per call; and (8192, 4096), bandwidth-bound,
where GB/s counts the bytes the math needs: 7 N K elements forward (c and the four gates read, c_next and h_next
written), 12 N K backward (c, the gates, ec and eh read; dc and the four gate gradients written), 2 N K for sparse_relu.
Each is run in fp32 and bf16. Per case the implementations alternate window by window (CUDA events around N calls each,
after warm-up) and the median over R windows is reported. "us" is our C entry and "ref_us" the reference's launcher,
both called through ctypes on preallocated outputs, so both pay the same host cost; "op_us" is the Python op (output
allocation and argument checks included) and "torch_us" the torch composition. The first line names the device and its
power limit.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from dense_softmax import device_label, window  # noqa: E402


def timed(torch, fns, calls, reps):
    """Median ms per call of each fn, the fns alternating window by window."""
    for fn in fns:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(reps):
        for t, fn in zip(times, fns):
            t.append(window(torch, fn, calls))
    return [sorted(t)[reps // 2] for t in times]


def ref_entries(torch):
    """Raw callables of the reference's LSTM launchers, or None without the library."""
    from oracle import ref_kernels as rk
    from oracle import ref_lstm
    if not ref_lstm.available():
        return None
    lib = rk.load()
    fns = {}
    for name, args in ref_lstm.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, ctypes.c_int
        fns[name] = fn
    return fns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    from blocksparse_b200 import BlocksparseMatMul, _lib, layer_norm, lstm
    if not torch.cuda.is_available():
        raise SystemExit("scripts/lstm_step.py needs a CUDA device")
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power})]
    print(lines[0], flush=True)
    ref = ref_entries(torch)
    L = _lib.load()
    DT = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}

    def stream():
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def emit(rec, fns, elems, esize):
        """fns: ours (raw entry), torch, the Python op, the reference (or None)."""
        ms = timed(torch, [f for f in fns if f is not None], args.calls, args.reps)
        ours, tms = ms[0], ms[1]
        rec.update({"us": round(ours * 1e3, 2), "op_us": round(ms[2] * 1e3, 2), "torch_us": round(tms * 1e3, 2),
                    "ref_us": round(ms[3] * 1e3, 2) if len(ms) > 3 else None,
                    "GB/s": round(elems * esize / (ours * 1e6)), "torch_GB/s": round(elems * esize / (tms * 1e6)),
                    "vs_torch": round(tms / ours, 2), "vs_ref": round(ms[3] / ours, 2) if len(ms) > 3 else None})
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)

    sig, tanh = torch.sigmoid, torch.tanh
    for N, K in ((128, 2048), (8192, 4096)):
        for dt in (torch.float32, torch.bfloat16):
            es = torch.empty((), dtype=dt).element_size()
            g = torch.Generator(device="cuda").manual_seed(0)
            r = lambda *s: torch.randn(*s, device="cuda", generator=g).to(dt)       # noqa: E731
            c, h, ec, eh = r(N, K), r(N, 4 * K), r(N, K), r(N, K)
            gates = [t.contiguous() for t in h.split(K, -1)]
            base = {"N": N, "K": K, "dtype": str(dt)[6:]}
            outs = [torch.empty_like(c) for _ in range(2)]
            douts = [torch.empty_like(c), torch.empty_like(h)] + [torch.empty_like(c) for _ in range(5)]
            dc_ = _lib.dtype_code(dt)
            hp = [h.data_ptr() + j * K * es for j in range(4)]
            dhp = [douts[1].data_ptr() + j * K * es for j in range(4)]
            gp = [t.data_ptr() for t in gates]
            d4p = [t.data_ptr() for t in douts[2:6]]

            def torch_fwd(c, i, u, f, o):
                cn = sig(f + 1.0) * c + sig(i) * tanh(u)
                return cn, sig(o) * tanh(cn)

            # forward, fused form
            ref_fn = None
            if ref:
                ref_fn = lambda: ref["bsref_lstm_gates"](DT[dt], outs[0].data_ptr(), outs[1].data_ptr(), c.data_ptr(),  # noqa: E731
                                                         h.data_ptr(), None, 1.0, N, 4 * K, stream())
            emit(dict(base, case="gates_fused_fwd"),
                 [lambda: L.bsmm_lstm_gates(dc_, 0, c.data_ptr(), *hp, 4 * K, None, outs[0].data_ptr(),
                                            outs[1].data_ptr(), N, K, 1.0, _lib.stream_ptr()),
                  lambda: torch_fwd(c, *h.split(K, -1)), lambda: lstm._gates_fwd(c, [h], None, N, K, 1.0), ref_fn],
                 7 * N * K, es)
            # backward, fused form
            cl, hl = c.clone().requires_grad_(), h.clone().requires_grad_()
            tout = torch_fwd(cl, *hl.split(K, -1))
            if ref:
                ref_fn = lambda: ref["bsref_lstm_gates_grad"](DT[dt], douts[0].data_ptr(), douts[1].data_ptr(),  # noqa: E731
                                                              ec.data_ptr(), eh.data_ptr(), c.data_ptr(), h.data_ptr(),
                                                              None, 1.0, N, 4 * K, stream())
            emit(dict(base, case="gates_fused_bwd"),
                 [lambda: L.bsmm_lstm_gates_grad(dc_, 0, c.data_ptr(), *hp, 4 * K, None, ec.data_ptr(), eh.data_ptr(),
                                                 douts[0].data_ptr(), *dhp, N, K, 1.0, _lib.stream_ptr()),
                  lambda: torch.autograd.grad(tout, (cl, hl), (ec, eh), retain_graph=True),
                  lambda: lstm._gates_bwd(c, [h], None, ec, eh, N, K, 1.0), ref_fn], 12 * N * K, es)
            # four-tensor form
            if ref:
                ref_fn = lambda: ref["bsref_lstm_gates4"](DT[dt], outs[0].data_ptr(), outs[1].data_ptr(), c.data_ptr(),  # noqa: E731
                                                          *[t.data_ptr() for t in gates], 1.0, N, K, stream())
            emit(dict(base, case="gates_four_fwd"),
                 [lambda: L.bsmm_lstm_gates(dc_, 0, c.data_ptr(), *gp, K, None, outs[0].data_ptr(),
                                            outs[1].data_ptr(), N, K, 1.0, _lib.stream_ptr()),
                  lambda: torch_fwd(c, *gates), lambda: lstm._gates_fwd(c, gates, None, N, K, 1.0), ref_fn],
                 7 * N * K, es)
            gl = [t.clone().requires_grad_() for t in gates]
            tout4 = torch_fwd(cl, *gl)
            if ref:
                ref_fn = lambda: ref["bsref_lstm_gates4_grad"](DT[dt], douts[0].data_ptr(),  # noqa: E731
                                                               *[t.data_ptr() for t in douts[2:6]], ec.data_ptr(),
                                                               eh.data_ptr(), c.data_ptr(),
                                                               *[t.data_ptr() for t in gates], 1.0, N, K, stream())
            emit(dict(base, case="gates_four_bwd"),
                 [lambda: L.bsmm_lstm_gates_grad(dc_, 0, c.data_ptr(), *gp, K, None, ec.data_ptr(), eh.data_ptr(),
                                                 douts[0].data_ptr(), *d4p, N, K, 1.0, _lib.stream_ptr()),
                  lambda: torch.autograd.grad(tout4, [cl] + gl, (ec, eh), retain_graph=True),
                  lambda: lstm._gates_bwd(c, gates, None, ec, eh, N, K, 1.0), ref_fn], 12 * N * K, es)
            # sparse_relu
            x = r(N, K)
            if ref:
                ref_fn = lambda: ref["bsref_sparse_relu"](DT[dt], outs[0].data_ptr(), x.data_ptr(), 1.0, K, N,  # noqa: E731
                                                          stream())

            def torch_srelu():
                xf = x.float()
                cut = xf.mean(-1, keepdim=True) + xf.std(-1, unbiased=False, keepdim=True)
                return (xf - cut).clamp_min_(0).to(x.dtype)
            emit(dict(base, case="sparse_relu"),
                 [lambda: L.bsmm_sparse_relu(dc_, x.data_ptr(), outs[0].data_ptr(), N, K, 1.0, _lib.stream_ptr()),
                  torch_srelu, lambda: lstm._srelu_fwd(x, N, K, 1.0), ref_fn], 2 * N * K, es)

    # one block-sparse LSTM timestep, features last, bf16: BlocksparseMatMul (K -> 4K), layer_norm(segments=4), gates
    N, K, bs = 128, 2048, 32
    dt = torch.bfloat16
    gen = torch.Generator().manual_seed(0)
    lay = (torch.rand(K // bs, 4 * K // bs, generator=gen) < 0.25).int().numpy()
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=1)
    w = (torch.randn(bsmm.w_shape, generator=gen) * 0.05).to(dt).cuda().requires_grad_()
    lg = torch.ones(4 * K, device="cuda", requires_grad=True)
    lb = torch.zeros(4 * K, device="cuda", requires_grad=True)
    x = torch.randn(N, 4 * K, device="cuda").to(dt)
    c0 = torch.randn(N, K, device="cuda").to(dt).requires_grad_()
    h0 = torch.randn(N, K, device="cuda").to(dt).requires_grad_()
    e = torch.randn(N, K, device="cuda").to(dt)

    def step(gates_fn):
        def run():
            z = layer_norm(bsmm(h0, w) + x, lg, lb, axis=1, segments=4)
            cn, hn = gates_fn(c0, z)
            return torch.autograd.grad((cn, hn), (w, lg, lb, c0, h0), (e, e))
        return run

    def torch_gates(c, z):
        i, u, f, o = z.split(K, -1)
        cn = sig(f + 1.0) * c + sig(i) * tanh(u)
        return cn, sig(o) * tanh(cn)
    ours, tms = timed(torch, [step(lambda c, z: lstm.fused_lstm_gates(c, z)), step(torch_gates)], args.calls,
                      args.reps)
    lines.append(json.dumps({"case": "bsmm_lstm_step_fwd_bwd", "N": N, "K": K, "dtype": "bfloat16", "density": 0.25,
                             "op_us": round(ours * 1e3, 2), "torch_gates_us": round(tms * 1e3, 2),
                             "vs_torch": round(tms / ours, 2)}))
    print(lines[-1], flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
