#!/usr/bin/env python
"""Time of grouped_lstm, forward and forward + backward, against the hand-rolled loop of existing ops it replaces, and of
its fused layer-norm / gates step against the two-kernel composition. Needs a CUDA device.

  python scripts/lstm_layer.py [--n N] [--t T] [--width W] [--reps R] [--calls C] [--out FILE]

Default sizes: N = 128, T = 64, in = width = 1024, in bf16 and fp16, with and without layernorm. Three things are
compared, each alternating window by window (CUDA events around C calls, after warm-up; the median over R windows):
  * layer: grouped_lstm (ms per call);
  * loop: per step torch.cat([x_t, h]) through a dense-layout BlocksparseMatMul (its per-step dW from autograd, which
    accumulates the T products), then layer_norm(segments=4) + fused_lstm_gates, or fused_lstm_gates with the bias;
  * step: one bsmm_lstm_ln_gates (forward) and bsmm_lstm_ln_gates_grad + _grad_reduce (backward) against
    bsmm_layer_norm + bsmm_lstm_gates and bsmm_lstm_gates_grad + bsmm_layer_norm_grad at (N, 4 width), in us per call:
    the raw C entries through ctypes on preallocated buffers, 200 calls per window, so both pay the same host cost.
The first line names the device and its power limit; every record repeats them.
"""
import argparse
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
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(reps):
        for t, fn in zip(times, fns):
            t.append(window(torch, fn, calls))
    return [sorted(t)[reps // 2] for t in times]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=128)
    ap.add_argument("--t", type=int, default=64)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import numpy as np
    import torch
    from blocksparse_b200 import BlocksparseMatMul, _lib, fused_lstm_gates, grouped_lstm, layer_norm
    from blocksparse_b200.lstm_layer import _StepProduct
    if not torch.cuda.is_available():
        raise SystemExit("scripts/lstm_layer.py needs a CUDA device")
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power})]
    print(lines[0], flush=True)
    N, T, W = args.n, args.t, args.width
    In = W
    g = torch.Generator(device="cuda").manual_seed(0)

    def emit(rec):
        rec.update(device=name, power_limit=power)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)

    for dtype in (torch.bfloat16, torch.float16):
        x = torch.randn(N, T, In, device="cuda", generator=g).to(dtype).requires_grad_()
        c0 = torch.randn(N, W, device="cuda", generator=g).to(dtype).requires_grad_()
        h0 = torch.randn(N, W, device="cuda", generator=g).to(dtype).requires_grad_()
        kernel = (torch.randn(In + W, 4 * W, device="cuda", generator=g) / (In + W) ** 0.5).requires_grad_()
        bias = torch.zeros(4 * W, device="cuda").requires_grad_()
        gain = torch.ones(4 * W, device="cuda").requires_grad_()
        d_out = torch.randn(N, T, W, device="cuda", generator=g).to(dtype)
        prod = _StepProduct.get(In + W, 4 * W)
        bsmm = BlocksparseMatMul(np.ones((prod.Cp // 32, prod.Kp // 32), np.int32), block_size=32, feature_axis=1)
        wb = prod.weights(kernel, dtype).detach().requires_grad_()
        for ln in (True, False):
            def layer_fwd():
                with torch.no_grad():
                    grouped_lstm(x, W, T, [c0, h0], kernel, bias, gain if ln else None, layernorm=ln)

            def layer_step():
                out, _ = grouped_lstm(x, W, T, [c0, h0], kernel, bias, gain if ln else None, layernorm=ln)
                out.backward(d_out)

            def loop(backward):
                c, h, outs = c0, h0, []
                with torch.set_grad_enabled(backward):
                    for t in range(T):
                        z = bsmm(torch.cat([x[:, t], h], 1), wb)
                        if ln:
                            c, h = fused_lstm_gates(c, layer_norm(z, gain, bias, axis=1, segments=4), forget_bias=1.0)
                        else:
                            c, h = fused_lstm_gates(c, z, bias=bias, forget_bias=1.0)
                        outs.append(h)
                    out = torch.stack(outs, 1)
                if backward:
                    out.backward(d_out)

            ms = timed(torch, [layer_fwd, lambda: loop(False), layer_step, lambda: loop(True)], args.calls, args.reps)
            emit({"what": "layer", "dtype": str(dtype)[6:], "layernorm": ln, "N": N, "T": T, "in": In, "width": W,
                  "fwd_ms": round(ms[0], 3), "loop_fwd_ms": round(ms[1], 3), "fwd_bwd_ms": round(ms[2], 3),
                  "loop_fwd_bwd_ms": round(ms[3], 3)})
        # the fused step alone against its two-kernel composition: the raw C entries on preallocated buffers
        K, K4 = W, 4 * W
        L, st = _lib.load(), _lib.stream_ptr
        dt, F32 = _lib.dtype_code(dtype), _lib.F32
        z = torch.randn(N, K4, device="cuda", generator=g).to(dtype)
        c, e = (torch.randn(N, K, device="cuda", generator=g).to(dtype) for _ in range(2))
        gn, bs = torch.ones(K4, device="cuda"), torch.zeros(K4, device="cuda")
        y, dy, dz = torch.empty_like(z), torch.empty_like(z), torch.empty_like(z)
        cn, hn, dc = torch.empty_like(c), torch.empty_like(c), torch.empty_like(c)
        mean, rstd = torch.empty(N, 4, device="cuda"), torch.empty(N, 4, device="cuda")
        dg, db = torch.empty_like(gn), torch.empty_like(bs)
        ws_ln = torch.empty(L.bsmm_layer_norm_workspace_bytes(1, N, K4, 4) // 4, device="cuda")
        ws_f = torch.empty(L.bsmm_lstm_ln_gates_workspace_bytes(N, K) // 4, device="cuda")
        gates = lambda t: [t.data_ptr() + j * K * t.element_size() for j in range(4)]
        P = lambda t: t.data_ptr()

        def fused_fwd():
            L.bsmm_lstm_ln_gates(dt, F32, P(c), P(z), K4, P(gn), P(bs), P(cn), P(hn), P(mean), P(rstd), N, K, 1e-6,
                                 1.0, st())

        def comp_fwd():
            L.bsmm_layer_norm(dt, F32, 1, P(z), P(gn), P(bs), P(y), P(mean), P(rstd), None, N, K4, 4, 1e-6, 0, st())
            L.bsmm_lstm_gates(dt, F32, P(c), *gates(y), K4, None, P(cn), P(hn), N, K, 1.0, st())

        def fused_bwd():
            L.bsmm_lstm_ln_gates_grad(dt, F32, P(c), P(z), K4, P(gn), P(bs), P(mean), P(rstd), P(e), P(e), P(dc),
                                      P(dz), P(ws_f), 0, N, K, 1.0, st())
            L.bsmm_lstm_ln_gates_grad_reduce(F32, P(ws_f), N, K, P(dg), P(db), st())

        def comp_bwd():
            L.bsmm_lstm_gates_grad(dt, F32, P(c), *gates(y), K4, None, P(e), P(e), P(dc), *gates(dy), N, K, 1.0, st())
            L.bsmm_layer_norm_grad(dt, F32, 1, P(dy), P(z), P(gn), P(bs), P(mean), P(rstd), P(dz), P(dg), P(db),
                                   P(ws_ln), N, K4, 4, 1e-6, 0, st())

        comp_fwd()
        ms = timed(torch, [fused_fwd, comp_fwd, fused_bwd, comp_bwd], 200, args.reps)
        emit({"what": "step", "dtype": str(dtype)[6:], "N": N, "K": K, "fused_fwd_us": round(ms[0] * 1e3, 1),
              "composed_fwd_us": round(ms[1] * 1e3, 1), "fused_bwd_us": round(ms[2] * 1e3, 1),
              "composed_bwd_us": round(ms[3] * 1e3, 1)})
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
