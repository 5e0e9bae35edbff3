#!/usr/bin/env python
"""Kernel time and bandwidth of ConvEdgeBias and cwise_linear, forward and backward, beside the reference's own kernels
(oracle/_ref/libbsref.so, when built) and the torch eager code a user would write for the same math. Needs a CUDA
device.

  python scripts/conv_bias.py [--reps R] [--calls N] [--out FILE]

Cases (activations bf16 unless named, gains and biases fp32):
  * edge bias, 3x3 SAME: N 32, K 256, 64x64 in NHWC and NCHW, bf16 and fp32; the reference test's 1 x 512 x 128x128
    in both formats; a 3x3x3 NDHWC conv at N 4, K 64, 32x32x32; a stride-2 3x3 deconv to N 32, K 128, 64x64;
    forward (training), inference in place, and backward (dx, dg, db);
  * cwise_linear: (32, 256, 64, 64) with gain + bias + relu and with a bias only, (8192, 1024) and
    (4, 64, 16, 64, 64) with gain + bias + relu; forward and backward (dx and the channel sums).
Per case and direction one JSON line: ms (median over R windows of N calls, CUDA events around each window, after
warm-up, the three implementations alternating, each call a replay of a CUDA graph holding one call), the spread
(max - min window) of each, GB/s and the share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s) from the op's algorithmic bytes: the forward reads x and writes y;
inference reads and writes the edge elements; the edge backward reads dy, writes dx and reads x at the edges; the
cwise backward reads dy, reads x (y) and writes dx where a gain or relu needs them. Tables, gains and biases are left
out. The reference's backward scales dy in place and its forward copies x first; its time is for the same op. The
first line names the device and its power limit.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from dense_softmax import HBM_TBS, device_label, window  # noqa: E402


def graphed(torch, fn):
    """fn captured once in a CUDA graph, so that the windows time the kernels rather than the Python that launches
    them; fn itself where capture fails (reported as graph: false)."""
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                fn()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        return g.replay, True
    except Exception:
        torch.cuda.synchronize()
        return fn, False


def timed(torch, fns, calls, reps):
    """Median and spread (ms per call) of each fn, windows alternating between them."""
    for fn in fns:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    t = [[] for _ in fns]
    for _ in range(reps):
        for i, fn in enumerate(fns):
            t[i].append(window(torch, fn, calls))
    return [(sorted(v)[reps // 2], max(v) - min(v)) for v in t]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--out")
    args = ap.parse_args()
    import numpy as np
    import torch
    from blocksparse_b200 import conv_bias as cb
    if not torch.cuda.is_available():
        raise SystemExit("scripts/conv_bias.py needs a CUDA device")
    ref = None
    try:
        from oracle import ref_conv_bias as ref
        if ref.missing():
            ref = None
    except ImportError:
        ref = None
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power, "reference_kernels": ref is not None})]
    print(lines[0], flush=True)

    def emit(rec, fns, nbytes):
        keys = ["ours", "ref", "torch"]
        fns = [(k, graphed(torch, f)) for k, f in zip(keys, fns) if f is not None]
        rec["graph"] = all(ok for _, (_, ok) in fns)
        res = timed(torch, [f for _, (f, _) in fns], args.calls, args.reps)
        for (k, _), (ms, spread) in zip(fns, res):
            rec[k + "_ms"] = round(ms, 4)
            rec[k + "_spread_ms"] = round(spread, 4)
        gbs = nbytes / (rec["ours_ms"] * 1e6)
        rec.update({"MB": round(nbytes / 1e6, 1), "GB/s": round(gbs), "hbm_share": round(gbs / (HBM_TBS * 1e3), 3)})
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)

    gen = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda shape, dt: (torch.rand(shape, device="cuda", generator=gen) * 2 - 1).to(dt)

    # ---- edge bias ----
    edge_cases = []
    for fmt in ("NHWC", "NCHW"):
        for dt in (torch.bfloat16, torch.float32):
            edge_cases.append(("3x3 N32 K256 64x64", fmt, dt, [32, 64, 64, 256], [32, 64, 64, 256], [3, 3, 256, 256],
                               None, False))
    for fmt in ("NHWC", "NCHW"):
        edge_cases.append(("3x3 N1 K512 128x128", fmt, torch.bfloat16, [1, 128, 128, 512], [1, 128, 128, 512],
                           [3, 3, 512, 512], None, False))
    edge_cases.append(("3x3x3 N4 K64 32^3", "NDHWC", torch.bfloat16, [4, 32, 32, 32, 64], [4, 32, 32, 32, 64],
                       [3, 3, 3, 64, 64], None, False))
    edge_cases.append(("deconv s2 3x3 N32 K128 64x64", "NHWC", torch.bfloat16, [32, 32, 32, 256], [32, 64, 64, 128],
                       [3, 3, 128, 256], [1, 2, 2, 1], True))
    for label, fmt, dt, ys, xs, ws, st, deconv in edge_cases:
        last = fmt[-1] == "C"
        perm = lambda s: s if last else [s[0], s[-1]] + s[1:-1]
        ys, xs = perm(ys), perm(xs)
        op = cb.ConvEdgeBias(ys, xs, ws, st, "SAME", fmt, deconv=deconv)      # deconv: ys small, xs the output
        io = xs if deconv else ys         # what the op runs on: the conv's (deconv's) output
        x, dy = rnd(io, dt), rnd(io, dt)
        g, b = rnd(op.shape, torch.float32), rnd(op.shape, torch.float32)
        es, n = x.element_size(), x.numel()
        N, K = io[0], op.K
        edge_elems = N * op.edgeEntries * K
        pe = torch.as_tensor(op._pos_edge).long().cuda()
        on = pe >= 0
        idx = pe.clamp(min=0)
        P = int(np.prod(op.MPQ))
        view = (lambda t: t.view(N, P, K)) if last else (lambda t: t.view(N, K, P))
        mask = on[:, None] if last else on[None, :]
        pos_on = pe[on]
        on_idx = torch.nonzero(on).squeeze(1)

        def torch_fwd():
            G, B = (g[idx], b[idx]) if last else (g[:, idx], b[:, idx])
            xv = view(x)
            return torch.where(mask, xv * G + B, xv)

        def torch_bwd():
            G = g[idx] if last else g[:, idx]
            d, xv = view(dy), view(x)
            dx = torch.where(mask, d * G, d)
            if last:
                de, xe = d.index_select(1, on_idx).float(), xv.index_select(1, on_idx).float()
                dg = torch.zeros(op.shape, device="cuda").index_add_(0, pos_on, (de * xe).sum(0))
                db = torch.zeros(op.shape, device="cuda").index_add_(0, pos_on, de.sum(0))
            else:
                de, xe = d.index_select(2, on_idx).float(), xv.index_select(2, on_idx).float()
                dg = torch.zeros(op.shape, device="cuda").index_add_(1, pos_on, (de * xe).sum(0))
                db = torch.zeros(op.shape, device="cuda").index_add_(1, pos_on, de.sum(0))
            return dx, dg, db

        y = torch.empty_like(x)
        xi = x.clone()
        ours_f = lambda: op._forward(x, g, b, y, False)
        ours_i = lambda: op._forward(xi, g, b, xi, True)
        ours_b = lambda: op._backward(dy, x, g)
        ref_f = ref_i = ref_b = None
        if ref is not None:
            lut = torch.as_tensor(op.edgeBiasLut).cuda()
            ry, rxi, rdy = torch.empty_like(x), x.clone(), dy.clone()
            rdg, rdb = torch.empty(op.shape, device="cuda"), torch.empty(op.shape, device="cuda")
            ref_f = ref.launcher("bsref_edge_bias", *ref.edge_bias_args(op, x, g, b, ry, lut))
            ref_i = ref.launcher("bsref_edge_bias", *ref.edge_bias_args(op, rxi, g, b, rxi, lut, True))
            ref_b = ref.launcher("bsref_edge_bias_grad", ref.rk._dt(x), rdy.data_ptr(), rdg.data_ptr(),
                                 rdb.data_ptr(), x.data_ptr(), g.data_ptr(), lut.data_ptr(), op.edgeBiasDim, P, K, N,
                                 op.layout)
        rec = lambda d: {"op": "edge_bias", "case": label, "format": fmt, "dtype": str(dt).split(".")[-1],
                         "edges": op.edgeBiasDim, "edge_entries": op.edgeEntries, "dir": d}
        emit(rec("fwd"), [ours_f, ref_f, torch_fwd], 2 * n * es)
        emit(rec("inference"), [ours_i, ref_i, None], 2 * edge_elems * es)
        emit(rec("bwd"), [ours_b, ref_b, torch_bwd], 2 * n * es + edge_elems * es)
        del x, dy, y, xi

    # ---- cwise_linear ----
    for shape, gain, bias, relu, dt in (((32, 256, 64, 64), True, True, True, torch.bfloat16),
                                        ((32, 256, 64, 64), False, True, False, torch.bfloat16),
                                        ((32, 256, 64, 64), True, True, True, torch.float32),
                                        ((8192, 1024), True, True, True, torch.bfloat16),
                                        ((4, 64, 16, 64, 64), True, True, True, torch.bfloat16)):
        C = shape[1]
        x, dy = rnd(shape, dt), rnd(shape, dt)
        a = rnd([C], torch.float32) if gain else None
        b = rnd([C], torch.float32) if bias else None
        bc = [1, C] + [1] * (len(shape) - 2)
        axes = [0] + list(range(2, len(shape)))
        es, n = x.element_size(), x.numel()
        y = cb.cwise_linear(x, a, b, relu=relu)
        xy = x if gain else (y if relu else None)         # what the op saves for its gradient
        ours_f = lambda: cb.cwise_linear(x, a, b, relu=relu)
        ours_b = lambda: cb._cwise_linear_grad(dy, xy, a, b, relu, False)

        def torch_fwd():
            z = x * a.view(bc) if gain else x
            z = z + b.view(bc) if bias else z
            return torch.relu(z) if relu else z

        def torch_bwd():
            d = dy * (y > 0) if relu else dy
            out = [d * a.view(bc) if gain else d]
            if gain:
                out.append((d.float() * x.float()).sum(axes))
            if bias:
                out.append(d.float().sum(axes))
            return out

        ref_f = ref_b = None
        if ref is not None:
            N, DHW = shape[0], int(np.prod(shape[2:])) if len(shape) > 2 else 1
            ry, rdx = torch.empty_like(x), torch.empty_like(x)
            rda, rdb = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
            p = lambda t: None if t is None else t.data_ptr()
            ref_f = ref.launcher("bsref_cwise_linear", ref.rk._dt(x), ry.data_ptr(), x.data_ptr(), p(a), p(b), N, C,
                                 DHW, int(relu), 0)
            rd = gain or relu
            ref_b = ref.launcher("bsref_cwise_linear_grad", ref.rk._dt(x), rdx.data_ptr() if rd else None,
                                 p(rda) if gain else None, p(rdb) if bias else None, dy.data_ptr(),
                                 x.data_ptr() if gain else y.data_ptr(), p(a), p(b), N, C, DHW, int(relu), 0)
        rec = lambda d: {"op": "cwise_linear", "shape": list(shape), "gain": gain, "bias": bias, "relu": relu,
                         "dtype": str(dt).split(".")[-1], "dir": d}
        emit(rec("fwd"), [ours_f, ref_f, torch_fwd], 2 * n * es)
        emit(rec("bwd"), [ours_b, ref_b, torch_bwd], (3 if (gain or relu) else 1) * n * es)
        del x, dy, y, xy

    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
