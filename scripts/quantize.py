#!/usr/bin/env python
"""Kernel time and bandwidth of quantize against the reference's own Quantize / QuantizationStats kernels
(oracle/_ref/libbsref.so, when it was built), and the cost of the optimizer qspecs on a GPT-2 small Adam step. Needs a
CUDA device.

  python scripts/quantize.py [--reps R] [--calls N] [--out FILE]

Cases:
  * quantize at (16384, 4096) and at 64 M elements, fp32 and bf16, stochastic 0 and 2, without and with a statistics
    call before it (frequency 1: statistics, the exponent update on the device, then the rounding). The reference's
    side is its raw launcher: Quantize (stochastic 2 with its Tausworthe buffer), and with statistics QuantizationStats
    first, which copies its five values to the host and so synchronises on every call.
  * one AdamOptimizer step over GPT-2 small's 148 fp32 tensors (124 M parameters, fp32 grads): no qspecs, and
    param_qspec / mean_qspec / var_qspec all set (frequency 1024, so statistics run on the scheduled steps only).
Per case one JSON line with ms (the median over R windows of N calls, CUDA events around each window, after warm-up,
alternating with the reference), ref_ms (null without the library), and GB/s and the share of the H100 SXM data-sheet
HBM bandwidth (3.35 TB/s) from the algorithmic bytes: x read and y written once, x read once more for the statistics.
The first line names the device and its power limit.
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from dense_softmax import HBM_TBS, compare, device_label, window  # noqa: E402

GPT2_SMALL = ([(50257, 768), (1024, 768)] + [s for _ in range(12) for s in (
    (768,), (768,), (768, 2304), (2304,), (768, 768), (768,), (768,), (768,), (768, 3072), (3072,), (3072, 768),
    (768,))] + [(768,), (768,)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    import numpy as np
    import torch
    from blocksparse_b200 import AdamOptimizer, set_entropy
    from blocksparse_b200.quantize import QuantizeSpec, new_schedule, quantize_tensors
    from oracle import quantize_oracle as qo
    from oracle import ref_kernels as rk
    from oracle import ref_quantize as rq
    if not torch.cuda.is_available():
        raise SystemExit("scripts/quantize.py needs a CUDA device")
    torch.cuda.set_device(0)
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power, "reference": rq.missing() or "built"})]
    print(lines[0], flush=True)
    ref_lib = rk.load() if rq.available() else None
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    set_entropy(1)

    def raw(fn_name, *a):
        fn = getattr(ref_lib, fn_name)
        fn.argtypes, fn.restype = rq.SIGNATURES[fn_name], ctypes.c_int
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        return lambda: fn(*a, s)

    def emit(rec, ours, ref, nbytes):
        if ref is None:
            ours()
            torch.cuda.synchronize()
            ts = sorted(window(torch, ours, args.calls) for _ in range(args.reps))
            ms, rms = ts[args.reps // 2], None
        else:
            ms, rms = compare(torch, ours, ref, args.calls, args.reps)
        gbs = nbytes / (ms * 1e6)
        rec.update({"ms": round(ms, 4), "ref_ms": None if rms is None else round(rms, 4), "GB/s": round(gbs, 1),
                    "hbm_share": round(gbs / (HBM_TBS * 1e3), 3),
                    "vs_ref": None if rms is None else round(rms / ms, 3)})
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)

    e = 4
    for shape in ((16384, 4096), (64 << 20,)):
        n = int(np.prod(shape))
        for dtype, fbits in ((torch.float32, 7), (torch.bfloat16, 3)):
            x = (torch.randn(shape, device="cuda") * 8).to(dtype)
            y = torch.empty_like(x)
            exp = torch.full((), e, dtype=torch.int64, device="cuda")
            es = x.element_size()
            f = qo.fmt(e, 5, fbits, True)
            fl = lambda b: float(np.array([b], np.uint32).view(np.float32)[0])  # noqa: E731
            for stoch in (0, 2):
                for stats in (False, True):
                    spec = QuantizeSpec(ebits=5, fbits=fbits, stochastic=stoch, frequency=1 if stats else 0)
                    sched = new_schedule()
                    ours = lambda: quantize_tensors([x], [y], [exp], [sched], spec, ["bench"])  # noqa: E731
                    ref = None
                    if ref_lib is not None:
                        ent = None
                        if stoch:
                            ent = torch.randint(0, 2 ** 31, (3 * sms * 8 * 128,), dtype=torch.int32, device="cuda")
                        scale = fl((127 - fbits - 1 - (31 if stoch else 0)) << 23)
                        q = raw("bsref_quantize", rk.DT[dtype], y.data_ptr(), x.data_ptr(),
                                None if ent is None else ent.data_ptr(), scale, f["mask"], fl(f["max_float"]),
                                fl(f["min_float"]), f["exp_norm"], n, stoch)
                        if stats:
                            out = (ctypes.c_float * 5)()
                            scratch = torch.zeros(8, device="cuda")
                            st = raw("bsref_quantization_stats", rk.DT[dtype], out, scratch.data_ptr(), x.data_ptr(),
                                     fl(f["max_float"]), fl(f["ftz_float"]), n)
                            ref = (lambda q, st: lambda: (st(), q()))(q, st)
                        else:
                            ref = q
                    emit({"case": "quantize", "shape": list(shape), "dtype": str(dtype).replace("torch.", ""),
                          "stochastic": stoch, "stats": stats}, ours, ref, (3 if stats else 2) * n * es)
            del x, y
            torch.cuda.empty_cache()

    # GPT-2 small Adam step, with and without the three qspecs
    params = [torch.randn(s, device="cuda") * 0.02 for s in GPT2_SMALL]
    grads = [torch.randn(s, device="cuda") * 1e-3 for s in GPT2_SMALL]
    nparam = sum(p.numel() for p in params)
    plain = AdamOptimizer([p.clone() for p in params], learning_rate=1e-4)
    spec = QuantizeSpec(ebits=5, fbits=10, frequency=1024)
    quant = AdamOptimizer([p.clone() for p in params], learning_rate=1e-4, param_qspec=spec, mean_qspec=spec,
                          var_qspec=QuantizeSpec(ebits=6, fbits=9, frequency=1024))
    ms, qms = compare(torch, lambda: plain.step(grads=grads), lambda: quant.step(grads=grads), args.calls, args.reps)
    rec = {"case": "adam_gpt2_small", "tensors": len(params), "params": nparam, "ms": round(ms, 4),
           "ms_qspecs": round(qms, 4), "qspec_overhead_ms": round(qms - ms, 4),
           "qspec_GB/s": round(3 * 2 * nparam * 4 / ((qms - ms) * 1e6), 1) if qms > ms else None}
    lines.append(json.dumps(rec))
    print(lines[-1], flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
