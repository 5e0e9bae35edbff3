#!/usr/bin/env python
"""Time of one Adafactor step -- clip_by_global_norm + AdafactorOptimizer.step -- on GPT-2 small's parameter list (148
tensors, 124.4 M parameters), with fp32 and with fp16 grads, against two baselines on the same params and grads:
torch.optim.Adafactor(foreach=True) after torch.nn.utils.clip_grad_norm_(foreach=True) (a different update rule, so a
timing baseline only), and this project's clip_by_global_norm + AdamOptimizer. Needs a CUDA device.

  python scripts/adafactor_step.py [--reps R] [--calls N] [--out FILE] [--profile DIR]

Per grad dtype and implementation one JSON line with:
  * ms: median over R windows of N steps (CUDA events around each window, after warm-up; the implementations' windows
    alternate);
  * state_MB: optimizer state bytes; peak_extra_MB: the most device memory one step allocates beyond what existed
    before it (workspace, norm scratch, torch's temporaries);
  * GB/s and hbm_share of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s), from the algorithmic bytes of each rule:
    Adafactor reads the grad twice (norm and step), reads and writes the param, and reads and writes its moments once;
    Adam adds the two per-element moments read and written.
With --profile DIR, a separate run under torch.profiler writes each kernel's mean time for our Adafactor step to
DIR/adafactor_kernels.json. The first line names the device and its power limit.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from dense_softmax import HBM_TBS, device_label  # noqa: E402
from optimizer_step import gpt2_small_shapes  # noqa: E402


def window(torch, fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def peak_extra(torch, fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out")
    ap.add_argument("--profile")
    args = ap.parse_args()
    import torch
    from blocksparse_b200 import AdafactorOptimizer, AdamOptimizer, clip_by_global_norm
    if not torch.cuda.is_available():
        raise SystemExit("scripts/adafactor_step.py needs a CUDA device")
    name, power = device_label(torch)
    lines = [json.dumps({"device": name, "power_limit": power})]
    print(lines[0], flush=True)
    torch.manual_seed(0)
    shapes = gpt2_small_shapes()
    for gdtype in (torch.float32, torch.float16):
        ps = {k: [torch.randn(s, device="cuda") * 0.02 for s in shapes] for k in ("adafactor", "adam")}
        gs = [(torch.randn(s, device="cuda") * 1e-3).to(gdtype) for s in shapes]
        tps = [p.clone().requires_grad_() for p in ps["adafactor"]]
        for tp, g in zip(tps, gs):
            tp.grad = g.float()                          # torch's optimizers step fp32 params with fp32 grads
        ada = AdafactorOptimizer(ps["adafactor"], learning_rate=1e-4)
        adam = AdamOptimizer(ps["adam"], learning_rate=1e-4)
        theirs = torch.optim.Adafactor(tps, lr=1e-4, foreach=True)

        def ada_step():
            _, scale = clip_by_global_norm(gs, clip_norm=1.0)
            ada.step(grads=gs, norm_scale=scale)

        def adam_step():
            _, scale = clip_by_global_norm(gs, clip_norm=1.0)
            adam.step(grads=gs, norm_scale=scale)

        def torch_step():
            torch.nn.utils.clip_grad_norm_(tps, 1.0, foreach=True)
            theirs.step()

        fns = {"ours-adafactor": ada_step, "ours-adam": adam_step, "torch-adafactor": torch_step}
        for fn in fns.values():
            for _ in range(3):
                fn()
        peaks = {k: peak_extra(torch, fn) for k, fn in fns.items()}
        t = {k: [] for k in fns}
        for _ in range(args.reps):
            for k, fn in fns.items():
                t[k].append(window(torch, fn, args.calls))
        n = sum(p.numel() for p in tps)
        gb = 2 if gdtype == torch.float16 else 4
        factored = sum(s[0] + s[1] for s in shapes if len(s) == 2 and s[0] > 1)
        unfactored = sum(s[0] for s in shapes if len(s) == 1)
        state = {"ours-adafactor": 4 * (factored + unfactored), "ours-adam": 8 * n,
                 "torch-adafactor": sum(v.numel() * v.element_size() for st in theirs.state.values()
                                        for v in st.values() if torch.is_tensor(v))}
        ada_bytes = n * (2 * gb + 8) + 2 * state["ours-adafactor"]
        nbytes = {"ours-adafactor": ada_bytes, "torch-adafactor": n * (2 * 4 + 8) + 2 * state["torch-adafactor"],
                  "ours-adam": n * (2 * gb + 8 + 16)}
        for k in fns:
            ms = sorted(t[k])[args.reps // 2]
            gbs = nbytes[k] / (ms * 1e6)
            rec = {"op": "clip+step", "workload": "gpt2-small", "impl": k, "grad": str(gdtype)[6:],
                   "tensors": len(shapes), "params": n, "ms": round(ms, 4), "state_MB": round(state[k] / 2 ** 20, 2),
                   "peak_extra_MB": round(peaks[k] / 2 ** 20, 2), "GB/s": round(gbs),
                   "hbm_share": round(gbs / (HBM_TBS * 1e3), 3)}
            lines.append(json.dumps(rec))
            print(lines[-1], flush=True)
        if args.profile and gdtype == torch.float32:
            from torch.profiler import ProfilerActivity, profile
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.calls):
                    ada.step(grads=gs)
                torch.cuda.synchronize()
            per = {}
            for e in prof.key_averages():
                if e.device_type == torch.autograd.DeviceType.CUDA or "adafactor" in e.key:
                    per[e.key] = round(e.device_time_total / max(e.count, 1), 2)
            os.makedirs(args.profile, exist_ok=True)
            with open(os.path.join(args.profile, "adafactor_kernels.json"), "w") as f:
                json.dump({"device": name, "power_limit": power, "calls": args.calls, "mean_us": per}, f, indent=1)
        del ps, gs, tps, ada, adam, theirs
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
