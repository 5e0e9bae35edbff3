"""BASELINE cfg 4: block-size sweep {8,16,32,64} at 4096x4096, density 20 %, N=2048, bf16 -- which kernel family runs
each (axis, block size) and how fast (CUDA-core FMA vs wgmma crossover)."""
import json
import sys

import torch

sys.path.insert(0, ".")
from blocksparse_b200 import BlocksparseMatMul, _lib
from bench import make_layout, peaks

N = 2048
pk = peaks()
X = [(torch.randn((N, 4096), device="cuda") * 0.1).bfloat16() for _ in range(3)]
E = [(torch.randn((N, 4096), device="cuda") * 0.1).bfloat16() for _ in range(3)]


def timeit(fn, reps=10):
    for i in range(2):
        fn(i)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(reps):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


for bs, axis in [(8, 0), (16, 0), (32, 0), (32, 1), (64, 1), (8, 1), (16, 1), (64, 0)]:
    nb = 4096 // bs
    bsmm = BlocksparseMatMul(make_layout(0.20, nb, nb, seed=1238), block_size=bs, feature_axis=axis)
    W = (torch.randn(bsmm.w_shape, device="cuda") * 0.01).bfloat16()
    xs = [x.t().contiguous() for x in X] if axis == 0 else X
    es = [e.t().contiguous() for e in E] if axis == 0 else E
    fl = 2.0 * bsmm.blocks * bs * bs * N
    rec = {"block_size": bs, "feature_axis": axis, "nnz_blocks": bsmm.blocks, "in_reference_pairs": (axis, bs) in [(0, 8), (0, 16), (0, 32), (1, 32), (1, 64)]}
    for name, fn in [("fprop", lambda i: bsmm.fprop(xs[i % 3], W)), ("bprop", lambda i: bsmm.bprop(es[i % 3], W)),
                     ("updat", lambda i: bsmm.updat([xs[i % 3]], [es[i % 3]]))]:
        ms = timeit(fn)
        rec[name] = {"ms": round(ms, 4), "tflops": round(fl / ms / 1e9, 1), "frac_tensor_peak": round(fl / ms / 1e9 / pk["tf_burst"], 4),
                     "kernel": _lib.last_kernel()}
    print(json.dumps(rec), flush=True)
assert _lib.device_error() == 0
