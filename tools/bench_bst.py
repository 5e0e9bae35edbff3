"""BASELINE cfg 3: block-sparse attention ops, heads 16, ctx 4096, bs 64, local+strided causal layout, batch 4.

Prints one JSON line per op with CUDA-event time, algorithmic bytes/flops and the fraction of
the measured HBM / tensor peaks (MEASURED_PEAKS.json)."""
import json
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from blocksparse_b200 import BlocksparseTransformer, _lib
from bench import peaks
from tests.golden.make_golden import causal_callback

batch, heads, hs, bs, nb = 4, 16, 64, 64, 64
q, k = np.indices((nb, nb))
lay = ((k <= q) & ((q - k < 4) | (k % 8 == 7))).astype(np.int32)
bst = BlocksparseTransformer(lay, bs, heads=heads, mask_callback=causal_callback)
gen = torch.Generator(device="cuda").manual_seed(0)
Q, K, V, DY = ((torch.rand((batch, nb * bs, heads * hs), generator=gen, device="cuda") * 2 - 1).half() for _ in range(4))
scale = 1.0 / np.sqrt(hs)
pk = peaks()


def timeit(fn, reps=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


S = bst._nt(Q, K, torch.bfloat16)
P = bst._softmax(S, scale, True, None, torch.float16)
Y = bst._xn(P, V, False)
DP = bst._nt(DY, V, torch.float16)
blocks = bst.blocks
bh = batch * heads
gemm_flops = 2.0 * blocks * bs * bs * hs * bh
sparse_bytes = blocks * bs * bs * 2.0 * bh
dense_bytes = nb * bs * hs * 2.0 * bh
ops = [
    ("nt (q.k^T)", lambda: bst._nt(Q, K, torch.bfloat16), gemm_flops, 2 * dense_bytes + sparse_bytes),
    ("masked_softmax", lambda: bst._softmax(S, scale, True, None, torch.float16), 0.0, 2 * sparse_bytes),
    ("nn (p.v)", lambda: bst._xn(P, V, False), gemm_flops, sparse_bytes + 2 * dense_bytes),
    ("tn (p^T.dy)", lambda: bst._xn(P, DY, True), gemm_flops, sparse_bytes + 2 * dense_bytes),
    ("softmax_grad", lambda: bst._softmax_grad(DP, P, scale), 0.0, 3 * sparse_bytes),
]
for name, fn, fl, by in ops:
    ms = timeit(fn)
    kern = _lib.last_kernel()
    print(json.dumps({"op": name, "kernel": kern, "ms": ms, "tflops": fl / ms / 1e9, "gbs": by / ms / 1e6,
                      "frac_hbm_peak": by / ms / 1e6 / pk["hbm"], "frac_tensor_peak": fl / ms / 1e9 / pk["tf_burst"],
                      "algorithmic_bytes": by, "algorithmic_flops": fl,
                      "config": "batch 4 heads 16 head_state 64 ctx 4096 bs 64, 453 blocks, fp16 in / bf16 scores"}), flush=True)
assert _lib.device_error() == 0
