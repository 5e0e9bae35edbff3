"""Shared helpers for the test-suite."""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def golden_files(prefix):
    return sorted(f for f in os.listdir(GOLDEN) if f.startswith(prefix) and f.endswith(".npz"))


def ref_errors(got, ref):
    """The reference's own two metrics (test/blocksparse_matmul_test.py:408-418)."""
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    d = np.abs(got - ref)
    denom = np.abs(ref).mean()
    max_err = d.max() / denom if denom > 0 else d.max()
    nrm = np.sqrt((ref * ref).sum())
    l2_err = np.sqrt((d * d).sum()) / nrm if nrm > 0 else np.sqrt((d * d).sum())
    return float(max_err), float(l2_err)


# ---- elementwise error bounds for the attention kernels ------------------------------------------------------------
def softmax_row_sums(a, orc):
    """Sum of a (batch, heads, blocks, bs, bs) over each softmax row -- every key of every block of one query row --
    broadcast back to a's shape. orc: the TransformerOracle of the layout."""
    out = np.zeros_like(a)
    for h in range(a.shape[1]):
        for row in orc.nn_list[orc._hl(h)]:
            if row:
                bids = [b for b, _ in row]
                out[:, h, bids] = a[:, h, bids].sum(axis=(1, 3), keepdims=True)
    return out



EPS32 = 2.0 ** -24                    # unit roundoff of fp32
# unit roundoff of one round-to-nearest conversion to a storage dtype, by name: "bfloat16", "float16", "float32"
U_OUT = {"bfloat16": 2.0 ** -8, "float16": 2.0 ** -11, "float32": EPS32}


def softmax_grad_bound(ref, dy, y, row_abs_dyy, out_dtype, scale, longest):
    """Largest |got - ref| a softmax-gradient kernel may show, elementwise (float64 arrays).

    dx = (dy - acc) * y * scale with acc = sum_row(dy * y) accumulated in fp32. Every thread sums at most 8 keys per
    block over `longest` blocks in order, then a shuffle tree of <= 5 levels: |d acc| <= (8 L + 5) eps32 sum|dy y|
    (16-bit products are exact in fp32, fp32 products add one rounding each). The subtraction and the two multiplies
    round once each, at most eps32 (|dy| + sum|dy y|) y |scale| apiece; +4 covers the fp32 products and second-order
    terms. The result is then rounded once to the output dtype (relative u_out), and fp16 subnormals (< 2^-14) round
    with an absolute error of at most 2^-25."""
    return (U_OUT[out_dtype] * np.abs(ref)
            + EPS32 * (8 * longest + 12) * (np.abs(dy) + row_abs_dyy) * y * abs(scale) + 2.0 ** -25)


def fma_gemm_bound(ref, ref_abs, out_dtype, k_terms):
    """Largest |got - ref| of a CUDA-core (fp32 FMA) block-sparse GEMM, elementwise. ref_abs = the same product of the
    operands' absolute values. Each of the k_terms fmaf steps rounds once (eps32 * the running sum of |a b|); the
    fp32 oracle accumulates with the same worst case, hence 2 eps32 = 2^-23 per term. Then one output rounding of the
    computed value (relative u_out, applied to ref plus that error) and 2^-25 for fp16 subnormals."""
    u = U_OUT[out_dtype]
    return u * np.abs(ref) + k_terms * 2.0 ** -23 * (1 + u) * ref_abs + 2.0 ** -25
