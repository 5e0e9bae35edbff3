"""Shared helpers for the test-suite."""
import json
import os

import numpy as np
import torch

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


def dtype_name(dtype):
    """"bfloat16" for torch.bfloat16: the keys of U_OUT."""
    return str(dtype).replace("torch.", "")


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


# Units of eps32 * |a b| that one product of a wgmma GEMM may lose in its fp32 accumulation. Products of 16-bit values
# are exact in fp32, but the tensor cores do not round each addition to nearest: published models of Hopper's MMA align
# a group of products to the largest exponent and truncate. 4 allows two fp32 units per term; it is an assumption, not
# a derivation, so the checks below can log the worst ratio they see (BSMM_BOUND_LOG) to keep it honest. Measured with
# the GPU suite on an H100 80GB HBM3 (700 W power limit), the worst ratios were 0.11 for the fp32-output updat, where
# the accumulation shows directly; 0.77 with its alpha / gate / beta roundings, which the unit leaves out; and <= 0.05
# for the 16-bit outputs (xprop, xprop2, pair tiles, updat), whose own rounding hides most of it. Per MMA width of the
# updat kernel (tests/test_updat_persistent_gpu.py, H100 80GB HBM3 at a 400 W power limit), the fp32 dW showed 0.052,
# 0.058, 0.075 and 0.064 at N = 64, 128, 192 and 256. The wgmma attention GEMMs (csrc/tc_bst.cuh;
# tests/test_tc_gpu.py::test_tc_bst_gemms_match_oracle, H100 80GB HBM3; the same at 400 W and 700 W) showed 0.099 for the
# fp32-output NT, where the accumulation shows directly; 0.0079 / 0.0059 for NT to fp16 / bf16, 0.0032 / 0.0008 for NN
# and 0.025 / 0.0011 for TN to fp16 / bf16; <= 0.007 for the ops of the attention chain in
# tests/test_bst_chain_elementwise_gpu.py.
MMA_C = 4


def mma_gemm_bound(ref, ref_abs, out_dtype, k_terms, extra=0):
    """Largest |got - ref| of a wgmma (tensor-core, fp32-accumulating) block-sparse GEMM, elementwise, built like
    fma_gemm_bound: one output rounding, MMA_C eps32 per accumulated term (k_terms per output element: bs x the LUT
    entries the kernel walks for its block, or the minibatch x pairs for updat), the fp16 subnormal floor. `extra`
    counts the fp32 roundings of the epilogue (alpha, gate, beta: one each), each at most eps32 * ref_abs. For an
    accumulating call, ref_abs includes |old value|."""
    u = U_OUT[out_dtype]
    return u * np.abs(ref) + (k_terms * MMA_C * EPS32 * (1 + u) + extra * EPS32) * ref_abs + 2.0 ** -25


# Largest absolute error of one round-to-nearest conversion in the subnormal range of a storage dtype: half its
# smallest subnormal. fp32 and bf16 share fp32's exponent range, so their floor lies far below any value checked here.
SUBNORMAL_FLOOR = {"float16": 2.0 ** -25, "bfloat16": 2.0 ** -134, "float32": 2.0 ** -150}


def chain_bound(ref, ref_abs, out_dtype, k_terms):
    """Largest |got - ref| of an fp32 CUDA-core computation that is rounded once to out_dtype, elementwise.

    k_terms counts the fp32 roundings on the path to the result, each worth at most eps32 * ref_abs: one per addition
    in the order the kernel sums (serial loop, then shuffle levels or partials), one per product that is not exact,
    2 ulp = 4 eps32 for rsqrtf (CUDA C Programming Guide, math appendix) and one for sqrtf and division, which are
    correctly rounded without --use_fast_math. A value that depends on a computed quantity q as q^p carries |p| times
    q's relative error. ref_abs is the same expression on absolute values, so that cancelling terms keep their
    rounding budget; callers that weigh parts of a result differently pass the weighted sum with k_terms = 1. The
    first-order sum undercounts by a factor below 1 + k eps32, which the 2^-10 margin covers for k < 2^14. Then one
    rounding to out_dtype (relative u_out) and the subnormal floor of out_dtype."""
    u = U_OUT[out_dtype]
    return u * np.abs(ref) + k_terms * EPS32 * (1 + u) * (1 + 2.0 ** -10) * ref_abs + SUBNORMAL_FLOOR[out_dtype]


def assert_within(got, ref, bound, what, ref_abs=None, k_terms=None, out_dtype=None, family=None):
    """Every element of got (tensor or array) lies within bound of the float64 ref.

    With family, ref_abs, k_terms and out_dtype given and BSMM_BOUND_LOG naming a file, one JSON line is appended with
    the worst accumulation error seen, in units of k_terms * eps32 * ref_abs: the part of |got - ref| that the output
    rounding cannot explain. That is the number MMA_C has to stay above."""
    if hasattr(got, "detach"):
        got = got.detach().double().cpu().numpy()
    g = np.asarray(got, dtype=np.float64).reshape(np.shape(ref))
    err = np.abs(g - ref)
    log = os.environ.get("BSMM_BOUND_LOG")
    if log and family and ref_abs is not None:
        excess = np.maximum(err - U_OUT[out_dtype] * np.abs(ref) - 2.0 ** -25, 0.0)
        unit = np.broadcast_to(k_terms * EPS32 * ref_abs, err.shape)
        ratio = float(np.max(np.where(unit > 0, excess / np.where(unit > 0, unit, 1.0), 0.0), initial=0.0))
        with open(log, "a") as f:
            f.write(json.dumps({"family": family, "what": what, "ratio": ratio}) + "\n")
    bad = ~(err <= bound)
    assert not bad.any(), "%s: %d of %d elements out of bound, worst excess %.3e (err %.3e)" % (
        what, int(bad.sum()), bad.size, float(np.nanmax(np.where(bad, err - bound, -np.inf))), float(np.nanmax(err)))


def oracle_dense(orc, op, a, b):
    """MatmulOracle.fprop_dense / bprop_dense / updat_dense in float64 ("fprop" / "bprop": a = activations, b = W;
    "updat": a = X, b = DY), the same dense restatement evaluated through BLAS instead of einsum loops."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if op == "updat":
        full = a.T @ b if orc.axis else a @ b.T
        bs = orc.bsize
        return full.reshape(orc.C // bs, bs, orc.K // bs, bs)[orc.updat_lut[:, 0], :, orc.updat_lut[:, 1], :]
    D = orc.dense_weight(b)
    if op == "fprop":
        return a @ D if orc.axis else D.T @ a
    return a @ D.T if orc.axis else D @ a


def _bst_entries(orc, op):
    """(out, blk, inp) index arrays of shape (heads, blocks) for a BST product: output block, sparse block and input
    block of every LUT entry, read from nt_list ("nt": out = blk) or the rows of nn_list / tn_list, per head (lut_heads 1
    broadcasts its layout to every head). Entries are grouped by output block, in row order."""
    out, blk, inp = [], [], []
    for h in range(orc.heads):
        hl = orc._hl(h)
        if op == "nt":
            pairs = np.array(orc.nt_list[hl], dtype=np.int64).reshape(-1, 2)
            out.append(pairs[:, 0]); blk.append(np.arange(len(pairs))); inp.append(pairs[:, 1])
            continue
        rows = orc.nn_list[hl] if op == "nn" else orc.tn_list[hl]
        e = [(o, b, i) for o, row in enumerate(rows) for b, i in row]
        out.append([o for o, _, _ in e]); blk.append([b for _, b, _ in e]); inp.append([i for _, _, i in e])
    return tuple(np.array(x, dtype=np.int64) for x in (out, blk, inp))


def bst_dense(orc, op, a, b, with_abs=False):
    """The BST products of TransformerOracle.nt / nn / tn in float64, through batched matmuls instead of per-block loops.

    "nt": a, b dense (batch, ctx, heads * head_state) -> (batch, heads, blocks, bs, bs), block (q, k) of nt_list.
    "nn": a sparse (batch, heads, blocks, bs, bs), b dense over the key blocks -> dense over the query blocks, each
          query block the sum over its nn_list row of a[block] . b[key block].
    "tn": the same with a[block]^T over the tn_list row of each key block, b dense over the query blocks.
    with_abs: also return the product of |a| and |b|, the ref_abs of the error bounds."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    res = _bst_dense(orc, op, a, b)
    return (res, _bst_dense(orc, op, np.abs(a), np.abs(b))) if with_abs else res


def _bst_dense(orc, op, a, b):
    bs, H = orc.blk_size, orc.heads
    out, blk, inp = _bst_entries(orc, op)
    hidx = np.arange(H)[:, None]

    def heads_view(x):                       # (batch, ctx, H * hs) -> (batch, H, ctx blocks, bs, hs)
        n, ctx, S = x.shape
        return x.reshape(n, ctx // bs, bs, H, S // H).transpose(0, 3, 1, 2, 4)
    if op == "nt":
        A, B = heads_view(a), heads_view(b)
        return np.matmul(A[:, hidx, out], B[:, hidx, inp].swapaxes(-1, -2))
    B = heads_view(b)
    sp = a[:, hidx, blk]                                           # (batch, H, blocks, bs, bs)
    prod = np.matmul(sp.swapaxes(-1, -2) if op == "tn" else sp, B[:, hidx, inp])
    n_out = orc.ctx_blks_q if op == "nn" else orc.ctx_blks_k
    n, S = b.shape[0], b.shape[2]
    C = np.zeros((n, H, n_out, bs, S // H))
    for h in range(H):                       # sum each output block's run of entries (entries are grouped by block)
        counts = np.bincount(out[h], minlength=n_out)
        live = np.nonzero(counts)[0]
        if len(live):
            C[:, h, live] = np.add.reduceat(prod[:, h], (np.cumsum(counts) - counts)[live], axis=1)
    return C.transpose(0, 2, 3, 1, 4).reshape(n, n_out * bs, S)


def bst_terms(orc, op, head_state):
    """k_terms of a BST product, broadcastable against its output: head_state for "nt"; for "nn" / "tn", bs x the
    length of each output block's nn_list / tn_list row in its head."""
    if op == "nt":
        return float(head_state)
    bs = orc.blk_size
    rows = orc.nn_list if op == "nn" else orc.tn_list
    k = np.array([[len(r) for r in rows[orc._hl(h)]] for h in range(orc.heads)], dtype=np.float64) * bs   # (H, n_out)
    k = np.repeat(np.repeat(k.T[:, None, :, None], bs, axis=1), head_state, axis=3)                      # (n_out, bs, H, hs)
    return k.reshape(1, -1, orc.heads * head_state)


def feature_terms(layout, bs, bprop, axis):
    """k_terms of a single-block-per-CTA xprop, broadcastable against its (n_out*bs, N) or (N, n_out*bs) output:
    bs x the LUT row length of every output block (column counts for fprop, row counts for bprop)."""
    lay = np.asarray(layout) != 0
    counts = lay.sum(axis=1 if bprop else 0)
    kf = np.repeat(counts * bs, bs).astype(np.float64)
    return kf[None, :] if axis else kf[:, None]


def out_block(y, blk, bs, axis):
    """Output feature block blk of a dense (features on `axis`) matmul result."""
    return y[:, blk * bs:(blk + 1) * bs] if axis else y[blk * bs:(blk + 1) * bs]


def assert_zero_filled(y, empty, bs, axis, what):
    """A kernel wrote every element of y (fresh from _on_poisoned_output: no NaN is left) and the output blocks whose
    LUT row is empty are exactly zero."""
    assert not bool(torch.isnan(y).any()), "%s: %d elements never written" % (what, int(torch.isnan(y).sum()))
    for blk in empty:
        v = out_block(y, int(blk), bs, axis)
        assert bool((v == 0).all()), "%s: output block %d is not zero-filled (max %s)" % (what, blk, v.float().abs().max().item())


def record_kernels(monkeypatch, obj, names, seen):
    """Wrap the methods `names` of obj so that every call appends (name, kernel it launched last) to seen. The library
    keeps the last kernel's name per thread, and autograd runs the backward on a thread of its own, so the name is read
    in the thread that made the call."""
    from blocksparse_b200 import _lib

    def wrap(name, fn):
        def run(*a, **kw):
            out = fn(*a, **kw)
            seen.append((name, _lib.last_kernel()))
            return out
        return run
    for name in names:
        monkeypatch.setattr(obj, name, wrap(name, getattr(obj, name)))


def _on_poisoned_output(fn):
    """Run fn() with every floating-point tensor it allocates through torch.empty / torch.empty_like (its output and
    any temporaries) filled with NaN first, so an element a kernel never writes shows up as NaN. The returned tensor,
    or every tensor of a returned tuple, must be one of those: an output allocated any other way would make the NaN
    checks vacuous, so it fails here."""
    empty, empty_like = torch.empty, torch.empty_like
    ptrs = set()

    def poisoned(t):
        if t.is_floating_point():
            t.fill_(float("nan"))
            ptrs.add(t.data_ptr())
        return t
    torch.empty = lambda *a, **kw: poisoned(empty(*a, **kw))
    torch.empty_like = lambda *a, **kw: poisoned(empty_like(*a, **kw))
    try:
        out = fn()
    finally:
        torch.empty, torch.empty_like = empty, empty_like
    for i, t in enumerate(out if isinstance(out, tuple) else (out,)):
        assert t.data_ptr() in ptrs, "output %d was not allocated through torch.empty / torch.empty_like: nothing poisoned it" % i
    return out
