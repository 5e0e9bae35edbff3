"""Every kernel family on tensors of more than 2^31 elements, where 32-bit and 64-bit index arithmetic part ways.

A signed 32-bit product wraps at element offset 2^31: the kernel then reads or writes the wrong rows, silently, or faults.
The rest of the suite runs on a few million elements, where `int` and `long long` agree. Here each operation runs once
on a tensor past 2^31 elements, with inputs drawn on the device from a seeded generator, and is checked two ways:
  * its output starts as NaN (_on_poisoned_output) and no NaN may be left anywhere in it: a kernel that wraps writes
    the low rows twice and leaves the high ones untouched;
  * sampled rows or blocks -- the first, the last, both sides of element offset 2^31, and seeded random ones -- are
    recomputed in float64 from the device inputs gathered for those rows only, under the bounds of the small tests.

The float64 references are the suite's full oracles run on a sub-problem: a query block's row (or a key block's column)
of the attention layout is a 1 x L (L x 1) layout of its own (sub_problem), a set of minibatch rows is a minibatch, a
set of logit rows is a batch. tests/test_large_offsets_reference.py runs them over every row of small problems and
requires the full oracles' results.

The attention chain is run op by op through the raw ops (_nt, _softmax, _xn, _softmax_grad) in the order autograd runs
them; tests/test_bst_chain_elementwise_gpu.py asserts that wiring. Each case states its peak device memory and skips,
with the numbers, when that much is not free.
"""
import gc

import numpy as np
import pytest
import torch

from tests._util import (U_OUT, _on_poisoned_output, assert_within, bst_dense, dtype_name, feature_terms, fma_gemm_bound,
                         mma_gemm_bound, softmax_grad_bound, softmax_row_sums)
from tests.test_bst_attention_bwd_gpu import grad_bound
from tests.test_bst_attention_gpu import attention_bound
from tests.test_bst_softmax_gpu import softmax_bound
from tests.test_optimizer_gpu import _check_codes, _check_update
from tests.test_xent_transpose_gpu import _check_forward, _check_grad, _int_view
from tests._attention_oracle import oracle_attention
from blocksparse_b200 import (AdamOptimizer, BlocksparseMatMul, BlocksparseTransformer, Ema, _lib, clip_by_global_norm,
                              transpose_0213, transpose_2d)
from blocksparse_b200 import transformer as tr
from blocksparse_b200.layouts import bernoulli_layout
from oracle import optimize_oracle as oo
from oracle.bsmm_oracle import MatmulOracle
from oracle.bst_oracle import TransformerOracle

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
TWO31 = 2 ** 31
GB = 2.0 ** 30


# ---- memory, sampling -------------------------------------------------------------------------------------------------
def _need(gb, what):
    """Skip unless gb GB of device memory are free: the device is shared."""
    gc.collect()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < gb * GB:
        pytest.skip("%s needs %.1f GB of free device memory, %.1f GB are free" % (what, gb, free / GB))


def _no_nan(t, what):
    """No element of t is NaN, looked at in slices of 2^28 so that the mask stays small."""
    flat = t.reshape(-1)
    for i in range(0, flat.numel(), 1 << 28):
        part = flat[i:i + (1 << 28)]
        assert not bool(torch.isnan(part).any()), "%s: %d elements from offset %d on were never written" % (
            what, int(torch.isnan(part).sum()), i)


def sample_ids(n, cross, rng, n_rand=24, edge=2):
    """Sorted indices in [0, n): the first and last `edge`, the two on either side of `cross` (the index whose element
    offset passes 2^31), and n_rand seeded random ones."""
    ids = set(range(min(edge, n))) | set(range(max(n - edge, 0), n))
    ids |= {c for c in (cross - 1, cross, cross + 1) if 0 <= c < n}
    ids |= set(int(i) for i in rng.integers(0, n, n_rand))
    return sorted(ids)


# ---- attention: one row or column of the layout as a problem of its own -----------------------------------------------
def causal(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    """tests/golden/make_golden.py's causal_callback without its Python loop over the block's elements."""
    m = np.ones(blk_shape, dtype=bool)
    return np.tril(m) if qry_idx == key_idx else m


def tril_layout(n):
    return np.tril(np.ones((n, n), np.int32))


def band_layout(n, width):
    """causal band: query block q holds key blocks q - width + 1 .. q"""
    return np.tril(np.ones((n, n), np.int32)) - np.tril(np.ones((n, n), np.int32), -width)


_SUBS = {}


def sub_problem(lists, cb, bs, h, idx, column=False):
    """Query block idx with its key blocks (column: key block idx with its query blocks) of head h of a shared layout,
    as a TransformerOracle of the 1 x L (L x 1) all-ones layout whose block e carries the mask of the row's e-th block.
    lists: anything with the nn_list / tn_list of the big layout. Returns (oracle, the row's block ids in the big
    sparse tensor, its key (query) blocks)."""
    key = (id(lists), cb, bs, h, idx, column)
    if key in _SUBS and _SUBS[key][0] is lists:
        return _SUBS[key][1]
    row = (lists.tn_list if column else lists.nn_list)[0][idx]
    bids, others = [b for b, _ in row], [o for _, o in row]

    def sub_cb(blk_shape, head, q, k, e):
        qq, kk = (others[e], idx) if column else (idx, others[e])
        return cb(blk_shape, h, qq, kk, bids[e])
    lay = np.ones((len(row), 1) if column else (1, len(row)), np.int32)
    if len(_SUBS) > 256:
        _SUBS.clear()
    res = TransformerOracle(lay, bs, heads=1, mask_callback=sub_cb if cb is not None else None), bids, others
    _SUBS[key] = (lists, res)             # every op of a chain asks for the same rows
    return res


def dense_blocks(x, b, h, blks, bs, hs):
    """Context blocks blks of head h of batch element b of a dense (batch, ctx, heads * hs) tensor, as float64
    (1, len(blks) * bs, hs)."""
    idx = torch.as_tensor(blks, device=x.device)
    v = x[b].reshape(-1, bs, x.shape[2])[idx][:, :, h * hs:(h + 1) * hs]
    return v.reshape(1, -1, hs).double().cpu().numpy()


def sparse_blocks(w, b, h, bids):
    """Blocks bids of (batch, heads, blocks, bs, bs) as float64 (1, 1, len(bids), bs, bs)."""
    return w[b, h, torch.as_tensor(bids, device=w.device)].double().cpu().numpy()[None, None]


def crossing(bst, bs):
    """(z, block) of the sparse block that holds element offset 2^31."""
    g = TWO31 // (bs * bs)
    return g // bst.blocks, g % bst.blocks


def sample_rows(bst, bs, Z, rng, column=False, n_rand=8):
    """(z, query block) pairs (column: key block): the first, the last -- which holds the last block of the sparse
    tensor --, the rows around the block at offset 2^31 and seeded random ones, half of those past the crossing."""
    n = bst.ctx_blks_k if column else bst.ctx_blks_q
    zc, blk = crossing(bst, bs)
    at = bst.nt_list[0][blk][1 if column else 0]
    rows = {(0, 0), (0, n - 1), (Z - 1, 0), (Z - 1, n - 1)}
    rows |= {(zc, r) for r in (at - 1, at, at + 1) if 0 <= r < n}
    rows |= {(int(z), int(r)) for z, r in zip(rng.integers(0, Z, n_rand), rng.integers(0, n, n_rand))}
    rows |= {(int(z), int(r)) for z, r in zip(rng.integers(zc, Z, n_rand), rng.integers(0, n, n_rand))}
    return sorted(rows)


def _gemm_bound(kernel):
    return fma_gemm_bound if kernel.startswith("fma_") else mma_gemm_bound


def check_nt(bst, cb, rows, heads, hs, a, b, got, kernel, what):
    """got = a . b^T on the blocks of the sampled query rows."""
    bs = bst.blk_size
    for z, q in rows:
        so, bids, kbs = sub_problem(bst, cb, bs, z % heads, q)
        A, B = dense_blocks(a, z // heads, z % heads, [q], bs, hs), dense_blocks(b, z // heads, z % heads, kbs, bs, hs)
        ref, ref_abs = bst_dense(so, "nt", A, B, with_abs=True)
        out = dtype_name(got.dtype)
        assert_within(sparse_blocks(got, z // heads, z % heads, bids), ref, _gemm_bound(kernel)(ref, ref_abs, out, float(hs)),
                      "%s z %d row %d (%s)" % (what, z, q, kernel))


def check_xn(bst, cb, rows, heads, hs, w, x, got, column, kernel, what):
    """got = w . x (column: w^T . x) on the sampled output blocks."""
    bs = bst.blk_size
    for z, r in rows:
        so, bids, others = sub_problem(bst, cb, bs, z % heads, r, column)
        W, X = sparse_blocks(w, z // heads, z % heads, bids), dense_blocks(x, z // heads, z % heads, others, bs, hs)
        ref, ref_abs = bst_dense(so, "tn" if column else "nn", W, X, with_abs=True)
        out = dtype_name(got.dtype)
        g = dense_blocks(got, z // heads, z % heads, [r], bs, hs)
        assert_within(g, ref, _gemm_bound(kernel)(ref, ref_abs, out, float(bs * len(bids))),
                      "%s z %d block %d (%s)" % (what, z, r, kernel))


def check_softmax(bst, cb, rows, heads, x, p, scale, amax, what):
    bs = bst.blk_size
    for z, q in rows:
        so, bids, _ = sub_problem(bst, cb, bs, z % heads, q)
        xs = sparse_blocks(x, z // heads, z % heads, bids)
        pr = so.masked_softmax(xs, scale=scale).astype(np.float64)
        assert_within(sparse_blocks(p, z // heads, z % heads, bids), pr, softmax_bound(pr, p.dtype, amax, bst.nn_max),
                      "%s z %d row %d" % (what, z, q))


def check_softmax_grad(bst, cb, rows, heads, dy, y, dx, scale, what):
    bs = bst.blk_size
    for z, q in rows:
        so, bids, _ = sub_problem(bst, cb, bs, z % heads, q)
        d, yv = sparse_blocks(dy, z // heads, z % heads, bids), sparse_blocks(y, z // heads, z % heads, bids)
        ref = so.masked_softmax_grad(d, yv, scale=scale)
        bound = softmax_grad_bound(ref, d, yv, softmax_row_sums(np.abs(d * yv), so), dtype_name(dx.dtype), scale, bst.nn_max)
        assert_within(sparse_blocks(dx, z // heads, z % heads, bids), ref, bound, "%s z %d row %d" % (what, z, q))


def _randn(shape, dtype, gen, scale=1.0):
    t = torch.randn(shape, device="cuda", dtype=dtype, generator=gen)
    return t.mul_(scale) if scale != 1.0 else t


def _abs_max(t):
    lo, hi = torch.aminmax(t)
    return max(abs(float(lo)), abs(float(hi)))


def _run(fn):
    """fn() on poisoned memory, with the kernel it launched last."""
    out = _on_poisoned_output(fn)
    return out, _lib.last_kernel()


def _chain(lay, bs, batch, heads, hs, dtype, flags, seed, want_softmax, forward_only=False):
    """The attention chain, forward and backward, on a sparse tensor past 2^31 elements."""
    bst = BlocksparseTransformer(lay, bs, heads=heads, mask_callback=causal)
    Z = batch * heads
    numel = Z * bst.blocks * bs * bs
    assert TWO31 < numel < 2 ** 32, numel
    gen = torch.Generator(device="cuda").manual_seed(seed)
    rng = np.random.default_rng(seed)
    S, scale = heads * hs, 1.0 / np.sqrt(hs)
    q, k, v, dy = (_randn((batch, bst.ctx_blks_q * bs, S), dtype, gen) for _ in range(4))
    rows, cols = sample_rows(bst, bs, Z, rng), sample_rows(bst, bs, Z, rng, column=True, n_rand=4)
    past = [(z * bst.blocks + bst.nn_list[0][r][0][0]) * bs * bs >= TWO31 for z, r in rows]
    assert any(past) and not all(past) and (Z - 1, bst.ctx_blks_q - 1) in rows      # rows that start on either side of 2^31
    tc = bs == 64 and hs in (64, 128) and not flags
    nt_k = "wgmma_bst_nt" if tc else "fma_dds_nt"
    name = "bs%d %s" % (bs, dtype_name(dtype))

    scores, kern = _run(lambda: bst._nt(q, k, BF16, flags))
    assert kern == nt_k, kern
    assert scores.numel() == numel > TWO31
    _no_nan(scores, name + " scores")
    check_nt(bst, causal, rows, heads, hs, q, k, scores, kern, name + " scores")

    p, kern = _run(lambda: bst._softmax(scores, scale, True, None, dtype))
    assert kern == want_softmax, kern
    _no_nan(p, name + " probabilities")
    check_softmax(bst, causal, rows, heads, scores, p, scale, _abs_max(scores) * scale, name + " probabilities")
    del scores

    y, kern = _run(lambda: bst._xn(p, v, False, flags))
    assert kern == ("wgmma_bst_nn" if tc else "fma_sdd_xn"), kern
    _no_nan(y, name + " y")
    check_xn(bst, causal, rows, heads, hs, p, v, y, False, kern, name + " y")
    if forward_only:
        return
    dv, kern = _run(lambda: bst._xn(p, dy, True, flags))
    assert kern == ("wgmma_bst_tn" if tc else "fma_sdd_xn"), kern
    _no_nan(dv, name + " dv")
    check_xn(bst, causal, cols, heads, hs, p, dy, dv, True, kern, name + " dv")
    del y, dv

    dP, kern = _run(lambda: bst._nt(dy, v, dtype, flags))
    assert kern == nt_k, kern
    _no_nan(dP, name + " dP")
    check_nt(bst, causal, rows, heads, hs, dy, v, dP, kern, name + " dP")

    dS, kern = _run(lambda: bst._softmax_grad(dP, p, scale))
    assert kern == want_softmax.replace("softmax", "softmax_grad"), kern
    _no_nan(dS, name + " dS")
    check_softmax_grad(bst, causal, rows, heads, dP, p, dS, scale, name + " dS")
    del dP, p
    dS = dS.to(BF16)                                   # what autograd hands to the NT backward: the scores' dtype

    tc_b = tc and dtype == BF16                        # bf16 dS with fp16 q / k: mixed dtypes run on the CUDA cores
    dk, kern = _run(lambda: bst._xn(dS, q, True, flags))
    assert kern == ("wgmma_bst_tn" if tc_b else "fma_sdd_xn"), kern
    _no_nan(dk, name + " dk")
    check_xn(bst, causal, cols, heads, hs, dS, q, dk, True, kern, name + " dk")
    dq, kern = _run(lambda: bst._xn(dS, k, False, flags))
    assert kern == ("wgmma_bst_nn" if tc_b else "fma_sdd_xn"), kern
    _no_nan(dq, name + " dq")
    check_xn(bst, causal, rows, heads, hs, dS, k, dq, False, kern, name + " dq")
    assert _lib.device_error() == 0, _lib.device_error_text()


@pytest.mark.parametrize("dtype", [BF16, F16], ids=dtype_name)
def test_chain_register_softmax(dtype):
    """Block 64, batch 2, heads 4, causal 362 x 362 blocks: 65703 blocks, 2.15e9 elements; rows of up to 362 blocks run
    the register softmax. Peak: three sparse tensors of 4.3 GB (p, dP, dS) and the slices of the NaN scan, 14 GB."""
    _need(22, "the causal chain")
    _chain(tril_layout(362), 64, 2, 4, 64, dtype, 0, 11, "bst_softmax")


@pytest.mark.parametrize("bs,ctx_blks", [(64, 520), (32, 2056)], ids=["bs64", "bs32"])
def test_chain_staged_softmax(bs, ctx_blks):
    """Batch 4, heads 16, a causal band of 16 blocks: 8200 blocks of 64 x 64 (32896 of 32 x 32), 2.15e9 elements; rows of
    at most 16 blocks run the TMA-staged softmax, in both of its instantiations. Peak 14 GB."""
    _need(22, "the banded chain")
    _chain(band_layout(ctx_blks, 16), bs, 4, 16, 64, BF16, 0, 12 + bs, "bst_softmax_staged")


def test_chain_cuda_core_gemms():
    """The causal layout of test_chain_register_softmax with the GEMMs forced onto the CUDA-core kernels. Peak 14 GB."""
    _need(22, "the causal chain on the CUDA cores")
    _chain(tril_layout(362), 64, 2, 4, 64, BF16, _lib.FLAG_FORCE_GENERIC, 13, "bst_softmax")


def test_cuda_core_gemms_fp32():
    """fp32 NT and NN on the same layout: 8.6 GB per sparse tensor, one held. Peak 9 GB."""
    _need(12, "the fp32 NT / NN")
    bs, batch, heads, hs = 64, 2, 4, 64
    bst = BlocksparseTransformer(tril_layout(362), bs, heads=heads, mask_callback=causal)
    gen = torch.Generator(device="cuda").manual_seed(14)
    rng = np.random.default_rng(14)
    q, k, v = (_randn((batch, 362 * bs, heads * hs), F32, gen) for _ in range(3))
    rows = sample_rows(bst, bs, batch * heads, rng)
    w, kern = _run(lambda: bst._nt(q, k, F32))
    assert kern == "fma_dds_nt" and w.numel() > TWO31
    _no_nan(w, "fp32 nt")
    check_nt(bst, causal, rows, heads, hs, q, k, w, kern, "fp32 nt")
    w.mul_(1.0 / 64)
    y, kern = _run(lambda: bst._xn(w, v, False))
    assert kern == "fma_sdd_xn"
    _no_nan(y, "fp32 nn")
    check_xn(bst, causal, rows, heads, hs, w, v, y, False, kern, "fp32 nn")
    assert _lib.device_error() == 0, _lib.device_error_text()


@pytest.mark.parametrize("lay,batch,heads", [(tril_layout(362), 2, 4), (band_layout(520, 16), 4, 16)], ids=["tril", "band"])
def test_fused_attention(lay, batch, heads):
    """The fused forward and the fused backward's dq on the layouts above. The sparse tensor they stand for has more
    than 2^31 elements but is never stored; the row statistics and the per-(batch, head) decompositions are. dk and dv
    are checked for unwritten elements. Peak under 2 GB."""
    _need(4, "fused attention")
    bs, hs, dtype = 64, 64, BF16
    bst = BlocksparseTransformer(lay, bs, heads=heads, mask_callback=causal)
    Z = batch * heads
    assert Z * bst.blocks * bs * bs > TWO31
    gen = torch.Generator(device="cuda").manual_seed(15)
    rng = np.random.default_rng(15)
    scale = 1.0 / np.sqrt(hs)
    q, k, v, dy = (_randn((batch, bst.ctx_blks_q * bs, heads * hs), dtype, gen) for _ in range(4))
    (o, m, l), kern = _run(lambda: bst._attention_train(q, k, v, scale, None))
    assert kern == "wgmma_bst_attention_train", kern
    (dq, dk, dv), kern = _run(lambda: bst._attention_grad(q, k, v, o, dy, m, l, scale, None))
    assert kern == "wgmma_bst_attention_bwd_dkdv", kern
    assert _lib.device_error() == 0, _lib.device_error_text()
    for t, what in ((o, "o"), (m, "row max"), (l, "row sum"), (dq, "dq"), (dk, "dk"), (dv, "dv")):
        _no_nan(t, "fused " + what)
    for z, r in sample_rows(bst, bs, Z, rng, n_rand=6):
        b, h = z // heads, z % heads
        so, _, kbs = sub_problem(bst, causal, bs, h, r)
        Q, dY = dense_blocks(q, b, h, [r], bs, hs), dense_blocks(dy, b, h, [r], bs, hs)
        K, V = dense_blocks(k, b, h, kbs, bs, hs), dense_blocks(v, b, h, kbs, bs, hs)
        ref = oracle_attention(so, Q, K, V, scale)
        bound, _ = attention_bound(so, ref, Q, K, V, scale, None, hs, dtype)
        assert_within(dense_blocks(o, b, h, [r], bs, hs), ref, bound, "fused o z %d row %d" % (z, r))
        (ref_dq, _, _), (bq, _, _) = grad_bound(so, Q, K, V, dY, scale, None, hs, dtype)
        assert_within(dense_blocks(dq, b, h, [r], bs, hs), ref_dq, bq, "fused dq z %d row %d" % (z, r))


# ---- block-sparse matmul ---------------------------------------------------------------------------------------------------
def minibatch_crossing(axis, feat, N):
    """The minibatch index at which a (N, feat) (axis 1) or (feat, N) (axis 0) activation tensor passes offset 2^31."""
    return TWO31 // feat if axis else TWO31 % N


def take(t, axis, idx):
    """Minibatch entries idx of an activation tensor, in the op's own layout, as float64."""
    i = torch.as_tensor(idx, device=t.device)
    return (t.index_select(0, i) if axis else t.index_select(1, i)).double().cpu().numpy()


def updat_dense64(X, E, axis, lut, bs, absolute=False, step=1 << 16):
    """dW of every block of the layout in float64: X^T . E (axis 1) or X . E^T (axis 0) accumulated over the minibatch
    in slices with torch's float64 matmul, on the tensors' own device, then the layout's blocks in updat_lut order."""
    N = X.shape[0] if axis else X.shape[1]
    C, K = (X.shape[1], E.shape[1]) if axis else (X.shape[0], E.shape[0])
    acc = torch.zeros((C, K), dtype=torch.float64, device=X.device)
    for i in range(0, N, step):
        xs, es = (X[i:i + step], E[i:i + step]) if axis else (X[:, i:i + step], E[:, i:i + step])
        xs, es = xs.double(), es.double()
        if absolute:
            xs, es = xs.abs(), es.abs()
        acc += xs.t() @ es if axis else xs @ es.t()
    lut = torch.as_tensor(np.asarray(lut), device=X.device).long()
    return acc.reshape(C // bs, bs, K // bs, bs)[lut[:, 0], :, lut[:, 1], :].cpu().numpy()


def _bsmm(feat, bs, axis, N, dtype, seed, prefix):
    """fprop, bprop and updat on activations past 2^31 elements. fprop / bprop: sampled minibatch entries, all features.
    updat: every dW element. Its float64 reference also runs on the GPU: it is torch's float64 GEMM, which shares
    nothing with this library, and a host matmul over 2^21 rows would take minutes. For updat all but about a thousand
    minibatch entries (the first and last 128, 256 around the crossing, 512 random ones) are zeroed first: products with
    an exact zero add no rounding error, so the bound counts the live entries only and stays far below the size of a dW
    element, while entries read from a wrapped offset would be zeros or miss the live rows past 2^31."""
    rng = np.random.default_rng(seed)
    lay = bernoulli_layout(rng, feat // bs, feat // bs, 0.25)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=axis)
    orc = MatmulOracle(lay, bs, axis)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    W = _randn(bsmm.w_shape, dtype, gen, 0.05)
    X, E = _randn(bsmm.i_shape(N), dtype, gen, 0.5), _randn(bsmm.o_shape(N), dtype, gen, 0.5)
    assert X.numel() > TWO31 and E.numel() > TWO31
    cross = minibatch_crossing(axis, feat, N)
    pick = sample_ids(N, cross, rng, n_rand=40, edge=4)
    assert pick[-1] == N - 1 and cross in pick
    name = dtype_name(dtype)
    W64 = W.double().cpu().numpy()
    for op, inp, fn in (("fprop", X, bsmm.fprop), ("bprop", E, bsmm.bprop)):
        out, kern = _run(lambda: fn(inp, W))
        assert kern.startswith(prefix[0]), (op, kern)
        assert out.numel() > TWO31
        _no_nan(out, "%s (%s)" % (op, kern))
        a = take(inp, axis, pick)
        ofn = orc.fprop if op == "fprop" else orc.bprop
        ref, ref_abs = ofn(a, W64), ofn(np.abs(a), np.abs(W64))
        kt = feature_terms(lay, bs, op == "bprop", axis)
        assert_within(take(out, axis, pick), ref, _gemm_bound(kern)(ref, ref_abs, name, kt), "%s bs %d axis %d (%s)" % (op, bs, axis, kern))
        del out
    live = sorted(set(sample_ids(N, cross, rng, n_rand=512, edge=128)) | set(range(max(cross - 128, 0), min(cross + 128, N))))
    keep = torch.zeros(N, dtype=dtype, device="cuda")
    keep[torch.as_tensor(live, device="cuda")] = 1
    for t in (X, E):
        t.mul_(keep[:, None] if axis else keep[None, :])
    dw, kern = _run(lambda: bsmm.updat([X], [E], dw_dtype=F32))
    assert kern.startswith(prefix[1]), kern
    assert _lib.device_error() == 0, _lib.device_error_text()
    ref = updat_dense64(X, E, axis, bsmm.updat_lut, bs)
    ref_abs = updat_dense64(X, E, axis, bsmm.updat_lut, bs, absolute=True)
    assert float(np.abs(ref).mean()) > 1.0                      # the bound below is a small fraction of an element
    assert_within(dw, ref, _gemm_bound(kern)(ref, ref_abs, "float32", float(len(live))), "updat bs %d axis %d (%s)" % (bs, axis, kern))


@pytest.mark.parametrize("bs,axis", [(32, 1), (32, 0), (64, 1)])        # the oracle's (block size, axis) pairs at 32 / 64
def test_bsmm_bf16(bs, axis):
    """1024 x 1024 features at 25 % density, N = 2^21 + 128 (a multiple of 8, as feature axis 0 needs): X, Y of 2.15e9
    elements each, on the wgmma kernels. Peak: X, E and one output of 4.3 GB, 13 GB."""
    _need(16, "bsmm bf16")
    _bsmm(1024, bs, axis, 2 ** 21 + 128, BF16, 20 + bs + axis, ("wgmma_xprop", "wgmma_updat"))


def test_bsmm_fp32_cuda_cores():
    """512 x 512 features, N = 2^22 + 128, fp32 on the CUDA-core kernels: 8.6 GB per activation tensor. Peak 26 GB."""
    _need(30, "bsmm fp32")
    _bsmm(512, 32, 1, 2 ** 22 + 128, F32, 29, ("fma_sdd_xn", "fma_dds_nt"))


# ---- cross entropy ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,K,dtype,ldtype", [(16400, 131072, F16, torch.int32), (42800, 50257, BF16, torch.int64)],
                         ids=["fp16-vector", "bf16-one-element"])
def test_softmax_cross_entropy(rows, K, dtype, ldtype):
    """Logits and their gradient of 2.15e9 elements on the CTA route: 16-byte loads (K a multiple of 8) and one element
    per load (K = 50257). Peak: logits and dx of 4.3 GB, 9 GB."""
    _need(12, "cross entropy")
    assert rows * K > TWO31
    gen = torch.Generator(device="cuda").manual_seed(K)
    rng = np.random.default_rng(K)
    x = _randn((rows, K), dtype, gen, 3.0)
    labels = torch.randint(0, K, (rows,), device="cuda", generator=gen).to(ldtype)
    vec = 8 if K % 8 == 0 else 1
    (loss, lse), kern = _run(lambda: tr._xent_fwd(x, labels))
    assert kern == "softmax_xent_cta", kern
    assert bool(torch.isfinite(loss).all()) and bool(torch.isfinite(lse).all())
    pick = torch.as_tensor(sample_ids(rows, TWO31 // K, rng), device="cuda")
    assert int(pick[-1]) == rows - 1
    what = "%d x %d %s" % (rows, K, dtype_name(dtype))
    ref_lse, b_lse = _check_forward(loss[pick], lse[pick], x[pick], labels[pick], vec, what)
    dy = torch.rand(rows, device="cuda", generator=gen) * 1.75 + 0.25
    dx, kern = _run(lambda: tr._xent_bwd(x, labels, lse, dy))
    assert kern == "softmax_xent_grad_cta", kern
    assert dx.numel() > TWO31
    _no_nan(dx, what + " dx")
    _check_grad(dx[pick], x[pick], labels[pick], dy[pick], ref_lse, b_lse, what)
    assert _lib.device_error() == 0, _lib.device_error_text()


# ---- transposes ----------------------------------------------------------------------------------------------------------------
def _equal_in_slices(y, ref_of, n, step, what):
    for i in range(0, n, step):
        j = min(i + step, n)
        assert torch.equal(_int_view(y[:, i:j]), _int_view(ref_of(i, j))), "%s: output cells %d..%d differ" % (what, i, j)


@pytest.mark.parametrize("shape,route", [((1, 46400, 46400, 1), "transpose_tile"), ((1, 20000, 17900, 6), "transpose_tile"),
                                         ((1, 4100, 4100, 128), "transpose_rows")], ids=["2d", "tile-d3-6", "rows"])
def test_transposes(shape, route):
    """More than 2^31 elements inside one leading index, bit for bit against permute().contiguous() over the whole output,
    in slices. The first shape runs through transpose_2d. Peak: input, output and a slice, 9 GB."""
    _need(12, "transpose")
    assert shape[1] * shape[2] * shape[3] > TWO31
    gen = torch.Generator(device="cuda").manual_seed(shape[1])
    x = _randn(shape, F16, gen)
    if shape[3] == 1:
        y, kern = _run(lambda: transpose_2d(x.view(shape[1], shape[2])))
        y = y.view(1, shape[2], shape[1], 1)
    else:
        y, kern = _run(lambda: transpose_0213(x))
    assert kern == route, kern
    assert y.shape == (1, shape[2], shape[1], shape[3])
    _equal_in_slices(y, lambda i, j: x[:, :, i:j].permute(0, 2, 1, 3).contiguous(), shape[2], 2048, "x".join(map(str, shape)))
    assert torch.equal(y[0, -1, -1], x[0, -1, -1])              # the last cell, beyond 2^31 on both sides


# ---- optimizer -----------------------------------------------------------------------------------------------------------------
def windows(n, width=4096):
    """Element windows at the start, on both sides of offset 2^31 and at the end of a tensor of n > 2^31 elements."""
    return [(0, width), (TWO31 - width, TWO31), (TWO31, min(TWO31 + width, n)), (n - min(width, n), n)]


def _count_changed(a, b):
    """Elements of a that differ from b (a tensor of a's shape, or a number), counted in slices."""
    total = 0
    for i in range(0, a.numel(), 1 << 28):
        total += int((a[i:i + (1 << 28)] != (b[i:i + (1 << 28)] if torch.is_tensor(b) else b)).sum())
    return total


ADAM = dict(lr=0.1, beta1=0.9, beta2=0.999, epsilon=1e-8)


def adam_window_check(p_new, p_old, g, m_old, v_old, m_new, v_new, what):
    """One coded Adam step on a window: float64 arrays of the old and new state (moments as uint16 codes)."""
    kw = {k: float(np.float32(v)) for k, v in ADAM.items()}
    pr, mr, vr = oo.adam(g, p_old, oo.mean_decode(m_old), oo.var_decode(v_old), **kw)
    _check_update(p_new, p_old, pr, what + " p")
    _check_codes(m_new, mr, oo.mean_encode, oo.mean_decode, 9, what + " mean")
    _check_codes(v_new, vr, oo.var_encode, oo.var_decode, 10, what + " var")


def ema_window_check(e_new, e_old, p, decay, what):
    ref = oo.ema(e_old, p, decay)
    assert_within(e_new, ref, U_OUT["float16"] * np.abs(ref) * (1 + 2.0 ** -10) + 2.0 ** -24 * (np.abs(e_old) + np.abs(p)) + 2.0 ** -25,
                  what)


def test_optimizer():
    """One parameter of 2^31 + 5 elements (the odd tail leaves the 16-byte path) with a bf16 gradient and 16-bit moments:
    the global norm over it and two small tensors, two Adam steps (the second from non-zero moments, checked), two Ema
    applications. Peak: param 8.6 GB, its copy 8.6, grad 4.3, moments 8.6, 30 GB and slices."""
    _need(36, "the optimizer")
    n = TWO31 + 5
    gen = torch.Generator(device="cuda").manual_seed(7)
    p = _randn((n,), F32, gen, 0.5)
    g = _randn((n,), BF16, gen, 0.1)
    small = [_randn((1000,), F32, gen), _randn((77,), F16, gen)]

    total = sum(float(s.double().pow(2).sum()) for s in small)
    for i in range(0, n, 1 << 28):                              # the norm's reference: float64 on the device, in slices
        total += float(g[i:i + (1 << 28)].double().pow(2).sum())
    norm, scale = clip_by_global_norm([small[0], g, small[1]], clip_norm=1.0)
    rn = np.sqrt(total)
    # 1e-5: the second pass adds one fp32 partial per chunk, tens of thousands of them here
    assert abs(norm.item() - rn) <= 1e-5 * rn, (norm.item(), rn)
    assert abs(scale.item() - 1.0 / rn) <= 1e-5 / rn, (scale.item(), 1.0 / rn)

    opt = AdamOptimizer([p], learning_rate=ADAM["lr"], beta1=ADAM["beta1"], beta2=ADAM["beta2"], epsilon=ADAM["epsilon"],
                        fp16=True, zero_init_variables=True)
    opt.step(grads=[g])
    m, v = opt.state[p]["mean"], opt.state[p]["var"]
    assert m.dtype == torch.int16 and m.numel() == n
    wins = windows(n)
    codes = lambda t, a, b: t[a:b].cpu().numpy().view(np.uint16)
    f64 = lambda t, a, b: t[a:b].double().cpu().numpy()
    old = [(f64(p, a, b), codes(m, a, b).copy(), codes(v, a, b).copy()) for a, b in wins]
    before = p.clone()
    opt.step(grads=[g])
    for (a, b), (p0, m0, v0) in zip(wins, old):
        adam_window_check(f64(p, a, b), p0, f64(g, a, b), m0, v0, codes(m, a, b), codes(v, a, b), "adam [%d, %d)" % (a, b))
    # the generator draws an exact 0 about once in 2^23 values; with the same zero gradient in both steps the moments stay 0
    # and so does the update. Every other element has to move.
    zeros = n - _count_changed(g, 0.0)
    assert zeros < 4096 and _count_changed(p, before) == n - zeros, (zeros, n)
    del before, opt, m, v

    ema = Ema(decay=0.5, fp16=True)
    ema.apply([p])
    avg = ema.average(p)
    assert avg.dtype == F16 and avg.numel() == n
    e_old = [f64(avg, a, b) for a, b in wins]
    before = avg.clone()
    p.add_(1.0)
    ema.apply([p])
    for (a, b), e0 in zip(wins, e_old):
        ema_window_check(f64(avg, a, b), e0, f64(p, a, b), 0.5, "ema [%d, %d)" % (a, b))
    assert _count_changed(avg, before) == n
    assert _lib.device_error() == 0, _lib.device_error_text()
