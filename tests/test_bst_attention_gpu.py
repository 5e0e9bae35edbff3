"""BlocksparseTransformer.attention: the fused wgmma kernel (csrc/tc_bst_attn.cuh) elementwise against the float64
oracle, its determinism, its recompute backward (bit-identical to the three-op chain's gradients), what autograd keeps
alive, and the fallback to the chain where no fused kernel exists."""
import collections

import numpy as np
import pytest
import torch

from tests._util import EPS32, MMA_C, SUBNORMAL_FLOOR, U_OUT, _on_poisoned_output, assert_within
from tests.golden.make_golden import causal_callback
from blocksparse_b200 import BlocksparseTransformer, _lib
from blocksparse_b200.layouts import local_strided_layout
from oracle.bst_oracle import TransformerOracle
from tests._attention_oracle import oracle_attention

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
_NAME = {BF16: "bfloat16", F16: "float16", F32: "float32"}
BS = 64


# ---- layouts and masks ---------------------------------------------------------------------------------------------
def _tril(n):
    """query block q holds q + 1 key blocks: rows of every length 1..n"""
    return np.tril(np.ones((n, n), np.int32))


def _hole(lay, q):
    """query block q holds no key block"""
    lay = lay.copy()
    lay[..., q, :] = 0
    return lay


def _per_head(lay, heads):
    """one layout per head, query rows rotated by the head index: equal block counts, different row lengths"""
    return np.stack([np.roll(lay, h, axis=0) for h in range(heads)])


def _future_first(n):
    """tril, except that query block 0 holds only key block 1: with autoregress_at_key 0 each of its rows is hidden"""
    lay = _tril(n)
    lay[0, 0], lay[0, 1] = 0, 1
    return lay


def _rect():
    """6 query blocks x 9 key blocks, rows of 2..9 blocks"""
    lay = np.zeros((6, 9), np.int32)
    for q in range(6):
        lay[q, q % 3::1 + q % 2] = 1
        lay[q, 8] = 1
    return lay


def _ones_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    return np.ones(blk_shape, dtype=bool)


def _hide_row_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    """causal inside diagonal blocks, and row 3 of query block 1 sees no key at all (uniform weights)"""
    m = causal_callback(blk_shape, head_idx, qry_idx, key_idx, blk_idx)
    if qry_idx == 1:
        m[3, :] = False
    return m


def _per_head_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    """a different pattern in every head; in head 1, row 5 of query block 0 sees no key at all"""
    q, k = np.indices(blk_shape)
    m = ((q + 2 * k + head_idx) % 3) != 0
    if head_idx == 1 and qry_idx == 0:
        m[5, :] = False
    return m


Case = collections.namedtuple("Case", "name lay cb ak hs scale")
CASES = [
    Case("tril20-causal", _tril(20), causal_callback, None, 64, 0.125),           # rows of 1..20 blocks
    Case("tril20-nomask", _tril(20), None, None, 128, 0.125),
    Case("cfg3-causal", local_strided_layout(16), causal_callback, None, 64, 0.125),
    Case("cfg3-causal-ak", local_strided_layout(16), causal_callback, 300, 128, 0.125),
    Case("perhead-mask", _per_head(_tril(6), 3), _per_head_cb, None, 64, 0.25),
    Case("perhead-ak", _per_head(_tril(7), 3), _per_head_cb, 130, 128, -0.125),
    Case("hole-hiderow", _hole(_tril(6), 2), _hide_row_cb, None, 128, 0.125),
    Case("hole-nomask", _hole(_tril(5), 0), None, None, 64, 0.125),
    Case("rect-nomask", _rect(), None, None, 64, 0.125),
    Case("rect-ak", _rect(), _ones_cb, 100, 128, 0.125),
    Case("future-ak0", _future_first(5), _ones_cb, 0, 64, 0.125),
]
HEADS, BATCH = 3, 2


def _inputs(lay, hs, dtype, seed, heads=HEADS, batch=BATCH):
    lay3 = lay if lay.ndim == 3 else lay[None]
    cq, ck = lay3.shape[1:]
    rng = np.random.default_rng(seed)
    q = rng.normal(0, 1, (batch, cq * BS, heads * hs))
    k, v = (rng.normal(0, 1, (batch, ck * BS, heads * hs)) for _ in range(2))
    return [torch.as_tensor(a.astype(np.float32)).to(dtype) for a in (q, k, v)]


def attention_bound(orc, ref, Q, K, V, scale, ak, hs, dtype):
    """Largest |got - ref| of the fused kernel, elementwise (float64 arrays of shape (batch, ctx_q, heads*hs)).

    ref = P V with P the float64 softmax of the oracle; A = P |V| (the oracle on |V|) weighs every error that is
    relative to the probabilities. With L the key blocks of the element's query row:
      * one rounding of the output: U_OUT[dtype] |ref|;
      * the unnormalised probabilities (<= 1) enter P V rounded to the input dtype: u_in A, and below fp16's normal
        range an absolute 2^-25 per key, at most SUBNORMAL_FLOOR[in] 64 L max|V| (the row sum l is >= 1);
      * S = Q K^T accumulates hs products per score: MMA_C eps32 hs (|Q| |K|^T) <= MMA_C eps32 hs qk, qk the largest
        entry of |Q| |K|^T; scaled, that is an absolute error in the exponent, which changes every probability
        relatively by at most that much and O by twice it (P and its normalisation): 2 MMA_C eps32 hs |scale| qk A;
      * the exponent arithmetic (scale, subtraction of the running max, log2 e): 4 fp32 roundings of values up to
        amax = |scale| qk, the online rescales telescope to as much again: 2 * 8 eps32 amax A;
      * P V accumulates 64 L products: MMA_C eps32 64 L A; the rescales of O and l (one per block), the sums of l
        (16 per block and thread, 2 shuffle levels), exp2f (2 ulp), the reciprocal and the multiply: eps32 (16 L + 64) A;
      * the subnormal floor of the output."""
    u_in = U_OUT[_NAME[dtype]]
    B, ctxq, S = Q.shape
    heads = S // hs
    A = oracle_attention(orc, Q, K, np.abs(V), scale, autoregress_at_key=ak)
    Qh = np.abs(Q.reshape(B, ctxq, heads, hs)).transpose(0, 2, 1, 3).astype(np.float64)
    Kh = np.abs(K.reshape(B, -1, heads, hs)).transpose(0, 2, 1, 3).astype(np.float64)
    qk = float((Qh @ Kh.transpose(0, 1, 3, 2)).max())
    amax = abs(scale) * qk
    L = np.array([[len(orc.nn_list[orc._hl(h)][r // BS]) for h in range(heads)] for r in range(ctxq)], np.float64)
    L = np.broadcast_to(L[None, :, :, None], (B, ctxq, heads, hs)).reshape(B, ctxq, S)
    rel = u_in + EPS32 * (2 * MMA_C * hs * abs(scale) * qk + 16 * amax + MMA_C * 64 * L + 16 * L + 64)
    return (u_in * np.abs(ref) + rel * A + SUBNORMAL_FLOOR[_NAME[dtype]] * 64 * L * float(np.abs(V).max())
            + SUBNORMAL_FLOOR[_NAME[dtype]]), L


def _case_id(c):
    return c.name + "-hs%d" % c.hs


@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("idx", range(len(CASES)), ids=[_case_id(c) for c in CASES])
def test_attention_matches_oracle(idx, dtype):
    case = CASES[idx]
    bst = BlocksparseTransformer(case.lay, BS, heads=HEADS, mask_callback=case.cb)
    orc = TransformerOracle(case.lay, BS, heads=HEADS, mask_callback=case.cb)
    q, k, v = _inputs(case.lay, case.hs, dtype, 100 + idx)
    qc, kc, vc = q.cuda(), k.cuda(), v.cuda()
    out = _on_poisoned_output(lambda: bst.attention(qc, kc, vc, scale=case.scale, autoregress_at_key=case.ak))
    assert _lib.last_kernel() == "wgmma_bst_attention"
    assert _lib.device_error() == 0, _lib.device_error_text()
    assert out.dtype == dtype and tuple(out.shape) == tuple(q.shape)
    got = out.cpu()
    assert not bool(torch.isnan(got).any()), "%d elements never written" % int(torch.isnan(got).sum())
    Q, K, V = (t.double().numpy() for t in (q, k, v))
    ref = oracle_attention(orc, Q, K, V, case.scale, autoregress_at_key=case.ak)
    bound, L = attention_bound(orc, ref, Q, K, V, case.scale, case.ak, case.hs, dtype)
    empty = L == 0
    assert bool((got.double().numpy()[empty] == 0).all()), "empty query blocks are not zero"
    assert_within(got, ref, bound, "attention " + _case_id(case))
    # determinism: a second call gives the same bits
    again = bst.attention(qc, kc, vc, scale=case.scale, autoregress_at_key=case.ak)
    assert torch.equal(again, out)


def test_cases_cover_the_envelope():
    """The covering set reaches what the kernel has to handle (pure Python; guards later edits)."""
    assert {c.hs for c in CASES} == {64, 128}
    assert any(c.lay.shape[-1] == 20 for c in CASES)                                    # past the ring and 16 blocks
    assert any(c.lay.ndim == 3 for c in CASES) and any(c.lay.shape[-2] != c.lay.shape[-1] for c in CASES)
    assert any((c.lay.sum(axis=-1) == 0).any() for c in CASES)                          # an empty query block
    assert {None, causal_callback, _per_head_cb, _hide_row_cb} <= {c.cb for c in CASES}
    assert any(c.ak is not None for c in CASES) and any(c.scale < 0 for c in CASES)


# ---- backward ------------------------------------------------------------------------------------------------------
def _chain(bst, q, k, v, scale, ak):
    return bst.weight_value_op(bst.masked_softmax(bst.query_key_op(q, k), scale, ak), v)


@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("lay,cb,ak,hs", [(_tril(6), None, None, 64), (_tril(6), causal_callback, None, 64),
                                          (_per_head(_tril(7), 3), _per_head_cb, 130, 128)],
                         ids=["nomask", "causal", "perhead-ak-hs128"])
def test_backward_is_bit_identical_to_the_chain(lay, cb, ak, hs, dtype):
    bst = BlocksparseTransformer(lay, BS, heads=HEADS, mask_callback=cb)
    q, k, v = (t.cuda() for t in _inputs(lay, hs, dtype, 7))
    dy = torch.randn(q.shape, generator=torch.Generator().manual_seed(3)).to(dtype).cuda()
    grads = []
    for fused in (True, False):
        qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
        y = bst.attention(qq, kk, vv, scale=0.125, autoregress_at_key=ak) if fused else _chain(bst, qq, kk, vv, 0.125, ak)
        if fused:
            assert _lib.last_kernel() == "wgmma_bst_attention"
        y.backward(dy)
        grads.append((qq.grad, kk.grad, vv.grad))
    assert _lib.device_error() == 0, _lib.device_error_text()
    for name, a, b in zip("qkv", *grads):
        assert a.dtype == b.dtype and torch.equal(a, b), "d%s differs from the chain's" % name
    # only some inputs need a gradient
    vv = v.clone().requires_grad_()
    bst.attention(q, k, vv, scale=0.125, autoregress_at_key=ak).backward(dy)
    assert torch.equal(vv.grad, grads[1][2])


def test_attention_saves_no_sparse_tensor():
    lay = local_strided_layout(16)
    bst = BlocksparseTransformer(lay, BS, heads=HEADS, mask_callback=causal_callback)
    q, k, v = (t.cuda().requires_grad_() for t in _inputs(lay, 64, F16, 11))
    sparse = (BATCH, HEADS, bst.blocks, BS, BS)

    def saved_shapes(fn):
        shapes = []
        with torch.autograd.graph.saved_tensors_hooks(lambda t: shapes.append(tuple(t.shape)) or t, lambda t: t):
            fn()
        return shapes
    fused = saved_shapes(lambda: bst.attention(q, k, v, scale=0.125))
    chain = saved_shapes(lambda: _chain(bst, q, k, v, 0.125, None))
    assert sparse not in fused and len(fused) == 3, fused
    assert sparse in chain


@pytest.mark.parametrize("dtype,bs,hs", [(F32, 64, 64), (F16, 32, 64), (BF16, 64, 32)],
                         ids=["fp32", "bs32", "hs32"])
def test_fallback_runs_the_chain(dtype, bs, hs):
    lay = _tril(4)
    bst = BlocksparseTransformer(lay, bs, heads=2, mask_callback=causal_callback)
    rng = np.random.default_rng(5)
    q, k, v = (torch.as_tensor(rng.normal(0, 1, (2, 4 * bs, 2 * hs)).astype(np.float32)).to(dtype).cuda() for _ in range(3))
    got = bst.attention(q, k, v, scale=0.25, autoregress_at_key=70)
    assert _lib.last_kernel() != "wgmma_bst_attention"
    ref = _chain(bst, q, k, v, 0.25, 70)
    assert got.dtype == v.dtype and torch.equal(got, ref)


def test_autoregress_without_mask_is_refused():
    bst = BlocksparseTransformer(_tril(2), BS, heads=1)
    with pytest.raises(ValueError, match="mask_callback"):
        bst.attention(*(torch.zeros((1, 128, 64), dtype=F16, device="cuda") for _ in range(3)), autoregress_at_key=3)
