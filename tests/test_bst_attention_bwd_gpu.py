"""BlocksparseTransformer.attention(..., fused_backward=True): the fused backward kernels (csrc/tc_bst_attn_bwd.cuh)
elementwise against the float64 gradients of tests/_attention_grad_oracle.py, their determinism, what autograd keeps,
that the chain's kernels stay out of it, and the fallback to the chain's backward where no fused kernel exists."""
import collections
import json
import os

import numpy as np
import pytest
import torch

from tests._util import (EPS32, MMA_C, SUBNORMAL_FLOOR, U_OUT, _on_poisoned_output, assert_within, record_kernels,
                         ref_errors)
from tests.golden.make_golden import causal_callback
from tests.test_bst_attention_gpu import (_future_first, _hide_row_cb, _hole, _ones_cb, _per_head, _per_head_cb, _rect,
                                          _tril)
from blocksparse_b200 import BlocksparseTransformer, _lib
from blocksparse_b200.layouts import local_strided_layout
from oracle.bst_oracle import TransformerOracle
from tests._attention_grad_oracle import attention_probs, oracle_attention_grad

gpu = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
_NAME = {BF16: "bfloat16", F16: "float16", F32: "float32"}
BS = 64


def _key_hole(lay, k):
    """no query block sees key block k"""
    lay = lay.copy()
    lay[..., :, k] = 0
    return lay


Case = collections.namedtuple("Case", "name lay cb ak hs scale heads batch")
CASES = [
    Case("tril20-causal", _tril(20), causal_callback, None, 64, 0.125, 3, 2),           # rows of 1..20 blocks
    Case("tril20-nomask", _tril(20), None, None, 128, 0.125, 3, 2),
    Case("cfg3-causal", local_strided_layout(64), causal_callback, None, 64, 0.125, 1, 1),   # the cfg 3 layout
    Case("strided16-causal-ak", local_strided_layout(16), causal_callback, 300, 128, 0.125, 3, 2),
    Case("perhead-mask", _per_head(_tril(6), 3), _per_head_cb, None, 64, 0.25, 3, 2),
    Case("perhead-ak", _per_head(_tril(7), 3), _per_head_cb, 130, 128, -0.125, 3, 2),
    Case("hole-hiderow", _hole(_tril(6), 2), _hide_row_cb, None, 128, 0.125, 3, 2),
    Case("hole-nomask", _hole(_tril(5), 0), None, None, 64, 0.125, 3, 2),
    Case("keyhole-perhead", _per_head(_key_hole(_tril(6), 2), 3), causal_callback, None, 128, 0.125, 3, 2),
    Case("rect-nomask", _rect(), None, None, 64, 0.125, 3, 2),
    Case("rect-ak", _rect(), _ones_cb, 100, 128, 0.125, 3, 2),
    Case("future-ak0", _future_first(5), _ones_cb, 0, 64, 0.125, 3, 2),
]


def _inputs(lay, hs, dtype, seed, heads, batch):
    lay3 = lay if lay.ndim == 3 else lay[None]
    cq, ck = lay3.shape[1:]
    rng = np.random.default_rng(seed)
    q, dy = (rng.normal(0, 1, (batch, cq * BS, heads * hs)) for _ in range(2))
    k, v = (rng.normal(0, 1, (batch, ck * BS, heads * hs)) for _ in range(2))
    return [torch.as_tensor(a.astype(np.float32)).to(dtype) for a in (q, k, v, dy)]


def _split(X, heads):
    B, ctx, S = X.shape
    return np.abs(X.reshape(B, ctx, heads, S // heads).transpose(0, 2, 1, 3).astype(np.float64))


def _merge(Xh):
    B, H, ctx, hs = Xh.shape
    return Xh.transpose(0, 2, 1, 3).reshape(B, ctx, H * hs)


def grad_bound(orc, Q, K, V, dY, scale, ak, hs, dtype):
    """Largest |got - ref| of the fused dq, dk and dv, elementwise (float64 arrays of the inputs' shapes).

    With P the float64 probabilities, dP = dY V^T, D = rowsum(P dP), A = P |V| (what bounds |O|), L / T the longest
    nn_lut / tn_lut row in blocks, qk the largest entry of |Q| |K|^T and u_in the rounding of the input dtype:
      * P recomputed in the backward: the forward's bound on its relative error (attention_bound's rel without u_in:
        the scores' accumulation twice, in the backward's S and in the forward's m and l, the exponent arithmetic, l's
        sums and rescales), plus 8 eps32 for the backward's own scale, subtraction, log2 e, exp2f (2 ulp), 1/l and
        multiply: e_P;
      * dP accumulates hs products: MMA_C eps32 hs (|dY| |V|^T);
      * D is summed from the stored 16-bit o: |o - O| <= (u_in + rel) A, and hs + 2 fp32 roundings of its sum:
        e_D sum_c |dY| A;
      * dS = scale P (dP - D) in fp32 (three roundings), rounded to the input dtype (u_in): per element
        W = |scale| P ((e_P + u_in + 4 eps32) |dP - D| + MMA_C eps32 hs |dY||V|^T + e_D sum_c |dY| A);
      * dQ = dS K accumulates 64 L products, dK = dS^T Q 64 T: MMA_C eps32 64 L |dS| |K| and MMA_C eps32 64 T |dS|^T |Q|,
        plus W |K| and W^T |Q| from the errors of dS;
      * dV = P^T dY with P rounded to the input dtype: (e_P + u_in + MMA_C eps32 64 T) P^T |dY|;
      * one rounding of each output (u_in |ref|); below fp16's normal range P and dS round with an absolute 2^-25,
        at most 64 L (64 T) of them per element, and the output's own subnormal floor."""
    u = U_OUT[_NAME[dtype]]
    sub = SUBNORMAL_FLOOR[_NAME[dtype]]
    heads = orc.heads
    Qa, Ka, Va, dYa = (_split(X, heads) for X in (Q, K, V, dY))
    Qs, Ks, Vs, dYs = (X.reshape(X.shape[0], X.shape[1], heads, -1).transpose(0, 2, 1, 3).astype(np.float64)
                       for X in (Q, K, V, dY))
    P = attention_probs(orc, Q, K, scale, ak)
    dP = dYs @ Vs.transpose(0, 1, 3, 2)
    D = (P * dP).sum(axis=-1, keepdims=True)
    M = dYa @ Va.transpose(0, 1, 3, 2)
    A = P @ Va
    Dabs = (dYa * A).sum(axis=-1, keepdims=True)
    L = max(len(r) for rows in orc.nn_list for r in rows)
    T = max(len(r) for rows in orc.tn_list for r in rows)
    qk = float((Qa @ Ka.transpose(0, 1, 3, 2)).max())
    amax = abs(scale) * qk
    rel = EPS32 * (2 * MMA_C * hs * abs(scale) * qk + 16 * amax + MMA_C * 64 * L + 16 * L + 64)
    e_p = rel + 8 * EPS32
    e_d = u + rel + EPS32 * (hs + 2)
    dS = abs(scale) * P * np.abs(dP - D)
    W = abs(scale) * P * ((e_p + u + 4 * EPS32) * np.abs(dP - D) + MMA_C * EPS32 * hs * M + e_d * Dabs)
    dQ, dK, dV = oracle_attention_grad(orc, Q, K, V, dY, scale, ak)
    bq = (u * np.abs(dQ) + _merge((W + MMA_C * EPS32 * 64 * L * dS) @ Ka)
          + sub * 64 * L * float(np.abs(K).max()) + sub)
    Wt, dSt = W.transpose(0, 1, 3, 2), dS.transpose(0, 1, 3, 2)
    bk = (u * np.abs(dK) + _merge((Wt + MMA_C * EPS32 * 64 * T * dSt) @ Qa)
          + sub * 64 * T * float(np.abs(Q).max()) + sub)
    bv = (u * np.abs(dV) + (e_p + u + MMA_C * EPS32 * 64 * T) * _merge(P.transpose(0, 1, 3, 2) @ dYa)
          + sub * 64 * T * float(np.abs(dY).max()) + sub)
    return (dQ, dK, dV), (bq, bk, bv)


def _case_id(c):
    return c.name + "-hs%d" % c.hs


def _chain(bst, q, k, v, scale, ak):
    return bst.weight_value_op(bst.masked_softmax(bst.query_key_op(q, k), scale, ak), v)


def _grads(bst, q, k, v, dy, scale, ak, fused_backward, need=(True, True, True)):
    ins = [t.clone().requires_grad_(n) for t, n in zip((q, k, v), need)]
    y = bst.attention(*ins, scale=scale, autoregress_at_key=ak, fused_backward=fused_backward)
    y.backward(dy)
    return y, [t.grad for t in ins]


def _log(rec):
    path = os.environ.get("BSMM_GRAD_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(rec) + "\n")


@gpu
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("idx", range(len(CASES)), ids=[_case_id(c) for c in CASES])
def test_fused_backward_matches_oracle(idx, dtype):
    case = CASES[idx]
    bst = BlocksparseTransformer(case.lay, BS, heads=case.heads, mask_callback=case.cb)
    orc = TransformerOracle(case.lay, BS, heads=case.heads, mask_callback=case.cb)
    q, k, v, dy = _inputs(case.lay, case.hs, dtype, 200 + idx, case.heads, case.batch)
    qc, kc, vc, dyc = (t.cuda() for t in (q, k, v, dy))
    _, got = _grads(bst, qc, kc, vc, dyc, case.scale, case.ak, True)
    assert _lib.device_error() == 0, _lib.device_error_text()
    Q, K, V, dY = (t.double().numpy() for t in (q, k, v, dy))
    refs, bounds = grad_bound(orc, Q, K, V, dY, case.scale, case.ak, case.hs, dtype)
    _, chain = _grads(bst, qc, kc, vc, dyc, case.scale, case.ak, False)
    for name, g, ref, bound, c in zip(("dq", "dk", "dv"), got, refs, bounds, chain):
        assert g.dtype == dtype and not bool(torch.isnan(g).any()), name
        gd = g.double().cpu().numpy()
        frac = float(np.max(np.abs(gd - ref) / bound))
        l2 = ref_errors(gd, ref)[1]
        _log({"case": _case_id(case), "dtype": _NAME[dtype], "grad": name, "frac": frac, "l2": l2,
              "chain_l2": ref_errors(c.double().cpu().numpy(), ref)[1]})
        assert_within(g, ref, bound, "%s %s" % (name, _case_id(case)))
        assert l2 < 1e-2, (name, l2)
    # determinism: a second backward gives the same bits
    _, again = _grads(bst, qc, kc, vc, dyc, case.scale, case.ak, True)
    for a, b in zip(got, again):
        assert torch.equal(a, b)


@gpu
def test_fused_backward_zero_fills_empty_blocks_on_poisoned_memory():
    """Every gradient element is written, including those of the empty query block and the key block no query sees:
    outputs, statistics and the delta workspace come from NaN-filled allocations."""
    lay = _hole(_key_hole(_tril(6), 2), 4)
    bst = BlocksparseTransformer(lay, BS, heads=2, mask_callback=causal_callback)
    q, k, v, dy = (t.cuda() for t in _inputs(lay, 64, BF16, 5, 2, 2))

    def run():
        o, m, l = bst._attention_train(q, k, v, 0.125, None)
        return bst._attention_grad(q, k, v, o, dy, m, l, 0.125, None)
    dq, dk, dv = _on_poisoned_output(run)
    assert _lib.device_error() == 0, _lib.device_error_text()
    for g in (dq, dk, dv):
        assert not bool(torch.isnan(g).any())
    assert bool((dq[:, 4 * BS:5 * BS] == 0).all())
    assert bool((dk[:, 2 * BS:3 * BS] == 0).all()) and bool((dv[:, 2 * BS:3 * BS] == 0).all())


def test_cases_cover_the_envelope():
    """The covering set reaches what the kernels have to handle (pure Python; guards later edits)."""
    lays = [c.lay if c.lay.ndim == 3 else c.lay[None] for c in CASES]
    assert {c.hs for c in CASES} == {64, 128}
    assert any(l.shape[-1] >= 20 and l.sum(axis=-1).max() >= 20 for l in lays)          # rows of up to 20 blocks
    assert any(c.name.startswith("cfg3") and c.lay.shape == (64, 64) and c.lay.sum() == 453 for c in CASES)
    assert any(c.lay.ndim == 3 and c.cb is _per_head_cb for c in CASES)                  # per-head layouts and masks
    assert any(l.shape[-2] != l.shape[-1] for l in lays)                                  # rectangular
    assert any((l.sum(axis=-1) == 0).any() for l in lays)                                 # an empty query block
    assert any((l.sum(axis=-2) == 0).any() for l in lays)                                 # an empty key column
    assert any(c.ak is not None for c in CASES) and any(c.ak == 0 and c.lay[0, 0] == 0 for c in CASES)   # _future_first
    assert any(c.scale < 0 for c in CASES)
    assert {None, causal_callback, _per_head_cb, _hide_row_cb} <= {c.cb for c in CASES}


@gpu
def test_forward_and_gradient_subsets_are_unchanged():
    lay = _per_head(_tril(7), 3)
    for hs, dtype in ((64, F16), (128, BF16)):
        bst = BlocksparseTransformer(lay, BS, heads=3, mask_callback=_per_head_cb)
        q, k, v, dy = (t.cuda() for t in _inputs(lay, hs, dtype, 9, 3, 2))
        base = bst.attention(q, k, v, scale=0.125, autoregress_at_key=130)
        y, full = _grads(bst, q, k, v, dy, 0.125, 130, True)
        assert torch.equal(y, base), "the forward output differs from the default attention's"
        for need in ((False, False, True), (True, False, False), (False, True, True)):
            _, part = _grads(bst, q, k, v, dy, 0.125, 130, True, need)
            for n, a, b in zip(need, part, full):
                assert (a is None) if not n else torch.equal(a, b)
    assert _lib.device_error() == 0, _lib.device_error_text()


@gpu
def test_fused_backward_saves_no_sparse_tensor_and_skips_the_chain(monkeypatch):
    lay = local_strided_layout(16)
    bst = BlocksparseTransformer(lay, BS, heads=3, mask_callback=causal_callback)
    q, k, v, dy = (t.cuda() for t in _inputs(lay, 64, F16, 11, 3, 2))
    qq, kk, vv = (t.clone().requires_grad_() for t in (q, k, v))
    sparse = (2, 3, bst.blocks, BS, BS)
    shapes = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: shapes.append(tuple(t.shape)) or t, lambda t: t):
        y = bst.attention(qq, kk, vv, scale=0.125, fused_backward=True)
    assert sparse not in shapes and len(shapes) == 6, shapes
    calls, seen = [], []
    for name in ("_nt", "_softmax", "_softmax_grad", "_xn"):
        monkeypatch.setattr(bst, name, lambda *a, _n=name, **kw: calls.append(_n))
    record_kernels(monkeypatch, bst, ["_attention_grad"], seen)
    y.backward(dy)
    assert not calls, calls
    assert seen == [("_attention_grad", "wgmma_bst_attention_bwd_dkdv")], seen
    assert _lib.device_error() == 0, _lib.device_error_text()


@gpu
@pytest.mark.parametrize("dtype,bs,hs", [(F32, 64, 64), (F16, 32, 64), (BF16, 64, 32)], ids=["fp32", "bs32", "hs32"])
def test_outside_the_envelope_gradients_are_the_chains(dtype, bs, hs):
    lay = _tril(4)
    bst = BlocksparseTransformer(lay, bs, heads=2, mask_callback=causal_callback)
    rng = np.random.default_rng(5)
    q, k, v, dy = (torch.as_tensor(rng.normal(0, 1, (2, 4 * bs, 2 * hs)).astype(np.float32)).to(dtype).cuda()
                   for _ in range(4))
    y, got = _grads(bst, q, k, v, dy, 0.25, 70, True)
    ins = [t.clone().requires_grad_() for t in (q, k, v)]
    _chain(bst, *ins, 0.25, 70).backward(dy)
    assert torch.equal(y, _chain(bst, q, k, v, 0.25, 70))
    for a, b in zip(got, ins):
        assert torch.equal(a, b.grad)
