"""Every raw op of the public attention chain, elementwise, on the inputs it was actually given.

weight_value_op(masked_softmax(query_key_op(q, k), scale, autoregress_at_key), v) runs forward and backward with
BlocksparseTransformer._nt, _xn, _softmax and _softmax_grad wrapped, so that every call records its arguments, its
output and the kernel it launched. Then:
  * the wiring: the calls come in the chain's order, each takes the chain's own tensors (which tensor feeds which op, at
    which dtype), and the returned .grad tensors are those calls' outputs bit for bit;
  * each output against float64 of its own recorded inputs: the GEMMs within mma_gemm_bound on the wgmma route and
    fma_gemm_bound on the CUDA-core route (and the route is asserted), the softmax within softmax_bound, the softmax
    gradient within softmax_grad_bound plus one bfloat16 rounding where it is cast.
attention()'s default backward is asserted bit-identical to this chain elsewhere (tests/test_bst_attention_gpu.py), so
these checks cover it as well."""
import collections

import numpy as np
import pytest
import torch

from tests._util import (U_OUT, assert_within, bst_dense, bst_terms, dtype_name, fma_gemm_bound, mma_gemm_bound,
                         softmax_grad_bound, softmax_row_sums)
from tests.golden.make_golden import causal_callback
from tests.test_bst_softmax_gpu import _per_head, _per_head_cb, _tril, softmax_bound
from blocksparse_b200 import BlocksparseTransformer, _lib
from blocksparse_b200.layouts import local_strided_layout
from oracle.bst_oracle import TransformerOracle

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32

Case = collections.namedtuple("Case", "name lay cb ak bs hs dtype heads batch scale")
CASES = [
    Case("tril-f16", _tril(5), causal_callback, None, 64, 64, F16, 2, 2, 0.125),
    Case("tril-bf16", _tril(5), causal_callback, None, 64, 64, BF16, 2, 2, 0.125),
    Case("tril-f32", _tril(5), causal_callback, None, 64, 64, F32, 2, 2, 0.125),
    Case("strided-causal-f16", local_strided_layout(16), causal_callback, None, 64, 64, F16, 2, 1, 0.125),
    Case("strided-causal-bf16-hs128", local_strided_layout(16), causal_callback, None, 64, 128, BF16, 2, 1, 0.125),
    Case("perhead-ak-f16-hs128", _per_head(_tril(6), 3), _per_head_cb, 130, 64, 128, F16, 3, 2, -0.125),
    Case("perhead-ak-bf16", _per_head(_tril(6), 3), _per_head_cb, 130, 64, 64, BF16, 3, 2, 0.25),
    Case("nomask-f16-bs32", np.ones((3, 4), np.int32), None, None, 32, 64, F16, 2, 2, 0.125),
]


def _wgmma(bs, hs, *dtypes):
    """whether csrc/tc_bst.cuh runs a GEMM: one 16-bit dtype for all its operands, block 64, head_state 64 / 128"""
    return bs == 64 and hs in (64, 128) and len(set(dtypes)) == 1 and dtypes[0] in (F16, BF16)


def _record(bst, monkeypatch):
    """Wrap the raw ops of bst; returns the list every call appends (op, args, output, kernel) to. The kernel name is
    kept per thread and autograd runs the backward on a thread of its own, so it is read in the calling thread."""
    calls = []

    def wrap(name, fn):
        def run(*a, **kw):
            assert not kw, (name, kw)
            out = fn(*a)
            calls.append((name, a, out, _lib.last_kernel()))
            return out
        return run
    for name in ("_nt", "_xn", "_softmax", "_softmax_grad"):
        monkeypatch.setattr(bst, name, wrap(name, getattr(bst, name)))
    return calls


def _np(t):
    return t.detach().double().cpu().numpy()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_chain_ops_match_float64_on_their_own_inputs(case, monkeypatch):
    bs, hs, dt, heads, batch, scale = case.bs, case.hs, case.dtype, case.heads, case.batch, case.scale
    bst = BlocksparseTransformer(case.lay, bs, heads=heads, mask_callback=case.cb)
    orc = TransformerOracle(case.lay, bs, heads=heads, mask_callback=case.cb)
    rng = np.random.default_rng(sum(map(ord, case.name)))
    S = heads * hs
    mk = lambda ctx: torch.as_tensor(rng.uniform(-1, 1, (batch, ctx * bs, S)).astype(np.float32)).to(dt).cuda()
    q, k, v = mk(orc.ctx_blks_q), mk(orc.ctx_blks_k), mk(orc.ctx_blks_k)
    dy = torch.as_tensor(rng.normal(0, 1, (batch, orc.ctx_blks_q * bs, S)).astype(np.float32)).to(dt).cuda()
    q.requires_grad_(); k.requires_grad_(); v.requires_grad_()
    calls = _record(bst, monkeypatch)

    y = bst.weight_value_op(bst.masked_softmax(bst.query_key_op(q, k), scale, case.ak), v)
    y.backward(dy)
    assert _lib.device_error() == 0, _lib.device_error_text()

    # ---- wiring ----
    p_dtype = BF16 if dt == F32 else dt
    use_mask = case.cb is not None
    assert [c[0] for c in calls] == ["_nt", "_softmax", "_xn", "_xn", "_nt", "_softmax_grad", "_xn", "_xn"], \
        [c[0] for c in calls]
    (_, a_nt, scores, k_nt), (_, a_sm, p, k_sm), (_, a_nn, y_out, k_nn), (_, a_dv, dv, k_dv), (_, a_dp, dP, k_dp), \
        (_, a_sg, dS_p, k_sg), (_, a_dk, dk, k_dk), (_, a_dq, dq, k_dq) = calls
    dS = a_dk[0]

    def same(t, ref, what):
        assert t.dtype == ref.dtype and torch.equal(t, ref), what
    same(a_nt[0], q, "nt: q"); same(a_nt[1], k, "nt: k"); assert a_nt[2] == BF16 and scores.dtype == BF16
    same(a_sm[0], scores, "softmax: scores")
    assert a_sm[1:] == (scale, use_mask, case.ak, p_dtype) and p.dtype == p_dtype, a_sm[1:]
    same(a_nn[0], p, "nn: p"); same(a_nn[1], v, "nn: v"); assert a_nn[2] is False
    same(y_out, y.detach(), "y")
    same(a_dv[0], p, "dv: p"); same(a_dv[1], dy, "dv: dy"); assert a_dv[2] is True
    same(a_dp[0], dy, "dP: dy"); same(a_dp[1], v, "dP: v"); assert a_dp[2] == p_dtype
    same(a_sg[0], dP, "softmax grad: dP"); same(a_sg[1], p, "softmax grad: p"); assert a_sg[2] == scale
    same(dS, dS_p.to(BF16), "dS: the softmax grad cast to bfloat16")
    assert a_dk[2] is True and a_dq[2] is False
    same(a_dq[0], dS, "dq: dS"); same(a_dk[1], q, "dk: q"); same(a_dq[1], k, "dq: k")
    same(v.grad, dv, "v.grad"); same(k.grad, dk, "k.grad"); same(q.grad, dq, "q.grad")

    # ---- each GEMM against float64 of its recorded inputs, on the route it has to take ----
    for op, a, b, got, kern, what in [("nt", a_nt[0], a_nt[1], scores, k_nt, "scores"),
                                      ("nn", a_nn[0], a_nn[1], y_out, k_nn, "y"),
                                      ("tn", a_dv[0], a_dv[1], dv, k_dv, "dv"),
                                      ("nt", a_dp[0], a_dp[1], dP, k_dp, "dP"),
                                      ("tn", a_dk[0], a_dk[1], dk, k_dk, "dk"),
                                      ("nn", a_dq[0], a_dq[1], dq, k_dq, "dq")]:
        tc = _wgmma(bs, hs, a.dtype, b.dtype)
        want = "wgmma_bst_" + op if tc else ("fma_dds_nt" if op == "nt" else "fma_sdd_xn")
        assert kern == want, (what, kern, want)
        out = dtype_name(got.dtype)
        ref, ref_abs = bst_dense(orc, op, _np(a), _np(b), with_abs=True)
        kt = bst_terms(orc, op, hs)
        bound = (mma_gemm_bound if tc else fma_gemm_bound)(ref, ref_abs, out, kt)
        assert_within(got, ref, bound, "%s %s (%s)" % (case.name, what, kern), ref_abs, kt, out,
                      "wgmma_bst" if tc else None)
    if dt == F16:          # bf16 dS x fp16 q / k: mixed dtypes, which the wgmma kernels refuse
        assert k_dk == k_dq == "fma_sdd_xn"

    # ---- softmax and its gradient ----
    staged = bs in (32, 64) and bst.nn_max <= 16        # bf16 scores in, 16-bit probabilities out at every dtype
    assert k_sm == ("bst_softmax_staged" if staged else "bst_softmax"), k_sm
    assert k_sg == ("bst_softmax_grad_staged" if staged else "bst_softmax_grad"), k_sg
    x = _np(scores)
    pr = orc.masked_softmax(x, scale=scale, autoregress_at_key=case.ak).astype(np.float64)
    amax = float(np.abs(x * scale).max())
    assert_within(p, pr, softmax_bound(pr, p_dtype, amax, bst.nn_max), "%s probabilities (%s)" % (case.name, k_sm))
    dPn, pn = _np(dP), _np(p)
    ds_ref = orc.masked_softmax_grad(dPn, pn, scale=scale)                   # float64
    bound = softmax_grad_bound(ds_ref, dPn, pn, softmax_row_sums(np.abs(dPn * pn), orc), dtype_name(p_dtype), scale,
                               bst.nn_max)
    assert_within(dS_p, ds_ref, bound, "%s softmax grad (%s)" % (case.name, k_sg))
    if p_dtype != BF16:
        bound = bound + U_OUT["bfloat16"] * (np.abs(ds_ref) + bound)         # the cast to the scores' bfloat16
    assert_within(dS, ds_ref, bound, "%s dS" % case.name)
