"""BlocksparseTransformer.attention(..., keep_prob < 1): attention dropout inside the fused kernels
(csrc/tc_bst_attn.cuh, csrc/tc_bst_attn_bwd.cuh) elementwise against the float64 oracle of
tests/_attention_dropout_oracle.py, the mask against ewops.dropout's at the same (seed, call), the default backward bit
for bit against the chain with ewops.dropout, the dropout state, the fallback outside the fused envelope, side streams,
CUDA graphs and element indices past 2^32."""
import numpy as np
import pytest
import torch

from tests._util import EPS32, MMA_C, SUBNORMAL_FLOOR, U_OUT, _on_poisoned_output, assert_within, record_kernels
from tests.golden.make_golden import causal_callback
from tests import test_bst_attention_bwd_gpu as bwd_cases
from tests import test_bst_attention_gpu as fwd_cases
from tests.test_bst_attention_gpu import _per_head, _per_head_cb, _tril
from blocksparse_b200 import BlocksparseTransformer, _lib, ewops
from oracle.bst_oracle import TransformerOracle
from tests._attention_dropout_oracle import (attention_keep, oracle_attention_dropout, oracle_attention_dropout_grad)
from tests._attention_grad_oracle import attention_probs

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
_NAME = {BF16: "bfloat16", F16: "float16", F32: "float32"}
BS = 64
SEED, CALL = 0x0123_4567_89AB_CDEF, 41


def _state(seed=SEED, call=CALL):
    return torch.tensor([seed, call], dtype=torch.int64, device="cuda")


def _split(X, heads):
    B, ctx, S = X.shape
    return X.reshape(B, ctx, heads, S // heads).transpose(0, 2, 1, 3).astype(np.float64)


def _merge(Xh):
    B, H, ctx, hs = Xh.shape
    return Xh.transpose(0, 2, 1, 3).reshape(B, ctx, H * hs)


def dropout_attention_bound(orc, ref, Q, K, V, Z, kp, scale, ak, hs, dtype):
    """attention_bound of tests/test_bst_attention_gpu.py with |P| replaced by |P o Z| / keep_prob: A = (P o Z / kp)
    |V| weighs the relative errors, the subnormal floor of the unnormalised probabilities is scaled by 1 / kp, and the
    epilogue's fp32(1 / kp) / l adds one rounding."""
    u_in = U_OUT[_NAME[dtype]]
    B, ctxq, S = Q.shape
    heads = S // hs
    A = oracle_attention_dropout(orc, Q, K, np.abs(V), Z, kp, scale, ak)
    Qh, Kh = np.abs(_split(Q, heads)), np.abs(_split(K, heads))
    qk = float((Qh @ Kh.transpose(0, 1, 3, 2)).max())
    amax = abs(scale) * qk
    L = np.array([[len(orc.nn_list[orc._hl(h)][r // BS]) for h in range(heads)] for r in range(ctxq)], np.float64)
    L = np.broadcast_to(L[None, :, :, None], (B, ctxq, heads, hs)).reshape(B, ctxq, S)
    rel = u_in + EPS32 * (2 * MMA_C * hs * abs(scale) * qk + 16 * amax + MMA_C * 64 * L + 16 * L + 66)
    sub = SUBNORMAL_FLOOR[_NAME[dtype]]
    return u_in * np.abs(ref) + rel * A + sub * 64 * L * float(np.abs(V).max()) / kp + sub, L


def dropout_grad_bound(orc, Q, K, V, dY, Z, kp, scale, ak, hs, dtype):
    """grad_bound of tests/test_bst_attention_bwd_gpu.py with P o Z / keep_prob where the probabilities meet dY and V:
    dP = Z o (dY V^T) / kp, A = (P o Z / kp) |V|, dV's P^T |dY| becomes (P o Z / kp)^T |dY|; 1 / kp costs one more
    rounding in dS (scale / kp), in D (kp D) and in dV (the epilogue's 1 / kp)."""
    u = U_OUT[_NAME[dtype]]
    sub = SUBNORMAL_FLOOR[_NAME[dtype]]
    heads = orc.heads
    Qa, Ka, Va, dYa = (np.abs(_split(X, heads)) for X in (Q, K, V, dY))
    Vs, dYs = _split(V, heads), _split(dY, heads)
    P = attention_probs(orc, Q, K, scale, ak)
    Pz = np.where(Z, P, 0.0) / kp
    dP = np.where(Z, dYs @ Vs.transpose(0, 1, 3, 2), 0.0) / kp
    D = (P * dP).sum(axis=-1, keepdims=True)
    M = np.where(Z, dYa @ Va.transpose(0, 1, 3, 2), 0.0) / kp
    A = Pz @ Va
    Dabs = (dYa * A).sum(axis=-1, keepdims=True)
    L = max(len(r) for rows in orc.nn_list for r in rows)
    T = max(len(r) for rows in orc.tn_list for r in rows)
    qk = float((Qa @ Ka.transpose(0, 1, 3, 2)).max())
    amax = abs(scale) * qk
    rel = EPS32 * (2 * MMA_C * hs * abs(scale) * qk + 16 * amax + MMA_C * 64 * L + 16 * L + 64)
    e_p = rel + 8 * EPS32
    e_d = u + rel + EPS32 * (hs + 3)
    dS = abs(scale) * P * np.abs(dP - D)
    W = abs(scale) * P * ((e_p + u + 5 * EPS32) * np.abs(dP - D) + MMA_C * EPS32 * hs * M + e_d * Dabs)
    dQ, dK, dV = oracle_attention_dropout_grad(orc, Q, K, V, dY, Z, kp, scale, ak)
    bq = u * np.abs(dQ) + _merge((W + MMA_C * EPS32 * 64 * L * dS) @ Ka) + sub * 64 * L * float(np.abs(K).max()) + sub
    Wt, dSt = W.transpose(0, 1, 3, 2), dS.transpose(0, 1, 3, 2)
    bk = u * np.abs(dK) + _merge((Wt + MMA_C * EPS32 * 64 * T * dSt) @ Qa) + sub * 64 * T * float(np.abs(Q).max()) + sub
    bv = (u * np.abs(dV) + (e_p + u + EPS32 + MMA_C * EPS32 * 64 * T) * _merge(Pz.transpose(0, 1, 3, 2) @ dYa)
          + sub * 64 * T * float(np.abs(dY).max()) / kp + sub)
    return (dQ, dK, dV), (bq, bk, bv)


def _chain(bst, q, k, v, scale, ak, kp, mask=None):
    """weight_value_op(ewops.dropout(masked_softmax(query_key_op(q, k)), keep_prob), v): draws from the device state
    without `mask`"""
    p = bst.masked_softmax(bst.query_key_op(q, k), scale, ak)
    return bst.weight_value_op(ewops.dropout(p, kp, mask=mask)[0], v)


def _np(*ts):
    return [t.double().cpu().numpy() for t in ts]


KPS = [0.9, 0.5]


# ---- forward ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kp", KPS)
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("idx", range(len(fwd_cases.CASES)), ids=[fwd_cases._case_id(c) for c in fwd_cases.CASES])
def test_forward_matches_oracle(idx, dtype, kp):
    case = fwd_cases.CASES[idx]
    heads, batch = fwd_cases.HEADS, fwd_cases.BATCH
    bst = BlocksparseTransformer(case.lay, BS, heads=heads, mask_callback=case.cb)
    orc = TransformerOracle(case.lay, BS, heads=heads, mask_callback=case.cb)
    q, k, v = fwd_cases._inputs(case.lay, case.hs, dtype, 300 + idx)
    qc, kc, vc = q.cuda(), k.cuda(), v.cuda()
    st = _state(call=CALL + idx)
    out = _on_poisoned_output(lambda: bst.attention(qc, kc, vc, scale=case.scale, autoregress_at_key=case.ak,
                                                    keep_prob=kp, dropout_state=st))
    assert _lib.last_kernel() == "wgmma_bst_attention_dropout"
    assert _lib.device_error() == 0, _lib.device_error_text()
    assert out.dtype == dtype and not bool(torch.isnan(out).any())
    Q, K, V = _np(q, k, v)
    Z = attention_keep(orc, batch, SEED, CALL + idx, kp)
    ref = oracle_attention_dropout(orc, Q, K, V, Z, kp, case.scale, case.ak)
    bound, L = dropout_attention_bound(orc, ref, Q, K, V, Z, kp, case.scale, case.ak, case.hs, dtype)
    assert bool((out.double().cpu().numpy()[L == 0] == 0).all()), "empty query blocks are not zero"
    assert_within(out, ref, bound, "dropout attention %s kp %g" % (fwd_cases._case_id(case), kp))
    # the mask is ewops.dropout's at the same (seed, call): the chain lies within the same bound of the oracle, and of
    # the fused output (the chain's bf16 scores add their rounding)
    chain = _chain(bst, qc, kc, vc, case.scale, case.ak, kp,
                   mask=ewops._mask_at(qc, batch * heads * bst.blocks * BS * BS, kp, st))
    scores = U_OUT["bfloat16"] * 2 * abs(case.scale) * float(
        (np.abs(_split(Q, heads)) @ np.abs(_split(K, heads)).transpose(0, 1, 3, 2)).max())
    assert_within(out, chain.double().cpu().numpy(), 2 * bound + scores * oracle_attention_dropout(
        orc, Q, K, np.abs(V), Z, kp, case.scale, case.ak), "fused vs chain %s" % fwd_cases._case_id(case))


# ---- fused backward --------------------------------------------------------------------------------------------------
def _grads(bst, q, k, v, dy, scale, ak, fused_backward, kp, state=None):
    ins = [t.clone().requires_grad_() for t in (q, k, v)]
    y = bst.attention(*ins, scale=scale, autoregress_at_key=ak, fused_backward=fused_backward, keep_prob=kp,
                      dropout_state=state)
    y.backward(dy)
    return y, [t.grad for t in ins]


@pytest.mark.parametrize("kp", KPS)
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("idx", range(len(bwd_cases.CASES)), ids=[bwd_cases._case_id(c) for c in bwd_cases.CASES])
def test_fused_backward_matches_oracle(idx, dtype, kp, monkeypatch):
    case = bwd_cases.CASES[idx]
    bst = BlocksparseTransformer(case.lay, BS, heads=case.heads, mask_callback=case.cb)
    orc = TransformerOracle(case.lay, BS, heads=case.heads, mask_callback=case.cb)
    q, k, v, dy = bwd_cases._inputs(case.lay, case.hs, dtype, 400 + idx, case.heads, case.batch)
    qc, kc, vc, dyc = (t.cuda() for t in (q, k, v, dy))
    seen = []
    record_kernels(monkeypatch, bst, ["_attention_train", "_attention_grad"], seen)
    _, got = _grads(bst, qc, kc, vc, dyc, case.scale, case.ak, True, kp, _state(call=CALL + idx))
    assert [s[1] for s in seen] == ["wgmma_bst_attention_train_dropout", "wgmma_bst_attention_bwd_dkdv_dropout"], seen
    assert _lib.device_error() == 0, _lib.device_error_text()
    Q, K, V, dY = _np(q, k, v, dy)
    Z = attention_keep(orc, case.batch, SEED, CALL + idx, kp)
    refs, bounds = dropout_grad_bound(orc, Q, K, V, dY, Z, kp, case.scale, case.ak, case.hs, dtype)
    for name, g, ref, bound in zip(("dq", "dk", "dv"), got, refs, bounds):
        assert g.dtype == dtype and not bool(torch.isnan(g).any()), name
        assert_within(g, ref, bound, "%s %s kp %g" % (name, bwd_cases._case_id(case), kp))


def test_fused_backward_zero_fills_empty_blocks_on_poisoned_memory():
    lay = bwd_cases._hole(bwd_cases._key_hole(_tril(6), 2), 4)
    bst = BlocksparseTransformer(lay, BS, heads=2, mask_callback=causal_callback)
    q, k, v, dy = (t.cuda() for t in bwd_cases._inputs(lay, 64, BF16, 5, 2, 2))
    st = _state()

    def run():
        o, m, l = bst._attention_train(q, k, v, 0.125, None, 0.5, st)
        return bst._attention_grad(q, k, v, o, dy, m, l, 0.125, None, 0.5, st)
    dq, dk, dv = _on_poisoned_output(run)
    assert _lib.device_error() == 0, _lib.device_error_text()
    for g in (dq, dk, dv):
        assert not bool(torch.isnan(g).any())
    assert bool((dq[:, 4 * BS:5 * BS] == 0).all())
    assert bool((dk[:, 2 * BS:3 * BS] == 0).all()) and bool((dv[:, 2 * BS:3 * BS] == 0).all())


# ---- default backward: the chain's, bit for bit ----------------------------------------------------------------------
@pytest.mark.parametrize("kp", KPS)
@pytest.mark.parametrize("dtype", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("lay,cb,ak,hs", [(_tril(6), None, None, 64), (_tril(6), causal_callback, None, 64),
                                          (_per_head(_tril(7), 3), _per_head_cb, 130, 128),
                                          (fwd_cases._hole(_tril(6), 2), fwd_cases._hide_row_cb, None, 128)],
                         ids=["nomask", "causal", "perhead-ak-hs128", "hole-hiderow-hs128"])
def test_default_backward_is_bit_identical_to_the_chain(lay, cb, ak, hs, dtype, kp, monkeypatch):
    bst = BlocksparseTransformer(lay, BS, heads=3, mask_callback=cb)
    q, k, v = (t.cuda() for t in fwd_cases._inputs(lay, hs, dtype, 7))
    dy = torch.randn(q.shape, generator=torch.Generator().manual_seed(3)).to(dtype).cuda()
    state = ewops.get_entropy(q.device)
    saved = state.clone()
    seen = []
    record_kernels(monkeypatch, bst, ["_attention"], seen)
    _, fused = _grads(bst, q, k, v, dy, 0.125, ak, False, kp)            # draws from the device state
    assert seen == [("_attention", "wgmma_bst_attention_dropout")], seen
    state.copy_(saved)
    ins = [t.clone().requires_grad_() for t in (q, k, v)]
    _chain(bst, *ins, 0.125, ak, kp).backward(dy)                       # the same (seed, call)
    assert _lib.device_error() == 0, _lib.device_error_text()
    for name, a, b in zip("qkv", fused, ins):
        assert a.dtype == b.grad.dtype and torch.equal(a, b.grad), "d%s differs from the chain's" % name
    # only some inputs need a gradient
    vv = v.clone().requires_grad_()
    bst.attention(q, k, vv, scale=0.125, autoregress_at_key=ak, keep_prob=kp, dropout_state=saved).backward(dy)
    assert torch.equal(vv.grad, ins[2].grad)


# ---- state -----------------------------------------------------------------------------------------------------------
def _small():
    lay = _tril(4)
    bst = BlocksparseTransformer(lay, BS, heads=2, mask_callback=causal_callback)
    q, k, v, dy = (t.cuda() for t in bwd_cases._inputs(lay, 64, F16, 13, 2, 2))
    return bst, q, k, v, dy


@pytest.mark.parametrize("fused_backward", [False, True])
def test_device_state_advances_by_one_per_call(fused_backward):
    bst, q, k, v, dy = _small()
    state = ewops.get_entropy(q.device)
    before = state.clone()
    y1, g1 = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 0.8)
    assert state[0].item() == before[0].item() and state[1].item() == before[1].item() + 1
    y2, _ = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 0.8)
    assert state[1].item() == before[1].item() + 2 and not torch.equal(y1, y2)
    # the first call is what an explicit state at its (seed, call) gives
    y3, g3 = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 0.8, before.clone())
    assert torch.equal(y1, y3) and all(torch.equal(a, b) for a, b in zip(g1, g3))
    assert state[1].item() == before[1].item() + 2


@pytest.mark.parametrize("fused_backward", [False, True])
def test_keep_prob_one_reads_and_advances_nothing(fused_backward):
    bst, q, k, v, dy = _small()
    state = ewops.get_entropy(q.device)
    before = state.clone()
    y0, g0 = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 1.0)
    y1, g1 = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 1.0, _state())
    ins = [t.clone().requires_grad_() for t in (q, k, v)]
    y = bst.attention(*ins, scale=0.125, fused_backward=fused_backward)
    y.backward(dy)
    assert torch.equal(state, before)
    for a in (y0, y1):
        assert torch.equal(a, y)
    for g in (g0, g1):
        assert all(torch.equal(a, b.grad) for a, b in zip(g, ins))


@pytest.mark.parametrize("fused_backward", [False, True])
def test_given_state_is_neither_changed_nor_moves_the_device_state(fused_backward):
    bst, q, k, v, dy = _small()
    state = ewops.get_entropy(q.device)
    before = state.clone()
    st = _state()
    ya, ga = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 0.7, st)
    yb, gb = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 0.7, st)
    assert torch.equal(st, _state()) and torch.equal(state, before)
    assert torch.equal(ya, yb) and all(torch.equal(a, b) for a, b in zip(ga, gb))
    yc, _ = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 0.7, _state(call=CALL + 1))
    assert not torch.equal(ya, yc)


def test_bad_arguments_are_refused():
    bst, q, k, v, _ = _small()
    for kp in (0.0, -0.5, 1.5, True, "0.5", None):
        with pytest.raises(ValueError, match="keep_prob"):
            bst.attention(q, k, v, keep_prob=kp)
    for st in (torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.int32, device="cuda"),
               torch.zeros(3, dtype=torch.int64, device="cuda"), [SEED, CALL]):
        with pytest.raises(ValueError, match="dropout_state"):
            bst.attention(q, k, v, keep_prob=0.5, dropout_state=st)


# ---- outside the fused envelope: the chain with the same mask --------------------------------------------------------
@pytest.mark.parametrize("fused_backward", [False, True])
@pytest.mark.parametrize("dtype,bs,hs", [(F32, 64, 64), (F16, 32, 64), (BF16, 64, 32)], ids=["fp32", "bs32", "hs32"])
def test_fallback_runs_the_chain_with_the_same_mask(dtype, bs, hs, fused_backward):
    lay = _tril(4)
    heads, batch, kp = 2, 2, 0.6
    bst = BlocksparseTransformer(lay, bs, heads=heads, mask_callback=causal_callback)
    orc = TransformerOracle(lay, bs, heads=heads, mask_callback=causal_callback)
    rng = np.random.default_rng(5)
    q, k, v, dy = (torch.as_tensor(rng.normal(0, 1, (batch, 4 * bs, heads * hs)).astype(np.float32)).to(dtype).cuda()
                   for _ in range(4))
    state = ewops.get_entropy(q.device)
    saved = state.clone()
    y, got = _grads(bst, q, k, v, dy, 0.25, 70, fused_backward, kp)
    assert not _lib.last_kernel().startswith("wgmma_bst_attention")
    assert state[1].item() == saved[1].item() + 1
    state.copy_(saved)
    ins = [t.clone().requires_grad_() for t in (q, k, v)]
    ref = _chain(bst, *ins, 0.25, 70, kp)
    ref.backward(dy)
    assert torch.equal(y, ref)
    for a, b in zip(got, ins):
        assert torch.equal(a, b.grad)
    Q, K, V = _np(q, k, v)
    Z = attention_keep(orc, batch, int(saved[0].item()), int(saved[1].item()), kp)
    o = oracle_attention_dropout(orc, Q, K, V, Z, kp, 0.25, 70)
    err = np.linalg.norm(y.detach().double().cpu().numpy() - o) / np.linalg.norm(o)
    assert err < 2e-2, err


# ---- execution contexts ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fused_backward", [False, True])
def test_side_stream_matches_default_stream(fused_backward):
    bst, q, k, v, dy = _small()
    y0, g0 = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 0.75, _state())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        y1, g1 = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 0.75, _state())
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert torch.equal(y0, y1) and all(torch.equal(a, b) for a, b in zip(g0, g1))


@pytest.mark.parametrize("fused_backward", [False, True])
def test_cuda_graph_replays_draw_new_masks(fused_backward):
    bst, q, k, v, dy = _small()
    state = ewops.get_entropy(q.device)            # created before capture
    ins = [t.clone().requires_grad_() for t in (q, k, v)]

    def step():
        for t in ins:
            t.grad = None
        y = bst.attention(*ins, scale=0.125, fused_backward=fused_backward, keep_prob=0.8)
        y.backward(dy)
        return y

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                  # warm-up: LUT upload, tensor maps, allocator
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = step()
    for _ in range(3):
        before = state.clone()
        g.replay()
        torch.cuda.synchronize()
        assert state[1].item() == before[1].item() + 1
        ye, ge = _grads(bst, q, k, v, dy, 0.125, None, fused_backward, 0.8, before)
        assert torch.equal(y, ye)
        assert all(torch.equal(t.grad, e) for t, e in zip(ins, ge))


# ---- element indices past 2^32 ---------------------------------------------------------------------------------------
def test_element_index_past_2_32():
    """batch 32, one head of state 64, a dense 256 x 256-block layout: e reaches 2^33. o and the fused dq of sampled
    rows of the last batches against float64."""
    nb, batch, hs, kp, scale = 256, 32, 64, 0.5, 0.125
    lay = np.ones((nb, nb), np.int32)
    bst = BlocksparseTransformer(lay, BS, heads=1)
    orc = TransformerOracle(lay, BS, heads=1)
    assert batch * bst.blocks * BS * BS == 2 ** 33
    gen = torch.Generator(device="cuda").manual_seed(1)
    q, k, v, dy = ((torch.rand((batch, nb * BS, hs), generator=gen, device="cuda") * 2 - 1).half() for _ in range(4))
    y, (dq, _, _) = _grads(bst, q, k, v, dy, scale, None, True, kp, _state())
    assert _lib.device_error() == 0, _lib.device_error_text()
    rows = np.array([0, 777, nb * BS // 2 + 5, nb * BS - 1])
    for b in (batch // 2, batch - 1):
        Q, K, V, dY = (t[b].double().cpu().numpy() for t in (q, k, v, dy))
        Z = attention_keep(orc, batch, SEED, CALL, kp, batches=[b], rows=rows)[0, 0]
        s = Q[rows] @ K.T * scale
        P = np.exp(s - s.max(axis=1, keepdims=True))
        P /= P.sum(axis=1, keepdims=True)
        Pz = np.where(Z, P, 0.0) / kp
        o = Pz @ V
        A = Pz @ np.abs(V)
        qk = float((np.abs(Q[rows]) @ np.abs(K).T).max())
        rel = U_OUT["float16"] + EPS32 * (2 * MMA_C * hs * scale * qk + 16 * scale * qk + MMA_C * 64 * nb + 16 * nb + 66)
        bound = U_OUT["float16"] * np.abs(o) + rel * A + SUBNORMAL_FLOOR["float16"] * (64 * nb * np.abs(V).max() / kp + 1)
        assert_within(y[b, rows], o, bound, "o past 2^32, batch %d" % b)
        dP = np.where(Z, dY[rows] @ V.T, 0.0) / kp
        dS = scale * P * (dP - (dP * P).sum(axis=1, keepdims=True))
        ref = dS @ K
        err = np.linalg.norm(dq[b, rows].double().cpu().numpy() - ref) / np.linalg.norm(ref)
        assert err < 1e-2, (b, err)
