"""The float64 statement of attention with dropout (tests/_attention_dropout_oracle.py): with keep_prob = 1 it is the
existing attention oracles exactly; with keep_prob < 1 it equals the float64 chain nt -> masked_softmax ->
ewops_oracle.dropout_apply -> nn, forward and gradients; its gradients match central differences at a fixed mask; and
its keep bits are those ewops_oracle.dropout_bits draws for the chain's (batch, heads, blocks, bs, bs) probabilities."""
import numpy as np
import pytest

from oracle.bst_oracle import TransformerOracle
from oracle.ewops_oracle import dropout_apply, dropout_bits, dropout_mask, philox4x32_10
from tests._attention_dropout_oracle import (attention_keep, keep_bits_at, oracle_attention_dropout,
                                             oracle_attention_dropout_grad)
from tests._attention_grad_oracle import oracle_attention_grad
from tests._attention_oracle import oracle_attention
from tests.golden.make_golden import causal_callback


def _hide_row_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    """causal inside diagonal blocks; row 3 of query block 1 sees no key at all"""
    m = causal_callback(blk_shape, head_idx, qry_idx, key_idx, blk_idx)
    if qry_idx == 1:
        m[3, :] = False
    return m


def _edge_layout():
    """per-head 5 x 6 layouts: query block 2 holds no key block, query block 0 sees only key block 1"""
    lay = np.tril(np.ones((5, 6), np.int32))
    lay[0, 0], lay[0, 1] = 0, 1
    lay[2] = 0
    return np.stack([lay, np.roll(lay, 1, axis=1)])


def _inputs(orc, batch, hs, seed):
    rng = np.random.default_rng(seed)
    bs, H = orc.blk_size, orc.heads
    Q, dY = (rng.normal(0, 1, (batch, orc.ctx_blks_q * bs, H * hs)) for _ in range(2))
    K, V = (rng.normal(0, 1, (batch, orc.ctx_blks_k * bs, H * hs)) for _ in range(2))
    return Q, K, V, dY


@pytest.mark.parametrize("ak", [None, 0, 20])
def test_keep_prob_one_is_the_attention_oracles(ak):
    orc = TransformerOracle(_edge_layout(), 16, heads=2, mask_callback=_hide_row_cb)
    Q, K, V, dY = _inputs(orc, 2, 8, 1)
    Z = np.ones((2, 2, orc.ctx_blks_q * 16, orc.ctx_blks_k * 16), bool)
    assert np.array_equal(oracle_attention_dropout(orc, Q, K, V, Z, 1.0, 0.5, ak), oracle_attention(orc, Q, K, V, 0.5, ak))
    for got, ref in zip(oracle_attention_dropout_grad(orc, Q, K, V, dY, Z, 1.0, 0.5, ak),
                        oracle_attention_grad(orc, Q, K, V, dY, 0.5, ak)):
        assert np.array_equal(got, ref)


def _chain(orc, Q, K, V, dY, scale, ak, words, kp):
    """the float64 chain and its backward, with the dropout of the (batch, heads, blocks, bs, bs) probabilities"""
    P = orc.masked_softmax(orc.nt(Q, K), scale=scale, autoregress_at_key=ak)
    Pd = dropout_apply(P, words, kp)
    O = orc.nn(Pd, V)
    dP = dropout_apply(orc.nt(dY, V), words, kp)
    dS = orc.masked_softmax_grad(dP, P, scale=scale)
    return O, (orc.nn(dS, K), orc.tn(dS, Q), orc.tn(Pd, dY))


@pytest.mark.parametrize("kp", [0.9, 0.5])
@pytest.mark.parametrize("shared", [True, False], ids=["lut_heads1", "per_head"])
@pytest.mark.parametrize("ak", [None, 20])
def test_matches_the_chain_with_dropout(ak, shared, kp):
    lay = _edge_layout()
    orc = TransformerOracle(lay[0] if shared else lay, 16, heads=2, mask_callback=_hide_row_cb)
    batch, seed, call = 2, 0x1234_5678_9ABC_DEF0 - 2 ** 63, 77
    Q, K, V, dY = _inputs(orc, batch, 8, 2)
    M = batch * orc.heads * orc.blocks * 16 * 16
    words = dropout_mask(seed, call, M, kp)
    O, grads = _chain(orc, Q, K, V, dY, 0.5, ak, words, kp)
    Z = attention_keep(orc, batch, seed, call, kp)
    assert 0 < Z.sum() < sum(len(r) for r in orc.nt_list) * 256 * batch * (orc.heads if shared else 1)
    # the oracle's chain ops run in float32 (each rounds, and dS cancels in dP - D)
    for got, ref, name in zip((oracle_attention_dropout(orc, Q, K, V, Z, kp, 0.5, ak),)
                              + oracle_attention_dropout_grad(orc, Q, K, V, dY, Z, kp, 0.5, ak), (O,) + grads,
                              ("O", "dQ", "dK", "dV")):
        np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-5 * float(np.abs(ref).max()) + 1e-7, err_msg=name)


def test_grad_matches_central_differences_at_a_fixed_mask():
    bs, heads, hs = 8, 2, 4
    lay = np.stack([np.tril(np.ones((3, 3), np.int32)), np.array([[1, 0, 1], [1, 1, 0], [0, 1, 1]], np.int32)])
    orc = TransformerOracle(lay, bs, heads=heads, mask_callback=causal_callback)
    Q, K, V, dY = _inputs(orc, 1, hs, 3)
    kp, scale, step = 0.7, 0.7, 1e-6
    Z = attention_keep(orc, 1, 5, 9, kp)
    assert not Z.all() and Z.any()
    grads = oracle_attention_dropout_grad(orc, Q, K, V, dY, Z, kp, scale)
    args = [Q, K, V]
    for i, g in enumerate(grads):
        num = np.empty_like(args[i])
        for idx in np.ndindex(*args[i].shape):
            x0 = args[i][idx]
            vals = []
            for d in (step, -step):
                args[i][idx] = x0 + d
                vals.append(float((dY * oracle_attention_dropout(orc, *args, Z, kp, scale)).sum()))
            args[i][idx] = x0
            num[idx] = (vals[0] - vals[1]) / (2 * step)
        np.testing.assert_allclose(g, num, rtol=1e-6, atol=1e-7, err_msg="dQdKdV"[2 * i:2 * i + 2])


@pytest.mark.parametrize("shared", [True, False], ids=["lut_heads1", "per_head"])
def test_index_formula_matches_dropout_bits(shared):
    """Z scattered from dropout_bits of the whole (batch, heads, blocks, 64, 64) tensor, block b of head h at its
    (query block, key block) of the layout, equals attention_keep, which evaluates e per element."""
    lay = _edge_layout()
    heads, batch, bs, kp, seed, call = 3, 2, 64, 0.6, -5, 2 ** 33 + 7
    lay3 = np.stack([lay[0], lay[1], lay[0]]) if not shared else lay[0]
    orc = TransformerOracle(lay3, bs, heads=heads)
    bits = dropout_bits(seed, call, batch * heads * orc.blocks * bs * bs, kp).reshape(batch, heads, orc.blocks, bs, bs)
    ref = np.zeros((batch, heads, orc.ctx_blks_q * bs, orc.ctx_blks_k * bs), bool)
    for h in range(heads):
        for b, (q, k) in enumerate(orc.nt_list[orc._hl(h)]):
            ref[:, h, q * bs:(q + 1) * bs, k * bs:(k + 1) * bs] = bits[:, h, b]
    assert np.array_equal(attention_keep(orc, batch, seed, call, kp), ref)
    rows = np.array([0, 63, 64, 200, 319])
    assert np.array_equal(attention_keep(orc, batch, seed, call, kp, batches=[1], rows=rows), ref[1:, :, rows])


def test_keep_bits_past_2_32():
    """keep_bits_at is dropout_bits' draw near 0, and past 2^32 puts e / 4 into both words of the counter."""
    e = np.arange(4096, dtype=np.int64)
    assert np.array_equal(keep_bits_at(3, 4, e, 0.5), dropout_bits(3, 4, 4096, 0.5))
    for x in ((1 << 34) + 4 * 3 + 1, (1 << 35) + 4 * 7 + 3):
        g, w = x // 4, x % 4
        words = philox4x32_10(np.array([g & 0xFFFFFFFF, g >> 32, 4, 0], np.uint32), np.array([3, 0], np.uint32))
        assert bool(keep_bits_at(3, 4, np.array([x]), 0.5)[0]) == (int(words[w]) < 2 ** 31)
