"""oracle_attention_grad (tests/_attention_grad_oracle.py), the float64 statement of the fused attention backward, equals
the oracle's own chain backward: dV = tn(P, dY), dS = masked_softmax_grad(nt(dY, V), P, scale), dQ = nn(dS, K),
dK = tn(dS, Q) with P = masked_softmax(nt(Q, K), scale[, autoregress_at_key]). Those methods are pinned by the
reference fixtures (tests/test_oracle_golden.py), so this pins the gradients to the reference's semantics, edge cases
included. A central-difference check ties them to the forward oracle_attention as well."""
import os

import numpy as np
import pytest

from tests._util import GOLDEN, golden_files
from oracle.bst_oracle import TransformerOracle
from tests._attention_oracle import oracle_attention
from tests._attention_grad_oracle import oracle_attention_grad
from tests.golden.make_golden import causal_callback, checker_callback


def _chain_grad(orc, Q, K, V, dY, scale, ak=None):
    P = orc.masked_softmax(orc.nt(Q, K), scale=scale, autoregress_at_key=ak)
    dS = orc.masked_softmax_grad(orc.nt(dY, V), P, scale=scale)
    return orc.nn(dS, K), orc.tn(dS, Q), orc.tn(P, dY)


def _close(got, ref):
    # the chain runs in float32 (each op rounds, and dS cancels in dP - D), the new method in float64
    for g, r, name in zip(got, ref, ("dQ", "dK", "dV")):
        np.testing.assert_allclose(g, r, rtol=1e-4, atol=1e-5 * float(np.abs(r).max()) + 1e-7, err_msg=name)


@pytest.mark.parametrize("fname", golden_files("bst_"))
def test_grad_matches_the_chain_on_reference_fixtures(fname):
    g = np.load(os.path.join(GOLDEN, fname))
    has_mask = bool(g["has_mask"])
    cb = (checker_callback if "perhead" in fname else causal_callback) if has_mask else None
    orc = TransformerOracle(g["layout"], int(g["bs"]), heads=int(g["heads"]), mask_callback=cb)
    Q, K, V, scale = g["Q"], g["K"], g["V"], float(g["scale"])
    dY = np.random.default_rng(11).normal(0, 1, g["Y"].shape).astype(np.float32)
    _close(oracle_attention_grad(orc, Q, K, V, dY, scale), _chain_grad(orc, Q, K, V, dY, scale))
    if has_mask:
        ak = int(g["autoregress_at_key"])
        _close(oracle_attention_grad(orc, Q, K, V, dY, scale, ak), _chain_grad(orc, Q, K, V, dY, scale, ak))


def _hide_row_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    """causal inside diagonal blocks; row 3 of query block 1 sees no key at all"""
    m = causal_callback(blk_shape, head_idx, qry_idx, key_idx, blk_idx)
    if qry_idx == 1:
        m[3, :] = False
    return m


@pytest.mark.parametrize("ak", [None, 0, 20])
def test_grad_edge_cases_match_the_chain(ak):
    """Per-head layouts of 5 x 6 blocks. Query block 2 holds no key block; key block 5 (head 0) and key block 0 (head 1)
    are seen by no query block; row 3 of query block 1 is fully masked. With autoregress_at_key = 0 the rows of query
    block 0, which sees only key block 1, are hidden as well."""
    bs, heads = 16, 2
    lay = np.tril(np.ones((5, 6), np.int32))
    lay[0, 0], lay[0, 1] = 0, 1
    lay[2] = 0
    lay = np.stack([lay, np.roll(lay, 1, axis=1)])
    orc = TransformerOracle(lay, bs, heads=heads, mask_callback=_hide_row_cb)
    assert not orc.nn_list[0][2] and not orc.tn_list[0][5] and not orc.tn_list[1][0]
    rng = np.random.default_rng(7)
    Q, dY = (rng.normal(0, 1, (2, 5 * bs, heads * 8)).astype(np.float32) for _ in range(2))
    K, V = (rng.normal(0, 1, (2, 6 * bs, heads * 8)).astype(np.float32) for _ in range(2))
    got = oracle_attention_grad(orc, Q, K, V, dY, 0.5, ak)
    _close(got, _chain_grad(orc, Q, K, V, dY, 0.5, ak))
    dQ, dK, dV = (x.reshape(2, -1, heads, 8) for x in got)
    assert np.all(dQ[:, 2 * bs:3 * bs] == 0)
    for h, kb in ((0, 5), (1, 0)):
        assert np.all(dK[:, kb * bs:(kb + 1) * bs, h] == 0) and np.all(dV[:, kb * bs:(kb + 1) * bs, h] == 0)
    # the fully masked row still sends its dS into dQ (uniform P over the keys of its blocks)
    if ak is None:
        assert np.abs(dQ[:, bs + 3, 0]).max() > 0


def test_grad_matches_central_differences():
    """d(sum dY * O)/dX by central differences of oracle_attention, for every element of Q, K and V: a causal mask
    with per-head layouts and no fully masked row (there O does not depend on Q and K, while the chain's gradient is
    not zero)."""
    bs, heads, hs = 8, 2, 4
    lay = np.stack([np.tril(np.ones((3, 3), np.int32)), np.array([[1, 0, 1], [1, 1, 0], [0, 1, 1]], np.int32)])
    orc = TransformerOracle(lay, bs, heads=heads, mask_callback=causal_callback)
    rng = np.random.default_rng(3)
    Q, K, V, dY = (rng.normal(0, 1, (1, 3 * bs, heads * hs)) for _ in range(4))
    scale, step = 0.7, 1e-6
    grads = oracle_attention_grad(orc, Q, K, V, dY, scale)
    args = [Q, K, V]
    for i, g in enumerate(grads):
        num = np.empty_like(args[i])
        for idx in np.ndindex(*args[i].shape):
            x0 = args[i][idx]
            vals = []
            for d in (step, -step):
                args[i][idx] = x0 + d
                vals.append(float((dY * oracle_attention(orc, *args, scale)).sum()))
            args[i][idx] = x0
            num[idx] = (vals[0] - vals[1]) / (2 * step)
        np.testing.assert_allclose(g, num, rtol=1e-6, atol=1e-7, err_msg="dQdKdV"[2 * i:2 * i + 2])
