"""oracle_attention (tests/_attention_oracle.py), the float64 statement of the fused attention op, equals the
oracle's own three-op chain nn(masked_softmax(nt(Q, K), scale[, autoregress_at_key]), V). Those three methods are pinned
by the reference fixtures (tests/test_oracle_golden.py), so this pins it to the reference's semantics, edge cases included:
an empty query row gives 0, a row whose keys are all masked gets uniform weights over its blocks' keys."""
import os

import numpy as np
import pytest

from tests._util import GOLDEN, golden_files
from oracle.bst_oracle import TransformerOracle
from tests._attention_oracle import oracle_attention
from tests.golden.make_golden import causal_callback, checker_callback


def _chain(orc, Q, K, V, scale, ak=None):
    return orc.nn(orc.masked_softmax(orc.nt(Q, K), scale=scale, autoregress_at_key=ak), V)


def _close(got, ref):
    # the chain runs in float32 (nt, softmax and nn each round), the new method in float64
    np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("fname", golden_files("bst_"))
def test_attention_matches_the_chain_on_reference_fixtures(fname):
    g = np.load(os.path.join(GOLDEN, fname))
    has_mask = bool(g["has_mask"])
    cb = (checker_callback if "perhead" in fname else causal_callback) if has_mask else None
    orc = TransformerOracle(g["layout"], int(g["bs"]), heads=int(g["heads"]), mask_callback=cb)
    Q, K, V, scale = g["Q"], g["K"], g["V"], float(g["scale"])
    _close(oracle_attention(orc, Q, K, V, scale), _chain(orc, Q, K, V, scale))
    _close(oracle_attention(orc, Q, K, V, scale), g["Y"])
    if has_mask:
        ak = int(g["autoregress_at_key"])
        _close(oracle_attention(orc, Q, K, V, scale, autoregress_at_key=ak), _chain(orc, Q, K, V, scale, ak))


def _hide_row_cb(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
    """causal inside diagonal blocks; row 3 of query block 1 sees no key at all"""
    m = causal_callback(blk_shape, head_idx, qry_idx, key_idx, blk_idx)
    if qry_idx == 1:
        m[3, :] = False
    return m


@pytest.mark.parametrize("ak", [None, 0, 20])
def test_attention_edge_cases_match_the_chain(ak):
    """Query block 2 holds no key block; row 3 of query block 1 is fully masked; per-head layouts, 5 x 6 blocks.
    With autoregress_at_key = 0 the rows of query block 0, which sees only key block 1, are hidden as well."""
    bs, heads = 16, 2
    lay = np.tril(np.ones((5, 6), np.int32))
    lay[0, 0], lay[0, 1] = 0, 1
    lay[2] = 0
    lay = np.stack([lay, np.roll(lay, 1, axis=1)])
    orc = TransformerOracle(lay, bs, heads=heads, mask_callback=_hide_row_cb)
    assert not orc.nn_list[0][2] and not orc.nn_list[1][2]
    rng = np.random.default_rng(7)
    Q = rng.normal(0, 1, (2, 5 * bs, heads * 8)).astype(np.float32)
    K, V = (rng.normal(0, 1, (2, 6 * bs, heads * 8)).astype(np.float32) for _ in range(2))
    got = oracle_attention(orc, Q, K, V, 0.5, autoregress_at_key=ak)
    _close(got, _chain(orc, Q, K, V, 0.5, ak))
    assert np.all(got[:, 2 * bs:3 * bs] == 0)
    # the hidden row: uniform weights over every key of its blocks (head 0: key blocks 0 and 1)
    Vh = V.reshape(2, 6 * bs, heads, 8)[:, :2 * bs, 0].astype(np.float64)
    if ak is None:
        np.testing.assert_allclose(got.reshape(2, 5 * bs, heads, 8)[:, bs + 3, 0], Vh.mean(axis=1), rtol=1e-12, atol=1e-12)
