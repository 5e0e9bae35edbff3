"""Pins the float64 oracle of the dense softmax / top-k ops (oracle/dense_oracle.py) and the NumPy checkers of
blocksparse_b200.checkers to the reference's own checkers (tests/golden/dense_*.npz, made by
tests/golden/make_golden_dense.py), and checks the recorded differences from the reference on cases of their own: a
(D1, 1, D3) mask, fully masked rows, ties."""
import os

import numpy as np
import pytest

from tests._util import GOLDEN, golden_files
from blocksparse_b200 import checkers
from oracle import dense_oracle as orc

FILES = golden_files("dense_")


def test_fixtures_cover_ranks_masks_and_k():
    assert len(FILES) >= 10
    ranks, masks = set(), set()
    for f in FILES:
        g = np.load(os.path.join(GOLDEN, f))
        ranks.add(g["x"].ndim)
        if "mask" in g.files:
            masks.add(sum(d > 1 for d in g["mask"].shape[:-1]))
        D3 = g["x"].shape[-1]
        assert g["ks"][0] == 1 and g["ks"][-1] == D3 and 1 < g["ks"][1] < D3
    assert ranks == {2, 3, 4} and masks == {0, 1, 2}


@pytest.mark.parametrize("fname", FILES)
def test_oracle_and_checkers_match_reference(fname):
    g = np.load(os.path.join(GOLDEN, fname))
    x, scale = g["x"], float(g["scale"])
    mask = g["mask"] if "mask" in g.files else None
    np.testing.assert_allclose(orc.masked_softmax(x, mask, scale), g["P"], rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(checkers.masked_softmax_test(x, mask, scale), g["P"], rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(orc.masked_softmax_grad(g["DY"], g["P"], mask, scale), g["DX"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(checkers.masked_softmax_grad_test(g["DY"], g["P"], mask, scale), g["DX"], rtol=1e-5, atol=1e-6)
    for k, tk in zip(g["ks"], g["TK"]):
        np.testing.assert_allclose(orc.masked_top_k_softmax(x, int(k), mask, scale), tk, rtol=2e-6, atol=1e-7)
        np.testing.assert_allclose(checkers.masked_top_k_softmax_test(x, int(k), mask, scale), tk, rtol=2e-6, atol=1e-7)
        assert np.array_equal(orc.masked_top_k_softmax(x, int(k), mask, scale) != 0, tk != 0)
    if "R_rebase" in g.files:
        for k, rr, rp in zip(g["ks"], g["R_rebase"], g["R_plain"]):
            np.testing.assert_allclose(orc.rectified_top_k(x, int(k), True), rr, rtol=1e-6, atol=1e-6)
            np.testing.assert_allclose(orc.rectified_top_k(x, int(k), False), rp, rtol=1e-6, atol=1e-6)
            np.testing.assert_array_equal(checkers.rectified_top_k_test(x, int(k), True), rr)
            np.testing.assert_array_equal(checkers.rectified_top_k_test(x, int(k), False), rp)
            # top_k picks the entries the reference's rectified_top_k keeps: without rebase they are relu(x) there
            vals, idx = orc.top_k(x, int(k))
            assert np.array_equal(np.take_along_axis(x, idx.astype(np.int64), -1), vals)
            assert np.all(vals[..., :-1] >= vals[..., 1:])
            support = np.zeros(x.shape, bool)
            np.put_along_axis(support, idx.astype(np.int64), True, axis=-1)
            np.testing.assert_array_equal(rp, np.where(support, np.maximum(x, 0), 0))


def test_mask_with_broadcast_dim2_applies_to_its_own_rows():
    """mask (D1, 1, D3): row (d0, d1, d2) uses mask row d1 for every d2. The reference's kernel strides dim 1 by D2 * D3
    (transformer_op.cc:184-185) and its checker flattens the mask (transformer.py:613); neither gives this."""
    rng = np.random.default_rng(1)
    x = rng.normal(0, 1, (2, 3, 4, 8))
    mask = (rng.random((1, 3, 1, 8)) < 0.6).astype(np.float32) * 2.0
    mask[..., 1] = 1.0
    y = orc.masked_softmax(x, mask, 0.5)
    for d1 in range(3):
        for d2 in range(4):
            m = mask[0, d1, 0]
            v = np.where(m != 0, x[:, d1, d2] * m * 0.5, -orc.FLT_MAX)
            e = np.exp(v - v.max(-1, keepdims=True))
            np.testing.assert_allclose(y[:, d1, d2], e / e.sum(-1, keepdims=True), rtol=1e-12)
    np.testing.assert_allclose(checkers.masked_softmax_test(x, mask, 0.5), y, rtol=1e-5, atol=1e-7)


def test_fully_masked_rows():
    """Every entry of a fully masked row is 1 / D3 (the reference kernel's padding lanes make its rows sum below 1), and
    masked_top_k_softmax gives 1 / k on the first k columns of such a row."""
    x = np.arange(24, dtype=np.float64).reshape(2, 12)
    mask = np.ones((2, 12))
    mask[1] = 0
    y = orc.masked_softmax(x, mask)
    np.testing.assert_array_equal(y[1], np.full(12, 1 / 12))
    z = orc.masked_top_k_softmax(x, 5, mask)
    np.testing.assert_array_equal(z[1], np.r_[np.full(5, 0.2), np.zeros(7)])
    # fewer visible entries than k: the remaining slots go to the lowest-index masked columns, with probability 0
    mask[0, :] = 0
    mask[0, [3, 9]] = 1
    z = orc.masked_top_k_softmax(x, 4, mask)
    assert set(np.nonzero(z[0])[0]) == {3, 9}
    assert np.isclose(z[0].sum(), 1.0)


def test_ties_rank_by_index():
    x = np.array([[1, 3, 3, 2, 3, 1, 0, 3]], dtype=np.float32)
    vals, idx = orc.top_k(x, 5)
    np.testing.assert_array_equal(idx, [[1, 2, 4, 7, 3]])
    np.testing.assert_array_equal(vals, [[3, 3, 3, 3, 2]])
    z = orc.masked_top_k_softmax(x, 3)
    np.testing.assert_array_equal(np.nonzero(z[0])[0], [1, 2, 4])
    np.testing.assert_array_equal(checkers.masked_top_k_softmax_test(x, 3) != 0, z != 0)
    r = orc.rectified_top_k(x, 3, rebase=True)            # base = 3: every top-k entry becomes 0
    np.testing.assert_array_equal(r, np.zeros_like(r))
    r = orc.rectified_top_k(x, 6, rebase=False)           # relu of the top 6: columns 1, 2, 4, 7, 3 and 0
    np.testing.assert_array_equal(r[0], [1, 3, 3, 2, 3, 0, 0, 3])
    np.testing.assert_array_equal(checkers.rectified_top_k_test(x, 6, rebase=False), r)
