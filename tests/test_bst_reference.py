"""The float64 BST reference (tests/_util.py bst_dense) and the covering set of the wgmma attention-GEMM test, on the CPU.

bst_dense is what the GPU tests hold the NT / NN / TN kernels to, so it is pinned here against the per-block loops of
TransformerOracle and against the reference's own outputs stored in tests/golden/bst_*.npz. Both of those are float32,
so they may differ from float64 by one accumulation error: fma_gemm_bound with head_state terms for NT and bs x the LUT
row length for NN / TN, the same count the kernels are held to (float32 products of float32 operands round once more
than 16-bit ones, which the bound's 2 eps32 per term covers)."""
import os

import numpy as np
import pytest

from tests._util import GOLDEN, assert_within, bst_dense, bst_terms, fma_gemm_bound, golden_files
from oracle.bst_oracle import TransformerOracle


def _per_head_holes(rng):
    """3 per-head layouts over 5 x 7 blocks with equal block counts; query block 2 and key block 3 are empty in every
    head"""
    lay = np.zeros((3, 5, 7), np.int32)
    cells = [(q, k) for q in range(5) for k in range(7) if q != 2 and k != 3]
    for h in range(3):
        for i in rng.permutation(len(cells))[:13]:
            lay[(h,) + cells[i]] = 1
    return lay


def _fixtures():
    for fname in golden_files("bst_"):
        g = np.load(os.path.join(GOLDEN, fname))
        yield fname, g["layout"], int(g["bs"]), int(g["heads"]), {k: g[k] for k in ("Q", "K", "V", "DY", "S", "P", "Y", "DV", "DP")}


def _pinned(orc, op, a, b, oracle_out, what, hs):
    ref, ref_abs = bst_dense(orc, op, a, b, with_abs=True)
    assert ref.shape == oracle_out.shape, (what, ref.shape, oracle_out.shape)
    # |a| x |b| really is the product of the absolute values: bounds every |ref| and equals it on non-negative operands
    assert np.all(ref_abs >= np.abs(ref))
    np.testing.assert_array_equal(bst_dense(orc, op, np.abs(a), np.abs(b)), ref_abs)
    k = bst_terms(orc, op, hs)
    assert_within(oracle_out, ref, fma_gemm_bound(ref, ref_abs, "float32", k), what)
    return ref


@pytest.mark.parametrize("fname", golden_files("bst_") + ["perhead-holes"])
def test_bst_dense_matches_the_oracle(fname):
    """bst_dense agrees with TransformerOracle.nt / nn / tn and with the reference's stored S, DP, Y and DV, and an
    output block with an empty LUT row is exactly zero."""
    if fname == "perhead-holes":
        rng = np.random.default_rng(5)
        lay, bs, heads, hs, batch = _per_head_holes(rng), 16, 3, 24, 2
        orc = TransformerOracle(lay, bs, heads=heads)
        S = heads * hs
        g = {"Q": rng.normal(size=(batch, 5 * bs, S)), "K": rng.normal(size=(batch, 7 * bs, S)),
             "V": rng.normal(size=(batch, 7 * bs, S)), "DY": rng.normal(size=(batch, 5 * bs, S)),
             "P": rng.uniform(-1, 1, (batch, heads, orc.blocks, bs, bs))}
        g = {k: v.astype(np.float32) for k, v in g.items()}
        assert [len(r) for r in orc.nn_list[0]][2] == 0 and [len(r) for r in orc.tn_list[1]][3] == 0
    else:
        g = dict(np.load(os.path.join(GOLDEN, fname)))
        bs, heads = int(g["bs"]), int(g["heads"])
        orc = TransformerOracle(g["layout"], bs, heads=heads)
        hs = g["Q"].shape[2] // heads
    Q, K, V, DY, P = g["Q"], g["K"], g["V"], g["DY"], g["P"]
    outs = [("nt", Q, K, orc.nt(Q, K), "nt(q, k)"), ("nt", DY, V, orc.nt(DY, V), "nt(dy, v)"),
            ("nn", P, V, orc.nn(P, V), "nn(p, v)"), ("tn", P, DY, orc.tn(P, DY), "tn(p, dy)")]
    if "S" in g:                                       # the reference's own float32 outputs on the same operands
        outs += [("nt", Q, K, g["S"], "stored S"), ("nt", DY, V, g["DP"], "stored DP"),
                 ("nn", P, V, g["Y"], "stored Y"), ("tn", P, DY, g["DV"], "stored DV")]
    for op, a, b, oracle_out, what in outs:
        ref = _pinned(orc, op, a, b, oracle_out, "%s %s" % (fname, what), hs)
        if op != "nt":
            rows = orc.nn_list if op == "nn" else orc.tn_list
            for h in range(heads):
                for o, row in enumerate(rows[orc._hl(h)]):
                    if not row:
                        blk = ref[:, o * bs:(o + 1) * bs, h * hs:(h + 1) * hs]
                        assert np.all(blk == 0), "%s %s: empty output block %d of head %d is not zero" % (fname, what, o, h)


def test_bst_dense_reads_the_lut_of_each_head():
    """A product that used head 0's layout for every head, or mixed up batch and head offsets, would differ."""
    rng = np.random.default_rng(9)
    lay = _per_head_holes(rng)
    orc = TransformerOracle(lay, 16, heads=3)
    Q, K = rng.normal(size=(3, 80, 24)), rng.normal(size=(3, 112, 24))
    ref = bst_dense(orc, "nt", Q, K)
    for n in range(3):
        for h in range(3):
            for b, (q, k) in enumerate(orc.nt_list[h]):
                want = Q[n, q * 16:(q + 1) * 16, h * 8:(h + 1) * 8] @ K[n, k * 16:(k + 1) * 16, h * 8:(h + 1) * 8].T
                np.testing.assert_allclose(ref[n, h, b], want, rtol=1e-12, atol=1e-12)


# ---- the covering set of tests/test_tc_gpu.py::test_tc_bst_gemms_match_oracle ---------------------------------------
def test_bst_cases_cover_the_envelope():
    """BST_CASES reaches every shape and instantiation the wgmma attention GEMMs have to be checked at (pure Python:
    guards later edits of the case list)."""
    import torch
    from tests.test_tc_gpu import BST_CASES, BST_DTYPES, BST_NT_OUT, bst_case_layout
    nn_rows, tn_rows = set(), set()
    for case in BST_CASES:
        lh, heads, qb, kb, density, hs, batch, holes, *opt = case
        lay, _ = bst_case_layout(case)
        orc = TransformerOracle(lay if lh > 1 else lay[0], 64, heads=heads)
        nn_rows |= {len(r) for h in range(orc.lut_heads) for r in orc.nn_list[h]}
        tn_rows |= {len(r) for h in range(orc.lut_heads) for r in orc.tn_list[h]}
    for name, rows in (("nn", nn_rows), ("tn", tn_rows)):
        # 1 entry; 4 and 5 bracket the first refill of the 4-stage ring; 9+ wraps it twice, 20+ many times
        assert {1, 4, 5} <= rows, (name, sorted(rows))
        assert max(rows) >= 20 and any(9 <= r < 20 for r in rows), (name, sorted(rows))
    assert any(c[2] == c[3] == 24 and c[4] == 1.0 for c in BST_CASES)                 # dense 24 x 24
    # batch >= 3, ctx_q != ctx_k, a layout per head: a mixed-up batch / head / a / b offset cannot cancel
    assert any(c[6] >= 3 and c[2] != c[3] and c[0] == c[1] > 1 for c in BST_CASES)
    assert any(c[5] == 128 and c[0] > 1 and c[7] is not None for c in BST_CASES)      # hs 128, per head, holes
    assert {c[5] for c in BST_CASES if "pos" in c[8:]} == {64, 128}
    assert {c[5] for c in BST_CASES} == {64, 128}
    # all ten wgmma instantiations: NT for 2 input x 3 output dtypes, NN and TN for 2 dtypes
    assert set(BST_DTYPES) == {torch.float16, torch.bfloat16}
    assert {c for c, _ in BST_NT_OUT} == {torch.float32, torch.bfloat16, torch.float16}
