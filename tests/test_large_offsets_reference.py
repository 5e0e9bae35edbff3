"""The sampled float64 references of tests/test_large_offsets_gpu.py, run over every row of small problems on the CPU:
put together, the sub-problems have to give what the full oracles give (oracle/bst_oracle.py, oracle/bsmm_oracle.py,
tests/_xent_oracle.py, oracle/optimize_oracle.py). The checks are the GPU file's own, fed the full oracle's fp32 result
where the kernel's output goes, so they are rehearsed here as well."""
import numpy as np
import torch

from tests import _xent_oracle as xo
from tests._attention_oracle import oracle_attention
from tests._util import oracle_dense
from tests.golden.make_golden import causal_callback
from tests.test_large_offsets_gpu import (TWO31, adam_window_check, band_layout, causal, check_nt, check_softmax,
                                          check_softmax_grad, check_xn, dense_blocks, ema_window_check,
                                          minibatch_crossing, sample_ids, sample_rows, sub_problem, take, tril_layout,
                                          updat_dense64, windows)
from blocksparse_b200.layouts import bernoulli_layout
from oracle import optimize_oracle as oo
from oracle.bsmm_oracle import MatmulOracle
from oracle.bst_oracle import TransformerOracle


def test_causal_is_causal_callback():
    for q, k in ((3, 3), (3, 1)):
        assert np.array_equal(causal((16, 16), 0, q, k, 5), causal_callback((16, 16), 0, q, k, 5))


def test_attention_sub_problems_reassemble_the_full_oracle():
    bs, heads, batch, hs, scale = 16, 2, 2, 16, 0.25
    for lay in (tril_layout(5), band_layout(7, 3)):
        orc = TransformerOracle(lay, bs, heads=heads, mask_callback=causal)
        rng = np.random.default_rng(len(lay))
        n = lay.shape[0]
        q, k, v, dy = (rng.normal(0, 1, (batch, n * bs, heads * hs)).astype(np.float32) for _ in range(4))
        rows = [(z, r) for z in range(batch * heads) for r in range(n)]
        T = torch.as_tensor
        scores = orc.nt(q, k)
        check_nt(orc, causal, rows, heads, hs, T(q), T(k), T(scores), "fma_dds_nt", "nt")
        p = orc.masked_softmax(scores, scale=scale)
        check_softmax(orc, causal, rows, heads, T(scores), T(p), scale, float(np.abs(scores).max() * scale), "softmax")
        check_xn(orc, causal, rows, heads, hs, T(p), T(v), T(orc.nn(p, v)), False, "fma_sdd_xn", "nn")
        check_xn(orc, causal, rows, heads, hs, T(p), T(dy), T(orc.tn(p, dy)), True, "fma_sdd_xn", "tn")
        dP = orc.nt(dy, v)
        dS = orc.masked_softmax_grad(dP, p, scale=scale)
        check_softmax_grad(orc, causal, rows, heads, T(dP), T(p), T(dS), scale, "softmax grad")
        # the fused op: a query row's sub-problem gives that row of the whole attention
        full = oracle_attention(orc, q.astype(np.float64), k.astype(np.float64), v.astype(np.float64), scale)
        for z, r in rows:
            b, h = z // heads, z % heads
            so, _, kbs = sub_problem(orc, causal, bs, h, r)
            ref = oracle_attention(so, dense_blocks(T(q), b, h, [r], bs, hs), dense_blocks(T(k), b, h, kbs, bs, hs),
                                   dense_blocks(T(v), b, h, kbs, bs, hs), scale)
            assert np.allclose(ref[0], full[b, r * bs:(r + 1) * bs, h * hs:(h + 1) * hs], rtol=1e-12, atol=1e-14)


def test_a_wrong_row_is_out_of_bound():
    """The checks bite: the full oracle's scores with two blocks swapped fail them."""
    bs, heads, hs = 16, 1, 16
    orc = TransformerOracle(tril_layout(4), bs, heads=heads, mask_callback=causal)
    rng = np.random.default_rng(3)
    q, k = (torch.as_tensor(rng.normal(0, 1, (1, 4 * bs, hs)).astype(np.float32)) for _ in range(2))
    scores = torch.as_tensor(orc.nt(q.numpy(), k.numpy()))
    scores[0, 0, [8, 9]] = scores[0, 0, [9, 8]]
    try:
        check_nt(orc, causal, [(0, 3)], heads, hs, q, k, scores, "fma_dds_nt", "nt")
    except AssertionError:
        return
    raise AssertionError("swapped blocks passed")


def test_sampling_reaches_both_sides_of_2_31():
    rng = np.random.default_rng(0)
    ids = sample_ids(16400, TWO31 // 131072, rng)
    assert ids[0] == 0 and ids[-1] == 16399 and {16383, 16384, 16385} <= set(ids) and ids == sorted(set(ids))
    orc = TransformerOracle(band_layout(520, 16), 64, heads=1)
    rows = sample_rows(orc, 64, 64, rng)
    first = lambda z, r: (z * orc.blocks + orc.nn_list[0][r][0][0]) * 4096
    assert any(first(z, r) < TWO31 for z, r in rows) and any(first(z, r) >= TWO31 for z, r in rows)
    assert (63, 519) in rows and orc.nn_list[0][519][-1][0] == orc.blocks - 1          # the last block of the tensor
    for a, b in windows(TWO31 + 5):
        assert 0 <= a < b <= TWO31 + 5
    assert minibatch_crossing(1, 1024, 2 ** 21 + 128) == 2 ** 21
    n = minibatch_crossing(0, 1024, 2 ** 21 + 128)
    assert 1023 * (2 ** 21 + 128) + n == TWO31


def test_bsmm_references_match_the_oracle():
    rng = np.random.default_rng(5)
    for axis in (0, 1):
        bs, nb, N = 32, 3, 70
        lay = bernoulli_layout(rng, nb, nb, 0.5)
        orc = MatmulOracle(lay, bs, axis)
        shape = (N, nb * bs) if axis else (nb * bs, N)
        X, E = (torch.as_tensor(rng.normal(0, 1, shape).astype(np.float32)) for _ in range(2))
        W = rng.normal(0, 1, (orc.blocks, bs, bs))
        every = list(range(N))
        assert np.array_equal(take(X, axis, every), X.double().numpy())
        pick = sample_ids(N, 33, rng, n_rand=5)
        full = orc.fprop(X.double().numpy(), W)
        part = orc.fprop(take(X, axis, pick), W)
        assert np.allclose(part, full[pick] if axis else full[:, pick], rtol=1e-12, atol=1e-12)
        got = updat_dense64(X, E, axis, orc.updat_lut, bs, step=16)
        assert np.allclose(got, oracle_dense(orc, "updat", X.numpy(), E.numpy()), rtol=1e-12, atol=1e-12)
        assert np.allclose(got, orc.updat_blocks(X.numpy(), E.numpy(), np.arange(orc.blocks)), rtol=1e-5, atol=1e-5)
        ab = updat_dense64(X, E, axis, orc.updat_lut, bs, absolute=True, step=16)
        assert np.allclose(ab, oracle_dense(orc, "updat", np.abs(X.numpy()), np.abs(E.numpy())), rtol=1e-12, atol=1e-12)


def test_cross_entropy_on_sampled_rows_is_the_oracle_on_those_rows():
    rng = np.random.default_rng(6)
    x, lab = rng.normal(0, 3, (40, 100)), rng.integers(0, 100, 40)
    pick = sample_ids(40, 17, rng, n_rand=5)
    loss, lse = xo.softmax_cross_entropy(x, lab)
    l2, s2 = xo.softmax_cross_entropy(x[pick], lab[pick])
    assert np.array_equal(l2, loss[pick]) and np.array_equal(s2, lse[pick])
    dy = rng.uniform(0.5, 2, 40)
    assert np.array_equal(xo.softmax_cross_entropy_grad(x[pick], lab[pick], dy[pick]), xo.softmax_cross_entropy_grad(x, lab, dy)[pick])


def test_optimizer_window_checks_accept_the_oracle():
    rng = np.random.default_rng(7)
    n = 5000
    p, g = rng.normal(0, 0.5, n).astype(np.float32).astype(np.float64), rng.normal(0, 0.1, n).astype(np.float32).astype(np.float64)
    m0, v0 = oo.mean_encode(rng.normal(0, 0.05, n)), oo.var_encode(rng.uniform(0, 0.01, n))
    kw = dict(lr=float(np.float32(0.1)), beta1=float(np.float32(0.9)), beta2=float(np.float32(0.999)), epsilon=float(np.float32(1e-8)))
    p1, m1, v1 = oo.adam(g, p, oo.mean_decode(m0), oo.var_decode(v0), **kw)
    adam_window_check(p1, p, g, m0, v0, oo.mean_encode(m1), oo.var_encode(v1), "oracle")
    try:
        adam_window_check(np.roll(p1, 1), p, g, m0, v0, oo.mean_encode(m1), oo.var_encode(v1), "shifted")
    except AssertionError:
        pass
    else:
        raise AssertionError("a shifted window passed")
    e0 = p.astype(np.float16).astype(np.float64)
    e1 = oo.ema(e0, p + 1, 0.5).astype(np.float16).astype(np.float64)
    ema_window_check(e1, e0, p + 1, 0.5, "oracle")
