"""Grouped-query attention without a GPU: the four C entries are bound, a bad kv_heads is refused with BSMM_E_ARG and
configurations outside the fused envelope with BSMM_E_NOKERNEL before anything is launched, the Python ValueErrors come
before any device is touched, and the float64 GQA reference (k and v expanded to heads heads, then the multi-head
references; dk and dv summed over each group) is scaled_dot_product_attention(enable_gqa=True)."""
import ctypes

import numpy as np
import pytest
import torch

from tests._attention_grad_oracle import oracle_attention_grad
from tests._attention_oracle import oracle_attention
from tests._gqa_oracle import expand_kv, oracle_attention_gqa, oracle_attention_gqa_grad, sum_groups
from tests.golden.make_golden import causal_callback
from blocksparse_b200 import BlocksparseTransformer, _lib
from blocksparse_b200.layouts import local_strided_layout
from oracle.bst_oracle import TransformerOracle

E_ARG, E_NOKERNEL = -3, -7
LUT, Q, K, V, O, MASK, ST = 0x1000, 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
M, L, D, DQ, DK, DV, DY, POS, WS = (0x70000 + 0x1000 * i for i in range(9))
ENTRIES = ("bst_attention_gqa", "bst_attention_train_gqa", "bst_attention_grad_gqa", "bst_attention_decode_gqa")


def test_symbols_are_bound():
    lib = _lib.load()
    for name in ENTRIES:
        assert name in _lib.SIGNATURES
        assert hasattr(ctypes.CDLL(_lib.LIB_PATH), name)
        assert getattr(lib, name).argtypes is not None


def _call(entry, dtype=_lib.BF16, bs=64, hs=64, heads=4, kv=2, q=Q, k=K, v=V, kp=1.0, n=1):
    lib = _lib.load()
    if entry == "bst_attention_gqa":
        return lib.bst_attention_gqa(dtype, bs, LUT, 1, 6, None, 1, -1, q, k, v, O, 0.125, 2, heads, kv, hs, 3, 3,
                                     kp, ST, None)
    if entry == "bst_attention_train_gqa":
        return lib.bst_attention_train_gqa(dtype, bs, LUT, 1, 6, None, 1, -1, q, k, v, O, M, L, 0.125, 2, heads, kv, hs,
                                           3, 3, kp, ST, None)
    if entry == "bst_attention_grad_gqa":
        return lib.bst_attention_grad_gqa(dtype, bs, LUT, LUT, LUT, 1, 6, None, 1, -1, q, k, v, O, DY, M, L, D, DQ, DK,
                                          DV, 0.125, 2, heads, kv, hs, 3, 3, kp, ST, None)
    return lib.bst_attention_decode_gqa(dtype, bs, LUT, 1, 6, 5, None, 1, -1, q, k, v, O, POS, n, 0.125, 2, heads, kv,
                                        hs, 3, 3, WS, None)


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("heads,kv", [(4, 0), (4, -1), (4, 5), (4, 3), (6, 4), (1, 2)])
def test_bad_kv_heads_is_refused_before_any_launch(entry, heads, kv):
    lib = _lib.load()
    before = _lib.last_kernel()
    rc = _call(entry, heads=heads, kv=kv)
    assert rc == E_ARG, (rc, lib.bsmm_last_error())
    assert b"kv_heads" in lib.bsmm_last_error(), lib.bsmm_last_error()
    assert _lib.last_kernel() == before


@pytest.mark.parametrize("entry", ENTRIES[:3])
@pytest.mark.parametrize("kp", [1.0, 0.9])
def test_outside_the_envelope_is_no_kernel_before_any_launch(entry, kp):
    before = _lib.last_kernel()
    for kw in (dict(bs=32), dict(bs=8), dict(dtype=_lib.F32), dict(dtype=-1), dict(hs=32), dict(hs=192),
               dict(q=Q + 2), dict(k=K + 8), dict(v=V + 4)):
        rc = _call(entry, kp=kp, **kw)
        assert rc == E_NOKERNEL, (entry, kw, rc, _lib.load().bsmm_last_error())
    assert _lib.last_kernel() == before


@pytest.mark.parametrize("entry", ENTRIES)
def test_counterpart_errors_keep_their_codes(entry):
    before = _lib.last_kernel()
    assert _call(entry, q=None) == E_ARG
    assert _call(entry, heads=0, kv=0) == E_ARG
    if entry == "bst_attention_decode_gqa":
        assert _call(entry, dtype=_lib.F32) == -1                # BSMM_E_DTYPE
        assert _call(entry, n=2, bs=64, hs=72) == E_ARG
    else:
        assert _call(entry, kp=0.0) == E_ARG
        assert _call(entry, bs=12) == -2                         # BSMM_E_BSIZE
    assert _lib.last_kernel() == before


# ---- Python -------------------------------------------------------------------------------------------------------
def _bst(heads=4, bs=64):
    return BlocksparseTransformer(local_strided_layout(4), bs, heads=heads, mask_callback=causal_callback)


def _qkv(heads=4, kv=2, hs=64, bs=64, batch=2, dtype=torch.float16):
    ctx = 4 * bs
    return (torch.zeros(batch, ctx, heads * hs, dtype=dtype), torch.zeros(batch, ctx, kv * hs, dtype=dtype),
            torch.zeros(batch, ctx, kv * hs, dtype=dtype))


@pytest.mark.parametrize("case,what", [
    ("zero", r"kv_heads must be an int in \[1, heads"),
    ("negative", r"kv_heads must be an int in \[1, heads"),
    ("above", r"kv_heads must be an int in \[1, heads"),
    ("float", r"kv_heads must be an int in \[1, heads"),
    ("bool", r"kv_heads must be an int in \[1, heads"),
    ("divide", "does not divide heads"),
    ("kshape", r"k and v must be \(batch, ctx_k, kv_heads\*head_state\)"),
    ("vshape", r"k and v must be \(batch, ctx_k, kv_heads\*head_state\)"),
    ("ctx", r"k and v must be \(batch, ctx_k, kv_heads\*head_state\)"),
    ("mha_shape", r"k and v must be"),
])
@pytest.mark.parametrize("op", ["attention", "attention_decode"])
def test_python_argument_errors_before_any_device(op, case, what):
    """CPU tensors: a call that got past the checks would fail on the device instead of raising ValueError."""
    bst = _bst()
    q, k, v = _qkv()
    kv = {"zero": 0, "negative": -2, "above": 8, "float": 2.0, "bool": True, "divide": 3}.get(case, 2)
    if case == "kshape":
        k = k[..., :-64]
    elif case == "vshape":
        v = torch.zeros(2, v.shape[1], 4 * 64, dtype=v.dtype)
    elif case == "ctx":
        k, v = k[:, :-1], v[:, :-1]
    elif case == "mha_shape":        # k and v of heads heads, but kv_heads = 2
        k, v = q.clone(), q.clone()
    if op == "attention":
        with pytest.raises(ValueError, match=what):
            bst.attention(q, k, v, kv_heads=kv)
        return
    pos = torch.zeros(2, dtype=torch.int32)
    what = what.replace(r"k and v must be", "caches must be")
    with pytest.raises(ValueError, match=what):
        bst.attention_decode(q[:, :1], k, v, pos, kv_heads=kv)


def test_without_kv_heads_the_shape_check_is_unchanged():
    bst = _bst()
    q, k, v = _qkv()
    with pytest.raises(ValueError, match="caches must be"):
        bst.attention_decode(q[:, :1], k, v, torch.zeros(2, dtype=torch.int32))


# ---- the float64 reference ------------------------------------------------------------------------------------------
def _sdpa(Q, K, V, dY, heads, kv, scale, causal):
    """scaled_dot_product_attention(enable_gqa=True) in float64 on the CPU: (O, dQ, dK, dV) in the op's layout."""
    def split(X, h):
        B, C, S = X.shape
        return torch.tensor(X).reshape(B, C, h, S // h).transpose(1, 2).requires_grad_()
    q, k, v = split(Q, heads), split(K, kv), split(V, kv)
    o = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=causal, scale=scale, enable_gqa=True)
    o.backward(split(dY, heads).detach())
    merge = lambda t: t.detach().transpose(1, 2).reshape(t.shape[0], t.shape[2], -1).numpy()
    return merge(o), merge(q.grad), merge(k.grad), merge(v.grad)


@pytest.mark.parametrize("heads,kv", [(4, 4), (4, 2), (4, 1), (6, 3)])
@pytest.mark.parametrize("causal", [False, True])
def test_gqa_oracle_is_sdpa_with_enable_gqa(heads, kv, causal):
    """All-ones layout (causal: its lower triangle with the mask causal inside diagonal blocks): the reference pins the
    h // g convention."""
    bs, nb, hs, batch, scale = 8, 4, 16, 2, 0.3
    lay = np.tril(np.ones((nb, nb), np.int64)) if causal else np.ones((nb, nb), np.int64)
    orc = TransformerOracle(lay, bs, heads=heads, mask_callback=causal_callback if causal else None)
    rng = np.random.default_rng(heads * 10 + kv)
    ctx = nb * bs
    Qa, dYa = (rng.normal(0, 1, (batch, ctx, heads * hs)) for _ in range(2))
    Ka, Va = (rng.normal(0, 1, (batch, ctx, kv * hs)) for _ in range(2))
    o = oracle_attention_gqa(orc, kv, Qa, Ka, Va, scale)
    dq, dk, dv = oracle_attention_gqa_grad(orc, kv, Qa, Ka, Va, dYa, scale)
    want = _sdpa(Qa, Ka, Va, dYa, heads, kv, scale, causal)
    for got, ref in zip((o, dq, dk, dv), want):
        assert got.shape == ref.shape
        np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12)


def test_gqa_oracle_at_kv_heads_equal_heads_is_the_oracle():
    lay = local_strided_layout(5)
    heads, bs, hs = 3, 8, 16
    orc = TransformerOracle(lay, bs, heads=heads, mask_callback=causal_callback)
    rng = np.random.default_rng(3)
    Qa, Ka, Va, dYa = (rng.normal(0, 1, (2, 5 * bs, heads * hs)) for _ in range(4))
    assert np.array_equal(oracle_attention_gqa(orc, heads, Qa, Ka, Va, 0.5, 17),
                          oracle_attention(orc, Qa, Ka, Va, 0.5, 17))
    for a, b in zip(oracle_attention_gqa_grad(orc, heads, Qa, Ka, Va, dYa, 0.5, 17),
                    oracle_attention_grad(orc, Qa, Ka, Va, dYa, 0.5, 17)):
        assert np.array_equal(a, b)


def test_expand_and_sum_groups_follow_repeat_interleave():
    X = np.arange(2 * 3 * 2 * 4, dtype=np.float64).reshape(2, 3, 8)          # kv_heads 2, hs 4
    E = expand_kv(X, 6, 2)
    T = torch.tensor(X).reshape(2, 3, 2, 4).repeat_interleave(3, dim=2).reshape(2, 3, 24).numpy()
    assert np.array_equal(E, T)
    assert np.array_equal(sum_groups(E, 6, 2), 3 * X)
