"""attention_decode without a GPU: the C entries are bound, every argument error is refused before a launch, the
workspace query follows the documented split rule, the Python ValueErrors come before any device is touched, and the
float64 decode reference agrees with the attention reference where the two definitions coincide."""
import ctypes

import numpy as np
import pytest
import torch

from tests._attention_oracle import oracle_attention
from tests._decode_oracle import oracle_decode, oracle_rows
from tests.golden.make_golden import causal_callback
from blocksparse_b200 import BlocksparseTransformer, _lib
from blocksparse_b200.layouts import local_strided_layout
from oracle.bst_oracle import TransformerOracle

E_DTYPE, E_BSIZE, E_ARG = -1, -2, -3
FAKE = 0x10000                       # never dereferenced: every call below fails on the host
F32, F16, BF16 = _lib.F32, _lib.F16, _lib.BF16
SPLIT = 4                            # LUT entries per split (include/bsmm_b200.h)


def test_symbols_are_bound():
    lib = _lib.load()
    for name in ("bst_attention_decode", "bst_attention_decode_workspace_bytes"):
        assert name in _lib.SIGNATURES
        assert hasattr(ctypes.CDLL(_lib.LIB_PATH), name)
        assert getattr(lib, name).argtypes is not None


def _call(dtype=F16, bs=64, lut=FAKE, lut_heads=1, nn_max=5, mask=None, mask_heads=1, ak=-1, q=FAKE, k=FAKE, v=FAKE,
          o=FAKE, pos=FAKE, n=1, batch=2, heads=2, hs=64, cq=4, ck=4, ws=FAKE):
    return _lib.load().bst_attention_decode(dtype, bs, lut, lut_heads, 6, nn_max, mask, mask_heads, ak, q, k, v, o, pos,
                                            n, 0.125, batch, heads, hs, cq, ck, ws, None)


@pytest.mark.parametrize("kw,code,what", [
    (dict(dtype=F32), E_DTYPE, b"fp16 or bf16"),
    (dict(dtype=7), E_DTYPE, b"fp16 or bf16"),
    (dict(bs=8), E_BSIZE, b"block size"),
    (dict(bs=128), E_BSIZE, b"block size"),
    (dict(n=0), E_ARG, b"n must be"),
    (dict(n=65), E_ARG, b"n must be"),
    (dict(bs=16, n=17), E_ARG, b"n must be"),
    (dict(hs=8), E_ARG, b"head_state"),
    (dict(hs=72), E_ARG, b"head_state"),
    (dict(hs=272), E_ARG, b"head_state"),
    (dict(batch=0), E_ARG, b"bad batch"),
    (dict(nn_max=-1), E_ARG, b"bad batch"),
    (dict(ck=0), E_ARG, b"bad batch"),
    (dict(lut_heads=3), E_ARG, b"lut_heads"),
    (dict(mask=FAKE, mask_heads=3), E_ARG, b"mask_heads"),
    (dict(ak=3), E_ARG, b"needs a mask"),
    (dict(lut=None), E_ARG, b"null pointer"),
    (dict(q=None), E_ARG, b"null pointer"),
    (dict(k=None), E_ARG, b"null pointer"),
    (dict(v=None), E_ARG, b"null pointer"),
    (dict(o=None), E_ARG, b"null pointer"),
    (dict(pos=None), E_ARG, b"null pointer"),
    (dict(k=FAKE + 8), E_ARG, b"16-byte aligned"),
    (dict(v=FAKE + 2), E_ARG, b"16-byte aligned"),
    (dict(q=FAKE + 4), E_ARG, b"16-byte aligned"),
    (dict(ws=None), E_ARG, b"null workspace"),
    (dict(ws=FAKE + 4), E_ARG, b"workspace must be 16-byte aligned"),
])
def test_c_argument_errors_before_any_launch(kw, code, what):
    lib = _lib.load()
    before = _lib.last_kernel()
    rc = _call(**kw)
    assert rc == code, (rc, lib.bsmm_last_error())
    assert what in lib.bsmm_last_error(), lib.bsmm_last_error()
    assert _lib.last_kernel() == before
    with pytest.raises(ValueError):
        _lib.check(rc, "bst_attention_decode")


def test_workspace_follows_the_split_rule():
    lib = _lib.load()
    for bs in (16, 32, 64):
        for nn_max in (0, 1, 4, 5, 64, 1000):
            for batch, heads, hs, n in ((1, 1, 16, 1), (8, 16, 64, 1), (3, 5, 256, bs), (64, 16, 128, 16 % bs or bs)):
                got = lib.bst_attention_decode_workspace_bytes(bs, nn_max, batch, heads, hs, n)
                assert got == -(-nn_max // SPLIT) * batch * heads * n * (hs + 2) * 4, (bs, nn_max, batch, heads, hs, n)
    for bad in ((8, 4, 1, 1, 64, 1), (64, 4, 1, 1, 64, 0), (32, 4, 1, 1, 64, 33), (64, 4, 1, 1, 72, 1),
                (64, 4, 1, 1, 272, 1), (64, -1, 1, 1, 64, 1), (64, 4, 0, 1, 64, 1)):
        assert lib.bst_attention_decode_workspace_bytes(*bad) == 0, bad


def _bst(bs=64, hs=64, mask=True):
    lay = local_strided_layout(4)
    return BlocksparseTransformer(lay, bs, heads=2, mask_callback=causal_callback if mask else None), 2 * hs


def _args(bs=64, S=128, n=1, batch=2, dtype=torch.float16):
    ctx = 4 * bs
    return (torch.zeros(batch, n, S, dtype=dtype), torch.zeros(batch, ctx, S, dtype=dtype),
            torch.zeros(batch, ctx, S, dtype=dtype), torch.zeros(batch, dtype=torch.int32))


@pytest.mark.parametrize("case,what", [
    ("fp32", "float16 or bfloat16"),
    ("mixed", "share one dtype"),
    ("bs8", "block size must be 16, 32 or 64"),
    ("hs24", "multiple of 16 up to 256"),
    ("hs272", "multiple of 16 up to 256"),
    ("n0", r"n = 0 query rows"),
    ("n65", r"n = 65 query rows"),
    ("shape", "caches must be"),
    ("noncontig", "contiguous and 16-byte aligned"),
    ("misaligned", "contiguous and 16-byte aligned"),
    ("pos_dtype", "int32 tensor"),
    ("pos_shape", "int32 tensor"),
    ("ak_nomask", "mask_callback"),
    ("cpu", "CUDA tensors"),
])
def test_python_argument_errors_before_any_device(case, what):
    bst, S = _bst()
    q, k, v, pos = _args(S=S)
    kw = {}
    if case == "fp32":
        q, k, v = q.float(), k.float(), v.float()
    elif case == "mixed":
        v = v.to(torch.bfloat16)
    elif case == "bs8":
        bst = BlocksparseTransformer(local_strided_layout(4), 8, heads=2)
        q, k, v, pos = _args(bs=8, S=S)
    elif case == "hs24":
        q, k, v, pos = _args(S=48)
    elif case == "hs272":
        q, k, v, pos = _args(S=544)
    elif case == "n0":
        q = q[:, :0]
    elif case == "n65":
        q = torch.zeros(2, 65, S, dtype=torch.float16)
    elif case == "shape":
        k = k[:, :-1]
    elif case == "noncontig":
        k = torch.zeros(2, S, k.shape[1], dtype=torch.float16).transpose(1, 2)
    elif case == "misaligned":
        k = torch.zeros(k.numel() + 1, dtype=torch.float16)[1:].view(k.shape)
    elif case == "pos_dtype":
        pos = pos.long()
    elif case == "pos_shape":
        pos = pos[:1]
    elif case == "ak_nomask":
        bst, _ = _bst(mask=False)
        kw = dict(autoregress_at_key=3)
    with pytest.raises(ValueError, match=what):
        bst.attention_decode(q, k, v, pos, **kw)


@pytest.mark.parametrize("bs,ak", [(16, None), (32, None), (64, None), (32, 40)])
def test_decode_oracle_matches_attention_oracle(bs, ak):
    """Under a causal layout and mask the valid-key rule hides nothing attention shows: the decode reference of any
    chunk of rows equals the attention reference's rows."""
    lay = local_strided_layout(9)
    heads, hs, batch = 2, 16, 2
    orc = TransformerOracle(lay, bs, heads=heads, mask_callback=causal_callback)
    rng = np.random.default_rng(bs)
    ctx = 9 * bs
    Q, K, V = (rng.normal(0, 1, (batch, ctx, heads * hs)) for _ in range(3))
    full = oracle_attention(orc, Q, K, V, 0.5, autoregress_at_key=ak)
    rows_of, visible = oracle_rows(orc)
    for n, positions in ((1, [0, ctx - 1]), (bs, [bs * 3, 5]), (min(bs, 12), [bs - 3, ctx - 12])):
        Qc = np.stack([Q[b, p:p + n] for b, p in enumerate(positions)])
        got = oracle_decode(rows_of, visible, bs, heads, ctx, Qc, K, V, positions, 0.5, ak)[0]
        want = np.stack([full[b, p:p + n] for b, p in enumerate(positions)])
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
