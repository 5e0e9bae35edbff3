"""bst_attention refuses configurations without a fused kernel with BSMM_E_NOKERNEL before anything is launched, and
reports other argument errors with the existing codes (no GPU needed: the pointers are never dereferenced)."""
from blocksparse_b200 import _lib

LUT, Q, K, V, O, MASK = 0x1000, 0x10000, 0x20000, 0x30000, 0x40000, 0x50000


def _call(dtype=_lib.BF16, bs=64, hs=64, q=Q, k=K, v=V, o=O, mask=None, ak=-1, heads=2):
    lib = _lib.load()
    return lib.bst_attention(dtype, bs, LUT, 1, 6, mask, 1, ak, q, k, v, o, 0.125, 2, heads, hs, 3, 3, None)


def test_no_fused_kernel_is_reported_before_any_launch():
    before = _lib.last_kernel()
    cases = [dict(bs=32), dict(bs=8), dict(dtype=_lib.F32), dict(dtype=-1), dict(hs=32), dict(hs=192),
             dict(q=Q + 2), dict(k=K + 8), dict(v=V + 4), dict(o=O + 2), dict(dtype=_lib.F16, q=Q + 14, mask=MASK, ak=5)]
    for kw in cases:
        rc = _call(**kw)
        assert rc == _lib.E_NOKERNEL == -7, (kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before          # nothing was launched


def test_other_argument_errors_keep_their_codes():
    assert _call(bs=12) == -2                    # BSMM_E_BSIZE
    assert _call(ak=3) == -3                     # autoregress_at_key without a mask: BSMM_E_ARG
    assert _call(hs=60) == -3                    # head_state not a multiple of 8
    assert _call(q=None) == -3
    assert _call(heads=0) == -3
