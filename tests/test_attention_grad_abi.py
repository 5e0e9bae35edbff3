"""bst_attention_train and bst_attention_grad refuse configurations without a fused kernel with BSMM_E_NOKERNEL before
anything is launched, and report other argument errors with the existing codes (no GPU needed: the pointers are never
dereferenced)."""
from blocksparse_b200 import _lib

NN, TN, ORD, Q, K, V, O, DY, MASK = 0x1000, 0x2000, 0x3000, 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
M, L, DELTA, DQ, DK, DV = 0x70000, 0x80000, 0x90000, 0xA0000, 0xB0000, 0xC0000

# out of the envelope: block size, dtype (fp32 or mixed), head_state, alignment of any 16-bit tensor
NOKERNEL = [dict(bs=32), dict(bs=8), dict(dtype=_lib.F32), dict(dtype=-1), dict(hs=32), dict(hs=192),
            dict(q=Q + 2), dict(k=K + 8), dict(v=V + 4), dict(o=O + 2), dict(dtype=_lib.F16, q=Q + 14, mask=MASK, ak=5)]
NOKERNEL_GRAD = [dict(dy=DY + 2), dict(dq=DQ + 4), dict(dk=DK + 8), dict(dv=DV + 6)]


def _train(dtype=_lib.BF16, bs=64, hs=64, q=Q, k=K, v=V, o=O, m=M, l=L, mask=None, ak=-1, heads=2):
    return _lib.load().bst_attention_train(dtype, bs, NN, 1, 6, mask, 1, ak, q, k, v, o, m, l, 0.125, 2, heads, hs, 3, 3, None)


def _grad(dtype=_lib.BF16, bs=64, hs=64, q=Q, k=K, v=V, o=O, dy=DY, m=M, l=L, delta=DELTA, dq=DQ, dk=DK, dv=DV,
          mask=None, ak=-1, heads=2, tn=TN):
    return _lib.load().bst_attention_grad(dtype, bs, NN, tn, ORD, 1, 6, mask, 1, ak, q, k, v, o, dy, m, l, delta,
                                          dq, dk, dv, 0.125, 2, heads, hs, 3, 3, None)


def test_no_fused_kernel_is_reported_before_any_launch():
    before = _lib.last_kernel()
    for kw in NOKERNEL:
        rc = _train(**kw)
        assert rc == _lib.E_NOKERNEL == -7, ("train", kw, rc, _lib.device_error_text())
    for kw in NOKERNEL + NOKERNEL_GRAD:
        rc = _grad(**kw)
        assert rc == _lib.E_NOKERNEL, ("grad", kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before          # nothing was launched


def test_other_argument_errors_keep_their_codes():
    before = _lib.last_kernel()
    for call in (_train, _grad):
        assert call(bs=12) == -2                 # BSMM_E_BSIZE
        assert call(ak=3) == -3                  # autoregress_at_key without a mask: BSMM_E_ARG
        assert call(hs=60) == -3                 # head_state not a multiple of 8
        assert call(q=None) == -3
        assert call(heads=0) == -3
        assert call(m=None) == -3                # the row statistics are required
        assert call(l=None) == -3
    assert _grad(delta=None) == -3
    assert _grad(tn=None) == -3
    assert _grad(dy=None) == -3
    assert _lib.last_kernel() == before
