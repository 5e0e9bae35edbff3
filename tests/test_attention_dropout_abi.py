"""bst_attention_dropout, bst_attention_train_dropout and bst_attention_grad_dropout: keep_prob outside (0, 1] and a null
seed_call with keep_prob < 1 are argument errors, the counterparts' argument checks keep their codes, and calls outside
the fused envelope return BSMM_E_NOKERNEL; all before any launch (no GPU needed: the pointers are never
dereferenced)."""
import pytest

from blocksparse_b200 import _lib

NN, TN, ORD, Q, K, V, O, DY, MASK = 0x1000, 0x2000, 0x3000, 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
M, L, DELTA, DQ, DK, DV, SEED = 0x70000, 0x80000, 0x90000, 0xA0000, 0xB0000, 0xC0000, 0xD0000


def _fwd(kp=0.9, seed=SEED, dtype=_lib.BF16, bs=64, hs=64, q=Q, o=O, mask=None, ak=-1, heads=2, **_):
    return _lib.load().bst_attention_dropout(dtype, bs, NN, 1, 6, mask, 1, ak, q, K, V, o, 0.125, 2, heads, hs, 3, 3,
                                             kp, seed, None)


def _train(kp=0.9, seed=SEED, dtype=_lib.BF16, bs=64, hs=64, q=Q, o=O, m=M, l=L, mask=None, ak=-1, heads=2, **_):
    return _lib.load().bst_attention_train_dropout(dtype, bs, NN, 1, 6, mask, 1, ak, q, K, V, o, m, l, 0.125, 2, heads,
                                                   hs, 3, 3, kp, seed, None)


def _grad(kp=0.9, seed=SEED, dtype=_lib.BF16, bs=64, hs=64, q=Q, o=O, m=M, l=L, mask=None, ak=-1, heads=2, dy=DY,
          delta=DELTA, tn=TN, **_):
    return _lib.load().bst_attention_grad_dropout(dtype, bs, NN, tn, ORD, 1, 6, mask, 1, ak, q, K, V, o, dy, m, l, delta,
                                                  DQ, DK, DV, 0.125, 2, heads, hs, 3, 3, kp, seed, None)


CALLS = [_fwd, _train, _grad]


@pytest.mark.parametrize("call", CALLS, ids=["fwd", "train", "grad"])
def test_dropout_arguments_are_refused_before_any_launch(call):
    before = _lib.last_kernel()
    for kp in (0.0, -0.25, 1.0 + 1e-9, 2.0, float("nan"), float("inf")):
        assert call(kp=kp) == -3, kp                       # BSMM_E_ARG
        assert "keep_prob" in _lib.device_error_text()
    assert call(kp=0.5, seed=None) == -3                   # keep_prob < 1 needs the device [seed, call]
    assert "seed_call" in _lib.device_error_text()
    # the dropout checks come first: a bad keep_prob is reported even where the counterpart's checks would fail
    assert call(kp=0.0, bs=12) == -3 and "keep_prob" in _lib.device_error_text()
    assert _lib.last_kernel() == before


@pytest.mark.parametrize("call", CALLS, ids=["fwd", "train", "grad"])
def test_counterpart_checks_keep_their_codes(call):
    before = _lib.last_kernel()
    for kp in (0.5, 1.0):
        assert call(kp=kp, bs=12) == -2                    # BSMM_E_BSIZE
        assert call(kp=kp, ak=3) == -3                     # autoregress_at_key without a mask
        assert call(kp=kp, hs=60) == -3
        assert call(kp=kp, q=None) == -3
        assert call(kp=kp, heads=0) == -3
        if call is not _fwd:
            assert call(kp=kp, m=None) == -3 and call(kp=kp, l=None) == -3
    assert _grad(delta=None) == -3 and _grad(tn=None) == -3 and _grad(dy=None) == -3
    assert _lib.last_kernel() == before


@pytest.mark.parametrize("call", CALLS, ids=["fwd", "train", "grad"])
def test_outside_the_envelope_is_nokernel(call):
    """the counterparts' envelope, with and without dropout; keep_prob 1 needs no seed_call"""
    before = _lib.last_kernel()
    for kw in (dict(bs=32), dict(dtype=_lib.F32), dict(dtype=-1), dict(hs=32), dict(hs=192), dict(q=Q + 2),
               dict(o=O + 2), dict(dtype=_lib.F16, q=Q + 14, mask=MASK, ak=5)):
        assert call(**kw) == _lib.E_NOKERNEL, (kw, _lib.device_error_text())
        assert call(kp=1.0, seed=None, **kw) == _lib.E_NOKERNEL, kw
    assert _lib.last_kernel() == before
