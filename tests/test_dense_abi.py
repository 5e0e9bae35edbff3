"""The dense softmax / top-k entries refuse bad arguments with BSMM_E_ARG before anything is launched (no GPU needed:
the pointers are never dereferenced), and the Python ops raise ValueError before reaching them."""
import pytest

from blocksparse_b200 import _lib

X, Y, M, I = 0x10000, 0x20000, 0x30000, 0x40000
E_ARG = -3


def _softmax(dtype=_lib.F16, x=X, mask=None, y=Y, D=(2, 3, 4, 64), m1=0, m2=0):
    return _lib.load().bst_dense_softmax(dtype, x, mask, y, *D, m1, m2, 1.0, None)


def _grad(dtype=_lib.F16, dy=X, y=Y, mask=None, dx=I, D=(2, 3, 4, 64), m1=0, m2=0):
    return _lib.load().bst_dense_softmax_grad(dtype, dy, y, mask, dx, *D, m1, m2, 1.0, None)


def _tks(dtype=_lib.BF16, x=X, mask=None, y=Y, D=(2, 3, 4, 64), m1=0, m2=0, k=8):
    return _lib.load().bst_topk_softmax(dtype, x, mask, y, *D, m1, m2, k, 1.0, None)


def _topk(dtype=_lib.F32, x=X, y=Y, idx=I, rows=12, D3=64, k=8, mode=0):
    return _lib.load().bst_topk(dtype, x, y, idx, rows, D3, k, mode, None)


CASES = [
    (_softmax, dict(dtype=3)), (_softmax, dict(dtype=-1)), (_softmax, dict(x=None)), (_softmax, dict(y=None)),
    (_softmax, dict(D=(2, 3, 4, 0))), (_softmax, dict(D=(-1, 3, 4, 8))),
    (_softmax, dict(mask=M, m2=32)), (_softmax, dict(mask=M, m1=192)), (_softmax, dict(mask=M, m1=128, m2=64)),
    (_grad, dict(dtype=7)), (_grad, dict(dy=None)), (_grad, dict(y=None)), (_grad, dict(dx=None)),
    (_grad, dict(D=(2, 3, 4, 0))), (_grad, dict(mask=M, m2=1)),
    (_tks, dict(dtype=5)), (_tks, dict(x=None)), (_tks, dict(y=None)), (_tks, dict(k=0)), (_tks, dict(k=65)),
    (_tks, dict(D=(1, 1, 2, 1025), k=4)), (_tks, dict(D=(2, 3, 4, 0), k=1)),
    (_topk, dict(dtype=-2)), (_topk, dict(x=None)), (_topk, dict(y=None)), (_topk, dict(idx=None)),
    (_topk, dict(k=0)), (_topk, dict(k=65)), (_topk, dict(D3=1025, k=4)), (_topk, dict(D3=0, k=1)),
    (_topk, dict(mode=3)), (_topk, dict(rows=-1)),
]


@pytest.mark.parametrize("fn,kw", CASES, ids=["%s-%s" % (f.__name__.strip("_"), "-".join("%s%s" % i for i in kw.items()))
                                              for f, kw in CASES])
def test_bad_arguments_return_e_arg_before_any_launch(fn, kw):
    before = _lib.last_kernel()
    rc = fn(**kw)
    assert rc == E_ARG, (kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before


def test_valid_strides_and_empty_work_launch_nothing():
    """Zero rows is a valid call that launches nothing; the mask strides a (1|D1, 1|D2, D3) mask can have pass."""
    before = _lib.last_kernel()
    for m1, m2 in [(0, 0), (0, 64), (64, 0), (256, 64)]:
        assert _softmax(mask=M, m1=m1, m2=m2, D=(0, 3, 4, 64)) == 0
    assert _topk(rows=0) == 0 and _topk(rows=0, idx=None, mode=2) == 0
    assert _tks(D=(2, 0, 4, 64)) == 0
    assert _lib.last_kernel() == before


def test_python_ops_raise_value_error_before_any_launch():
    import torch
    from blocksparse_b200 import masked_softmax, masked_top_k_softmax, rectified_top_k, softmax, top_k
    x = torch.zeros(2, 3, 8)
    for call in [lambda: softmax(x), lambda: top_k(x, 2), lambda: masked_softmax(torch.zeros(()))]:
        with pytest.raises(ValueError):
            call()
    if not torch.cuda.is_available():
        return
    xc = x.cuda()
    bad = [lambda: masked_softmax(xc, torch.ones(3, 8)),               # rank differs
           lambda: masked_softmax(xc, torch.ones(1, 3, 1)),            # last dim 1
           lambda: masked_softmax(xc, torch.ones(2, 1, 8).unsqueeze(0)),
           lambda: masked_softmax(xc.int()),
           lambda: top_k(xc, 0), lambda: top_k(xc, 9), lambda: rectified_top_k(torch.zeros(2, 1025).cuda(), 3),
           lambda: masked_top_k_softmax(xc, 9)]
    for call in bad:
        with pytest.raises(ValueError):
            call()
