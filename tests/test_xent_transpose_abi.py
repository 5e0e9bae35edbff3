"""The softmax cross-entropy and transpose entries refuse bad arguments with BSMM_E_ARG before anything is launched (no
GPU needed: the pointers are never dereferenced), and the Python ops raise ValueError before reaching them."""
import pytest
import torch

from blocksparse_b200 import _lib

X, L, O, S, G = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000
E_ARG = -3


def _xent(dtype=_lib.F16, lt=_lib.LABEL_I32, x=X, labels=L, loss=O, lse=S, N=8, K=50257):
    return _lib.load().bst_softmax_xent(dtype, lt, x, labels, loss, lse, N, K, None)


def _grad(dtype=_lib.BF16, lt=_lib.LABEL_I64, x=X, labels=L, lse=S, dy=G, dx=O, N=8, K=1000):
    return _lib.load().bst_softmax_xent_grad(dtype, lt, x, labels, lse, dy, dx, N, K, None)


def _tr(dtype=_lib.F32, x=X, y=O, D=(2, 3, 4, 5)):
    return _lib.load().bst_transpose_0213(dtype, x, y, *D, None)


CASES = [
    (_xent, dict(dtype=3)), (_xent, dict(dtype=-1)), (_xent, dict(lt=4)), (_xent, dict(lt=-1)),
    (_xent, dict(x=None)), (_xent, dict(labels=None)), (_xent, dict(loss=None)), (_xent, dict(lse=None)),
    (_xent, dict(K=0)), (_xent, dict(K=-5)), (_xent, dict(N=-1)),
    (_grad, dict(dtype=9)), (_grad, dict(lt=8)), (_grad, dict(x=None)), (_grad, dict(labels=None)),
    (_grad, dict(lse=None)), (_grad, dict(dy=None)), (_grad, dict(dx=None)), (_grad, dict(K=0)), (_grad, dict(N=-2)),
    (_tr, dict(dtype=3)), (_tr, dict(x=None)), (_tr, dict(y=None)),
    (_tr, dict(D=(-1, 3, 4, 5))), (_tr, dict(D=(2, -3, 4, 5))), (_tr, dict(D=(2, 3, -4, 5))), (_tr, dict(D=(2, 3, 4, -5))),
]


@pytest.mark.parametrize("fn,kw", CASES, ids=["%s-%s" % (f.__name__.strip("_"), "-".join("%s%s" % i for i in kw.items()))
                                              for f, kw in CASES])
def test_bad_arguments_return_e_arg_before_any_launch(fn, kw):
    before = _lib.last_kernel()
    rc = fn(**kw)
    assert rc == E_ARG, (kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before


def test_zero_rows_launch_nothing():
    before = _lib.last_kernel()
    for lt in (_lib.LABEL_U8, _lib.LABEL_U16, _lib.LABEL_I32, _lib.LABEL_I64):
        assert _xent(lt=lt, N=0) == 0
        assert _grad(lt=lt, N=0) == 0
    for D in [(0, 3, 4, 5), (2, 0, 4, 5), (2, 3, 0, 5), (2, 3, 4, 0), (0, 0, 0, 0)]:
        assert _tr(D=D) == 0
    assert _lib.last_kernel() == before


def test_label_codes():
    assert _lib.label_code(torch.uint8) == _lib.LABEL_U8
    assert _lib.label_code(torch.int32) == _lib.LABEL_I32
    assert _lib.label_code(torch.int64) == _lib.LABEL_I64
    assert _lib.label_code(torch.uint16) == _lib.LABEL_U16
    for dt in (torch.float32, torch.int16, torch.int8, torch.bool):
        with pytest.raises(ValueError):
            _lib.label_code(dt)


def test_python_ops_raise_value_error_before_any_launch():
    from blocksparse_b200 import softmax_cross_entropy, transpose_0213, transpose_2d
    x, lab = torch.zeros(4, 10), torch.zeros(4, dtype=torch.int64)
    cpu = [lambda: softmax_cross_entropy(x, lab), lambda: softmax_cross_entropy(logits=x),
           lambda: softmax_cross_entropy(labels=lab), lambda: transpose_0213(torch.zeros(1, 2, 3, 4)),
           lambda: transpose_2d(torch.zeros(2, 3))]
    for call in cpu:
        with pytest.raises(ValueError):
            call()
    if not torch.cuda.is_available():
        return
    before = _lib.last_kernel()
    xc, labc = x.cuda(), lab.cuda()
    bad = [lambda: softmax_cross_entropy(xc, lab),                             # labels on the CPU
           lambda: softmax_cross_entropy(xc, labc.float()),                    # float labels
           lambda: softmax_cross_entropy(xc, labc.to(torch.int16)),            # unsupported label dtype
           lambda: softmax_cross_entropy(xc, labc[:3]),                        # wrong label count
           lambda: softmax_cross_entropy(xc.int(), labc),                      # unsupported logits dtype
           lambda: softmax_cross_entropy(xc.double(), labc),
           lambda: softmax_cross_entropy(torch.zeros((), device="cuda"), labc[:1]),   # rank 0
           lambda: softmax_cross_entropy(torch.zeros(4, 0, device="cuda"), labc),     # K = 0
           lambda: transpose_0213(torch.zeros(2, 3, 4, device="cuda")),        # rank 3
           lambda: transpose_0213(torch.zeros(1, 2, 3, 4, 5, device="cuda")),  # rank 5
           lambda: transpose_0213(torch.zeros(1, 2, 3, 4, device="cuda", dtype=torch.float64)),
           lambda: transpose_2d(torch.zeros(2, 3, 4, device="cuda")),          # rank 3
           lambda: transpose_2d(torch.zeros(5, device="cuda")),               # rank 1
           lambda: transpose_2d(torch.zeros(2, 3, device="cuda", dtype=torch.int32))]
    for call in bad:
        with pytest.raises(ValueError):
            call()
    assert _lib.last_kernel() == before
