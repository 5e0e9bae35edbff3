"""The bias_relu, dropout and embedding entries refuse bad arguments with BSMM_E_ARG before anything is launched, and
launch nothing for empty input (no GPU needed: the pointers are fake and never dereferenced). The Python layer raises
ValueError before reaching them, and keeps the reference's signatures."""
import ctypes
import inspect

import pytest
import torch

from blocksparse_b200 import _lib, bias_relu, dropout, embedding_lookup, get_entropy, set_entropy
from blocksparse_b200 import embed, ewops

E_ARG, E_LIMIT = -3, -4
X, B, Y, DY, DX, DB, W, M, S, I = (0x10000 * i for i in range(1, 11))
LL = ctypes.c_longlong


def _br(dtype=_lib.F16, bdt=_lib.F32, axis=1, x=X, b=B, y=Y, N=8, K=64, act=1):
    return _lib.load().bsmm_bias_relu(dtype, bdt, axis, x, b, y, N, K, act, None)


def _brg(dtype=_lib.BF16, bdt=_lib.BF16, axis=0, dy=DY, src=X, b=B, dx=DX, db=DB, ws=W, N=8, K=64, act=2):
    return _lib.load().bsmm_bias_relu_grad(dtype, bdt, axis, dy, src, b, dx, db, ws, N, K, act, None)


def _mask(mask=M, n=100, kp=0.5, state=S):
    return _lib.load().bsmm_dropout_mask(mask, n, kp, state, None)


def _apply(dtype=_lib.F32, x=X, mask=M, y=Y, shape=(4, 6), strides=(6, 1), words=1, kp=0.9, nd=None):
    dims = len(shape if shape is not None else strides)
    nd = dims if nd is None else nd
    arr = LL * max(dims, 1)
    return _lib.load().bsmm_dropout_apply(dtype, x, mask, y, nd, arr(*shape) if shape is not None else None,
                                          arr(*strides) if strides is not None else None, words, kp, None)


def _lookup(dtype=_lib.F16, itype=_lib.LABEL_I64, emb=W, idx=I, y=Y, n=10, C=50, K=16):
    return _lib.load().bsmm_embedding_lookup(dtype, itype, emb, idx, y, n, C, K, None)


def _egrad(dtype=_lib.F32, itype=_lib.LABEL_U8, dy=DY, idx=I, dw=DX, ws=W, n=10, C=50, K=16):
    return _lib.load().bsmm_embedding_grad(dtype, itype, dy, idx, dw, ws, n, C, K, None)


CASES = [
    (_br, dict(dtype=3)), (_br, dict(bdt=-1)), (_br, dict(axis=2)), (_br, dict(axis=-1)), (_br, dict(x=None)),
    (_br, dict(b=None)), (_br, dict(y=None)), (_br, dict(N=-1)), (_br, dict(K=0)), (_br, dict(act=3)),
    (_br, dict(act=-1)),
    (_brg, dict(dtype=5)), (_brg, dict(bdt=4)), (_brg, dict(axis=3)), (_brg, dict(dy=None)), (_brg, dict(src=None)),
    (_brg, dict(b=None)), (_brg, dict(dx=None)), (_brg, dict(db=None)), (_brg, dict(ws=None)), (_brg, dict(N=-2)),
    (_brg, dict(K=-1)), (_brg, dict(act=7)), (_brg, dict(act=0, db=None)),
    (_mask, dict(mask=None)), (_mask, dict(state=None)), (_mask, dict(n=-1)), (_mask, dict(kp=0.0)),
    (_mask, dict(kp=1.5)), (_mask, dict(kp=-0.5)), (_mask, dict(kp=float("nan"))),
    (_apply, dict(dtype=3)), (_apply, dict(x=None)), (_apply, dict(mask=None)), (_apply, dict(y=None)),
    (_apply, dict(nd=9, shape=(1,) * 9, strides=(0,) * 9)), (_apply, dict(nd=-1)), (_apply, dict(shape=(4, -6))),
    (_apply, dict(strides=(6, -1))), (_apply, dict(words=0)), (_apply, dict(shape=(4, 9), strides=(9, 1))),
    (_apply, dict(strides=(1, 4))), (_apply, dict(kp=0.0)), (_apply, dict(kp=2.0)), (_apply, dict(shape=None)),
    (_apply, dict(strides=None)),
    (_lookup, dict(dtype=3)), (_lookup, dict(itype=4)), (_lookup, dict(itype=-1)), (_lookup, dict(emb=None)),
    (_lookup, dict(idx=None)), (_lookup, dict(y=None)), (_lookup, dict(n=-1)), (_lookup, dict(C=-1)),
    (_lookup, dict(K=0)),
    (_egrad, dict(dtype=-2)), (_egrad, dict(itype=9)), (_egrad, dict(dy=None)), (_egrad, dict(idx=None)),
    (_egrad, dict(dw=None)), (_egrad, dict(ws=None)), (_egrad, dict(n=-3)), (_egrad, dict(C=-1)), (_egrad, dict(K=0)),
]


@pytest.mark.parametrize("fn,kw", CASES, ids=["%s-%s" % (f.__name__.strip("_"), "-".join("%s%s" % i for i in kw.items()))
                                              for f, kw in CASES])
def test_bad_arguments_return_e_arg_before_any_launch(fn, kw):
    before = _lib.last_kernel()
    rc = fn(**kw)
    assert rc == E_ARG, (kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before


def test_limits():
    before = _lib.last_kernel()
    assert _egrad(n=2 ** 31) == E_LIMIT
    assert _egrad(C=2 ** 31 - 1) == E_LIMIT
    assert _lib.last_kernel() == before


def test_zero_sizes_launch_nothing():
    before = _lib.last_kernel()
    for axis in (0, 1):
        assert _br(axis=axis, N=0) == 0
        assert _brg(axis=axis, N=0) == 0
    assert _brg(act=0, src=None, dx=None, N=0) == 0
    assert _mask(n=0) == 0
    assert _apply(shape=(4, 0), strides=(0, 1)) == 0
    assert _lookup(n=0) == 0
    assert _lookup(C=0, emb=None, n=0) == 0
    assert _egrad(n=0, ws=None) == 0
    assert _egrad(C=0) == 0
    assert _lib.last_kernel() == before


def test_workspace_bytes():
    ws = _lib.load().bsmm_bias_grad_workspace_bytes
    assert ws(1, 16384, 1024) >= 4 * 1024 and ws(0, 16384, 1024) >= 4 * 1024
    assert ws(1, 2 ** 33, 3) > 0 and ws(0, 2 ** 33, 3) > 0            # 64-bit N
    for bad in [(2, 8, 64), (1, 0, 64), (1, 8, 0), (-1, 8, 64)]:
        assert ws(*bad) == 0
    ew = _lib.load().bsmm_embedding_grad_workspace_bytes
    assert ew(16384, 256, 512) >= 4 * 4 * 16384
    for bad in [(0, 256, 512), (2 ** 31, 256, 512), (10, 0, 5), (10, 5, 0), (10, 2 ** 31 - 1, 4)]:
        assert ew(*bad) == 0


def test_python_argument_errors_raise_value_error():
    x, b = torch.zeros(4, 8), torch.zeros(8)
    cpu = [lambda: bias_relu(x, b),                                      # a CPU tensor: no CPU path
           lambda: bias_relu(x, b, relu=True, fast_gelu=True),
           lambda: bias_relu(x, b, use_tf=True),
           lambda: dropout(x, 0.0),
           lambda: dropout(x, 1.5),
           lambda: dropout(x, -0.1),
           lambda: dropout(x, 0.5),
           lambda: embedding_lookup(x, torch.zeros(3, dtype=torch.int64)),
           lambda: embedding_lookup(x, torch.zeros(3, dtype=torch.int64), use_tf=True),
           lambda: get_entropy("cpu"),
           lambda: set_entropy(1, "cpu")]
    for call in cpu:
        with pytest.raises(ValueError):
            call()
    if not torch.cuda.is_available():
        return
    before = _lib.last_kernel()
    xc, bc = x.cuda(), b.cuda()
    x3 = torch.zeros(2, 8, 3, device="cuda")
    i64 = torch.zeros(3, dtype=torch.int64, device="cuda")
    bad = [lambda: bias_relu(x3, bc, axis=1),                            # a middle axis
           lambda: bias_relu(xc, bc, axis=2),
           lambda: bias_relu(xc, bc[:7]),
           lambda: bias_relu(xc, b),                                     # b on the CPU
           lambda: bias_relu(xc.double(), bc),
           lambda: bias_relu(xc, bc, relu=True, fast_gelu=True),
           lambda: bias_relu(xc, bc, use_tf=True),
           lambda: bias_relu(torch.zeros(1, device="cuda").expand(1, 2 ** 31), bc),   # K past int
           lambda: dropout(xc, 0.0),
           lambda: dropout(xc, 1.01),
           lambda: dropout(xc.double(), 0.5),
           lambda: dropout(xc, 0.5, mask_shape=(4,)),                    # rank
           lambda: dropout(xc, 0.5, mask_shape=(2, 8)),                  # neither 1 nor x's dim
           lambda: dropout(xc, 0.5, mask=torch.zeros(1, dtype=torch.int64, device="cuda")),
           lambda: dropout(xc, 0.5, mask=torch.zeros(2, dtype=torch.int32, device="cuda")),
           lambda: dropout(xc, 0.5, mask=torch.zeros(1, dtype=torch.int32)),
           lambda: dropout(torch.zeros((1,) * 9, device="cuda"), 0.5),
           lambda: embedding_lookup(xc, i64.cpu()),
           lambda: embedding_lookup(xc, i64.float()),
           lambda: embedding_lookup(xc, i64.to(torch.int16)),
           lambda: embedding_lookup(xc[0], i64),
           lambda: embedding_lookup(xc.double(), i64),
           lambda: embedding_lookup(xc, i64, use_tf=True)]
    for call in bad:
        with pytest.raises(ValueError):
            call()
    assert _lib.last_kernel() == before


def test_reference_signatures():
    p = inspect.signature(bias_relu).parameters
    assert list(p) == ["x", "b", "axis", "relu", "fast_gelu", "atomics", "bench", "use_tf"]
    assert [p[k].default for k in list(p)[2:]] == [-1, False, False, True, 0, False]
    p = inspect.signature(dropout).parameters
    assert list(p) == ["x", "keep_prob", "mask", "mask_shape"]
    assert [p[k].default for k in list(p)[2:]] == [None, None]
    p = inspect.signature(embedding_lookup).parameters
    assert list(p) == ["emb", "idx", "sort_grad", "bench", "use_tf"]
    assert [p[k].default for k in list(p)[2:]] == [True, 0, False]
    assert [(k, v.default) for k, v in inspect.signature(set_entropy).parameters.items()] == [("init", None),
                                                                                              ("device", None)]
    assert [(k, v.default) for k, v in inspect.signature(get_entropy).parameters.items()] == [("device", None)]
    assert ewops.__all__ == ["bias_relu", "dropout", "set_entropy", "get_entropy"]
    assert embed.__all__ == ["embedding_lookup"]
