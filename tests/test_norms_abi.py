"""The layer norm entries refuse bad arguments with BSMM_E_ARG before anything is launched (no GPU needed: the pointers
are never dereferenced), and layer_norm raises ValueError before reaching them."""
import pytest
import torch

from blocksparse_b200 import _lib, layer_norm

X, G, B, Y, M, R, W, D, DG, DB = (0x10000 * i for i in range(1, 11))
E_ARG = -3


def _fwd(dtype=_lib.F16, gdtype=_lib.F32, axis=1, x=X, g=G, b=B, y=Y, mean=M, rstd=R, ws=W, N=8, K=64, S=1, eps=1e-6):
    return _lib.load().bsmm_layer_norm(dtype, gdtype, axis, x, g, b, y, mean, rstd, ws, N, K, S, eps, 0, None)


def _bwd(dtype=_lib.BF16, gdtype=_lib.BF16, axis=0, dy=D, x=X, g=G, b=B, mean=M, rstd=R, dx=Y, dg=DG, db=DB, ws=W, N=8,
         K=64, S=1, eps=1e-6):
    return _lib.load().bsmm_layer_norm_grad(dtype, gdtype, axis, dy, x, g, b, mean, rstd, dx, dg, db, ws, N, K, S, eps, 1,
                                            None)


CASES = [
    (_fwd, dict(dtype=3)), (_fwd, dict(gdtype=-1)), (_fwd, dict(axis=2)), (_fwd, dict(axis=-1)),
    (_fwd, dict(x=None)), (_fwd, dict(g=None)), (_fwd, dict(b=None)), (_fwd, dict(y=None)), (_fwd, dict(mean=None)),
    (_fwd, dict(rstd=None)), (_fwd, dict(axis=0, ws=None)), (_fwd, dict(N=-1)), (_fwd, dict(K=0)),
    (_fwd, dict(S=0)), (_fwd, dict(K=64, S=3)), (_fwd, dict(axis=0, S=2)), (_fwd, dict(eps=-1.0)),
    (_bwd, dict(dtype=7)), (_bwd, dict(gdtype=5)), (_bwd, dict(axis=3)), (_bwd, dict(dy=None)), (_bwd, dict(x=None)),
    (_bwd, dict(g=None)), (_bwd, dict(b=None)), (_bwd, dict(mean=None)), (_bwd, dict(rstd=None)),
    (_bwd, dict(dx=None)), (_bwd, dict(dg=None)), (_bwd, dict(db=None)), (_bwd, dict(ws=None)),
    (_bwd, dict(axis=1, ws=None)), (_bwd, dict(N=-5)), (_bwd, dict(K=-1)), (_bwd, dict(S=2)),
    (_bwd, dict(axis=1, K=10, S=4)),
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
    for axis in (0, 1):
        assert _fwd(axis=axis, N=0) == 0
        assert _bwd(axis=axis, N=0) == 0
    assert _lib.last_kernel() == before


def test_workspace_bytes():
    ws = _lib.load().bsmm_layer_norm_workspace_bytes
    assert ws(1, 8192, 1024, 1) > 0 and ws(0, 4096, 4096, 1) > 0 and ws(0, 256, 4096, 1) > 0
    assert ws(1, 8192, 1024, 4) >= 2 * 4 * 1024          # at least one partial row per owner
    for bad in [(2, 8, 64, 1), (1, 0, 64, 1), (1, 8, 0, 1), (1, 8, 64, 3), (1, 8, 64, 0), (-1, 8, 64, 1)]:
        assert ws(*bad) == 0
    assert ws(1, 2 ** 33, 64, 1) > 0                     # 64-bit N


def test_python_argument_errors_raise_value_error():
    x, g, b = torch.zeros(4, 8), torch.ones(8), torch.zeros(8)
    with pytest.raises(ValueError):
        layer_norm(x, g, b, axis=-1)                     # a CPU tensor: no CPU path
    with pytest.raises(ValueError):
        layer_norm(x, g, b, use_tf=True)
    if not torch.cuda.is_available():
        return
    before = _lib.last_kernel()
    xc, gc, bc = x.cuda(), g.cuda(), b.cuda()
    x3 = torch.zeros(2, 8, 3, device="cuda")
    bad = [lambda: layer_norm(x3, gc, bc, axis=1),                       # a middle axis
           lambda: layer_norm(xc, gc, bc, axis=-1, segments=3),          # K % segments
           lambda: layer_norm(xc.t(), gc, bc, axis=0, segments=2),       # segments on axis 0
           lambda: layer_norm(xc, gc[:7], bc, axis=-1),                  # wrong number of gains
           lambda: layer_norm(xc, gc, torch.zeros(9, device="cuda"), axis=-1),
           lambda: layer_norm(xc, gc, bc, axis=-1, use_tf=True),
           lambda: layer_norm(xc, g, bc, axis=-1),                       # g on the CPU
           lambda: layer_norm(xc.double(), gc, bc, axis=-1),
           lambda: layer_norm(xc, gc, bc, axis=2)]
    for call in bad:
        with pytest.raises(ValueError):
            call()
    assert _lib.last_kernel() == before


def test_reference_signature():
    import inspect
    p = inspect.signature(layer_norm).parameters
    assert list(p) == ["x", "g", "b", "axis", "segments", "epsilon", "relu", "atomics", "bench", "use_tf"]
    assert [p[k].default for k in list(p)[3:]] == [1, 1, 1e-6, False, True, 0, False]
