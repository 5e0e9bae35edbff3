"""The elementwise entries refuse bad arguments with BSMM_E_ARG before anything is launched and launch nothing for empty
input (no GPU needed: the pointers are fake and never dereferenced). The Python layer raises ValueError before reaching
them, keeps the reference's signatures, and its names stay out of the package's and ewops' __all__. The float64 oracle
agrees with torch float64 autograd for every op."""
import ast
import ctypes
import inspect
import os

import numpy as np
import pytest
import torch

import blocksparse_b200
from blocksparse_b200 import _lib, elementwise, ewops
from oracle import elementwise_oracle as eo

E_ARG, E_LIMIT = -3, -4
X, Y, B, Z, DZ, DX, DY, W = (0x10000 * i for i in range(1, 9))
U8, U16, I32, I64 = _lib.LABEL_U8, _lib.LABEL_U16, _lib.LABEL_I32, _lib.LABEL_I64


def _fwd(dtype=_lib.F32, bdt=_lib.F32, op=2, x=X, y=Y, b=B, z=Z, n=64, K=0):
    return _lib.load().bsmm_ew_forward(dtype, bdt, op, x, y, b, z, n, K, 1.0, None)


def _bwd(dtype=_lib.F16, op=3, dz=DZ, x=X, y=Y, dx=DX, dy=DY, n=64):
    return _lib.load().bsmm_ew_backward(dtype, op, dz, x, y, dx, dy, n, 1.0, None)


def _gmul(dtype=_lib.BF16, gdt=_lib.F32, dz=DZ, x=X, g=B, dx=DX, dg=DY, ws=W, N=8, K=16):
    return _lib.load().bsmm_gain_mul_grad(dtype, gdt, dz, x, g, dx, dg, ws, N, K, None)


def _cast(xdt=_lib.F32, ydt=_lib.BF16, x=X, y=Y, n=10):
    return _lib.load().bsmm_float_cast(xdt, ydt, x, y, n, None)


def _filt(dtype=_lib.F16, x=X, y=Y, n=10):
    return _lib.load().bsmm_filter_tensor(dtype, x, y, n, 1.0, None, 0.0, 1, 1, None)


def _addn(dtype=_lib.F32, ptrs=(X, Y, B), count=3, y=Z, n=10):
    arr = (ctypes.c_void_p * max(len(ptrs), 1))(*ptrs) if ptrs is not None else None
    return _lib.load().bsmm_add_n(dtype, arr, count, y, n, None)


def _gate(dtype=_lib.F32, loga=X, gate=Y, conc=Z, n=10, la=-0.1, lb=1.1, eps=1e-6, state=W):
    return _lib.load().bsmm_concrete_gate(dtype, loga, gate, conc, n, 1.5, la, lb, eps, state, None)


def _gate_grad(dtype=_lib.F32, dg=DZ, conc=Z, dl=DX, n=10, la=-0.1, lb=1.1):
    return _lib.load().bsmm_concrete_gate_grad(dtype, dg, conc, dl, n, 1.5, la, lb, None)


def _gate_infer(dtype=_lib.F16, loga=X, gate=Y, n=10, la=-0.1, lb=1.1):
    return _lib.load().bsmm_concrete_gate_infer(dtype, loga, gate, n, la, lb, None)


def _gather(es=4, x=X, idx=Y, y=Z, d0=4, d1=5, d2=6, grad=False):
    fn = _lib.load().bsmm_fancy_gather_grad if grad else _lib.load().bsmm_fancy_gather
    return fn(es, x, idx, y, d0, d1, d2, None)


def _rmax(dtype=_lib.F32, it=U8, x=X, y=Y, a=Z, d0=4, d1=5, d2=6, grad=False):
    if grad:
        return _lib.load().bsmm_reduce_max_grad(dtype, it, x, a, y, d0, d1, d2, None)
    return _lib.load().bsmm_reduce_max(dtype, it, x, y, a, d0, d1, d2, None)


CASES = [
    (_fwd, dict(dtype=3)), (_fwd, dict(op=-1)), (_fwd, dict(op=20)), (_fwd, dict(n=-1)), (_fwd, dict(x=None)),
    (_fwd, dict(z=None)), (_fwd, dict(y=None)), (_fwd, dict(op=18, b=None, K=8)), (_fwd, dict(op=19, bdt=5, K=8)),
    (_fwd, dict(op=18, K=0)), (_fwd, dict(op=19, K=7)),
    (_bwd, dict(dtype=-1)), (_bwd, dict(op=0)), (_bwd, dict(op=1)), (_bwd, dict(op=6)), (_bwd, dict(op=18)),
    (_bwd, dict(op=19)), (_bwd, dict(op=20)), (_bwd, dict(n=-1)), (_bwd, dict(dz=None)), (_bwd, dict(x=None)),
    (_bwd, dict(dx=None)), (_bwd, dict(y=None)), (_bwd, dict(dy=None)),
    (_gmul, dict(dtype=3)), (_gmul, dict(gdt=3)), (_gmul, dict(N=-1)), (_gmul, dict(K=0)), (_gmul, dict(dz=None)),
    (_gmul, dict(x=None)), (_gmul, dict(g=None)), (_gmul, dict(dx=None)), (_gmul, dict(dg=None)),
    (_gmul, dict(ws=None)),
    (_cast, dict(xdt=3)), (_cast, dict(ydt=-1)), (_cast, dict(n=-1)), (_cast, dict(x=None)), (_cast, dict(y=None)),
    (_filt, dict(dtype=4)), (_filt, dict(n=-2)), (_filt, dict(x=None)), (_filt, dict(y=None)),
    (_addn, dict(dtype=3)), (_addn, dict(count=0)), (_addn, dict(count=9, ptrs=(X,) * 9)), (_addn, dict(n=-1)),
    (_addn, dict(ptrs=None)), (_addn, dict(ptrs=(X, None, B))), (_addn, dict(y=None)),
    (_gate, dict(dtype=3)), (_gate, dict(n=-1)), (_gate, dict(la=1.2)), (_gate, dict(eps=0.5)),
    (_gate, dict(eps=-1e-3)), (_gate, dict(loga=None)), (_gate, dict(gate=None)), (_gate, dict(conc=None)),
    (_gate, dict(state=None)),
    (_gate_grad, dict(dtype=3)), (_gate_grad, dict(n=-1)), (_gate_grad, dict(la=2.0, lb=1.0)),
    (_gate_grad, dict(dg=None)), (_gate_grad, dict(conc=None)), (_gate_grad, dict(dl=None)),
    (_gate_infer, dict(dtype=3)), (_gate_infer, dict(loga=None)), (_gate_infer, dict(gate=None)),
    (_gate_infer, dict(la=1.0, lb=1.0)),
    (_gather, dict(es=8)), (_gather, dict(es=1)), (_gather, dict(d0=-1)), (_gather, dict(d2=-1)),
    (_gather, dict(x=None)), (_gather, dict(idx=None)), (_gather, dict(y=None)), (_gather, dict(es=3, grad=True)),
    (_gather, dict(d1=-1, grad=True)), (_gather, dict(y=None, grad=True)),
    (_rmax, dict(dtype=3)), (_rmax, dict(it=I64)), (_rmax, dict(it=7)), (_rmax, dict(d1=0)), (_rmax, dict(d0=-1)),
    (_rmax, dict(d1=257)), (_rmax, dict(it=U16, d1=65537)), (_rmax, dict(x=None)), (_rmax, dict(y=None)),
    (_rmax, dict(a=None)), (_rmax, dict(d1=300, grad=True)), (_rmax, dict(a=None, grad=True)),
]


@pytest.mark.parametrize("fn,kw", CASES, ids=["%s-%s" % (f.__name__.strip("_"), "-".join("%s%s" % i for i in kw.items()))
                                              for f, kw in CASES])
def test_bad_arguments_return_e_arg_before_any_launch(fn, kw):
    before = _lib.last_kernel()
    rc = fn(**kw)
    assert rc == E_ARG, (kw, rc, _lib.device_error_text())
    assert _lib.last_kernel() == before


def test_limits_and_zero_sizes_launch_nothing():
    before = _lib.last_kernel()
    assert _gmul(N=2 ** 62, K=4) == E_LIMIT
    assert _gather(d0=2 ** 40, d1=2 ** 20, d2=2 ** 20) == E_LIMIT
    assert _rmax(it=I32, d0=2 ** 40, d1=2 ** 20, d2=2 ** 20) == E_LIMIT
    for call in (lambda: _fwd(n=0), lambda: _fwd(op=18, n=0, K=8), lambda: _bwd(n=0), lambda: _gmul(N=0),
                 lambda: _cast(n=0), lambda: _filt(n=0), lambda: _addn(n=0), lambda: _gate(n=0),
                 lambda: _gate_grad(n=0), lambda: _gate_infer(n=0), lambda: _gather(d0=0), lambda: _gather(d2=0),
                 lambda: _gather(d1=0, grad=True), lambda: _rmax(d0=0), lambda: _rmax(d2=0, grad=True)):
        assert call() == 0
    # index types up to their capacity are accepted (and, with d0 = 0, launch nothing)
    assert _rmax(d0=0, d1=256) == 0 and _rmax(d0=0, it=U16, d1=65536) == 0 and _rmax(d0=0, it=I32, d1=70000) == 0
    assert _lib.last_kernel() == before


def test_python_argument_errors_raise_value_error():
    ew = elementwise
    x = torch.zeros(4, 8)
    cpu = [lambda: ew.add(x, x), lambda: ew.sigmoid(x), lambda: ew.float_cast(x, torch.float16),
           lambda: ew.filter_tensor(x), lambda: ew.add_n8([x, x]), lambda: ew.add_n([x, x, x]),
           lambda: ew.concrete_gate(x), lambda: ew.concrete_gate_infer(x),
           lambda: ew.fancy_gather(x, torch.zeros(4, dtype=torch.int32)), lambda: ew.reduce_max(x, 0),
           lambda: ew.assign_add(x, x), lambda: ew.add(1.0, x), lambda: ew.add_n([]), lambda: ew.add_n8([])]
    for call in cpu:
        with pytest.raises(ValueError):
            call()
    if not torch.cuda.is_available():
        return
    before = _lib.last_kernel()
    c = x.cuda()
    i = torch.zeros(4, dtype=torch.int32, device="cuda")
    bad = [lambda: ew.add(c, c.half()), lambda: ew.multiply(c, x), lambda: ew.add(c.double(), c.double()),
           lambda: ew.elu(c, alpha="1"), lambda: ew.swish(c, alpha=None), lambda: ew.sigmoid(c.int()),
           lambda: ew.float_cast(c, torch.float64), lambda: ew.float_cast(c, torch.float16, dx_dtype=torch.int32),
           lambda: ew.filter_tensor(c, scale="2"), lambda: ew.filter_tensor(c, scale=torch.ones(2, device="cuda")),
           lambda: ew.filter_tensor(c, scale=torch.ones(1)), lambda: ew.filter_tensor(c, saturate=None),
           lambda: ew.filter_tensor(c, scale=torch.ones(1, device="cuda", dtype=torch.float16)),
           lambda: ew.add_n8([c] * 9), lambda: ew.add_n8([c, c.half()]), lambda: ew.add_n8([c, c[:2]]),
           lambda: ew.add_n([c, c[:2]]), lambda: ew.add_n([c, c, c[:3]]),
           lambda: ew.concrete_gate(c, tempurature=0), lambda: ew.concrete_gate(c, limit_a=1.2),
           lambda: ew.concrete_gate(c, epsilon=0.5), lambda: ew.concrete_gate(c, tempurature="x"),
           lambda: ew.concrete_gate_infer(c, limit_a=1.1, limit_b=1.1),
           lambda: ew.fancy_gather(c, i.long()), lambda: ew.fancy_gather(c, i[:3]), lambda: ew.fancy_gather(c[0], i),
           lambda: ew.fancy_gather(c, i.cpu()), lambda: ew.fancy_gather(c.double(), i),
           lambda: ew.fancy_gather(c, i, use_tf=True),
           lambda: ew.reduce_max(c, 2), lambda: ew.reduce_max(c, -3), lambda: ew.reduce_max(c, 0.0),
           lambda: ew.reduce_max(c, (0,)), lambda: ew.reduce_max(c[:, :0], 1), lambda: ew.reduce_max(c, 0, use_tf=True),
           lambda: ew.assign_add(c, c[:2]), lambda: ew.assign_add(c, c.half()), lambda: ew.assign_add(c.t(), c.t())]
    for call in bad:
        with pytest.raises(ValueError):
            call()
    assert _lib.last_kernel() == before


def _reference_defs():
    src = os.path.join(os.environ.get("BLOCKSPARSE_REFERENCE") or "/root/reference", "blocksparse", "ewops.py")
    if not os.path.isfile(src):
        pytest.skip("no reference checkout")
    with open(src) as fh:
        tree = ast.parse(fh.read())
    return {f.name: f for f in tree.body if isinstance(f, ast.FunctionDef)}


def test_reference_signatures():
    """Parsed from the reference's ewops.py (not imported: it needs TensorFlow): same parameter names, same defaults."""
    defs = _reference_defs()
    for name in elementwise.__all__:
        f = defs[name]
        params = [a.arg for a in f.args.args]
        defaults = [eval(compile(ast.Expression(d), "<default>", "eval")) for d in f.args.defaults]
        p = inspect.signature(getattr(elementwise, name)).parameters
        assert list(p) == params, name
        ours = [v.default for v in p.values() if v.default is not inspect.Parameter.empty]
        assert ours == defaults, name


def test_names_and_all():
    assert len(set(elementwise.__all__)) == 29
    for name in elementwise.__all__:
        assert getattr(blocksparse_b200, name) is getattr(elementwise, name)
        assert getattr(ewops, name) is getattr(elementwise, name)
        assert name not in blocksparse_b200.__all__
        assert name not in ewops.__all__


UNARY = ["negative", "reciprocal", "square", "sqrt", "exp", "log", "sigmoid", "tanh", "relu", "elu", "gelu", "swish"]
TORCH_UNARY = {
    "negative": torch.neg, "reciprocal": torch.reciprocal, "square": torch.square, "sqrt": torch.sqrt,
    "exp": torch.exp, "log": torch.log, "sigmoid": torch.sigmoid, "tanh": torch.tanh, "relu": torch.relu,
    "elu": lambda x, a: torch.nn.functional.elu(x, a),
    "gelu": lambda x, a: 0.5 * x * (1 + torch.tanh(np.sqrt(2 / np.pi) * (x + a * x ** 3))),
    "swish": lambda x, a: x * torch.sigmoid(a * x),
}


@pytest.mark.parametrize("op", UNARY)
def test_unary_oracle_against_torch_float64_autograd(op):
    rng = np.random.default_rng(0)
    x = rng.normal(0, 2, 200)
    if op in ("sqrt", "log"):
        x = np.abs(x) + 0.1
    dz = rng.normal(0, 1, 200)
    alpha = {"elu": 0.7, "gelu": 0.044715, "swish": 1.702}.get(op)
    t = torch.tensor(x, requires_grad=True)
    z = TORCH_UNARY[op](t, alpha) if alpha is not None else TORCH_UNARY[op](t)
    z.backward(torch.tensor(dz))
    kw = {} if alpha is None else dict(alpha=alpha)
    zr = eo.unary(op, x, **kw)
    np.testing.assert_allclose(zr, z.detach().numpy(), rtol=1e-13, atol=1e-14)
    s = zr if op in eo.Z_GRAD else x
    np.testing.assert_allclose(eo.unary_grad(op, dz, s, **kw), t.grad.numpy(), rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("op", list(eo.BINARY))
def test_binary_oracle_against_torch_float64_autograd(op):
    rng = np.random.default_rng(1)
    x, y, dz = rng.normal(0, 2, (3, 50))
    tx, ty = torch.tensor(x, requires_grad=True), torch.tensor(y, requires_grad=True)
    fn = {"add": torch.add, "subtract": torch.sub, "multiply": torch.mul, "divide": torch.div,
          "maximum": torch.maximum, "minimum": torch.minimum}[op]
    fn(tx, ty).backward(torch.tensor(dz))
    np.testing.assert_allclose(eo.binary(op, x, y), fn(tx, ty).detach().numpy(), rtol=1e-14)
    for got, t in zip(eo.binary_grad(op, dz, x, y), (tx, ty)):
        np.testing.assert_allclose(got, t.grad.numpy(), rtol=1e-14)
    if op in ("maximum", "minimum"):
        # a tie gives dz to both operands (torch splits it)
        dx, dy = eo.binary_grad(op, [2.0], [1.5], [1.5])
        assert dx[0] == 2.0 and dy[0] == 2.0


def test_broadcast_oracle_against_torch_float64_autograd():
    rng = np.random.default_rng(2)
    x, dz = rng.normal(0, 1, (2, 6, 5, 7))
    b = rng.normal(0, 1, 7)
    tx, tb = torch.tensor(x, requires_grad=True), torch.tensor(b, requires_grad=True)
    (tx + tb).backward(torch.tensor(dz))
    np.testing.assert_allclose(eo.bias_add(x, b), x + b)
    dx, db = eo.bias_add_grad(dz, b)
    np.testing.assert_allclose(db, tb.grad.numpy(), rtol=1e-13)
    tx.grad = tb.grad = None
    (tx * tb).backward(torch.tensor(dz))
    dx, dg = eo.gain_mul_grad(dz, x, b)
    np.testing.assert_allclose(dx, tx.grad.numpy(), rtol=1e-14)
    np.testing.assert_allclose(dg, tb.grad.numpy(), rtol=1e-13)


def test_filter_and_gate_oracles():
    x = np.array([1.0, -np.inf, np.inf, np.nan, 3e5, -2.0])
    np.testing.assert_array_equal(eo.filter_tensor(x, 2.0, 65504.0, True, True), [2, 0, 0, 0, 65504, -4])
    np.testing.assert_array_equal(eo.filter_tensor(x, 1.0, 10.0), [1, -10, 10, 10, 10, -2])     # NaN saturates to +10
    assert np.isnan(eo.filter_tensor(x, 0.5)[3]) and eo.filter_tensor(x, 0.5, zero_nans=True)[1] == -np.inf
    # concrete gate: torch float64 autograd of the same formula from the same uniforms
    rng = np.random.default_rng(3)
    loga = rng.normal(0, 2, 300)
    f = eo.concrete_uniform(7, 3, 300)
    assert f.dtype == np.float32 and f.min() >= np.float32(1e-6) and f.max() <= 1 - 1e-6
    gate, c = eo.concrete_gate(loga, f, 0.5, -0.1, 1.1)
    tl = torch.tensor(loga, requires_grad=True)
    tf = torch.tensor(f.astype(np.float64))
    rcp = float(np.float32(1) / np.float32(0.5))
    la, lb = float(np.float32(-0.1)), float(np.float32(1.1))
    tc = torch.sigmoid((torch.log(tf) - torch.log1p(-tf) + tl) * rcp)
    tg = torch.clamp(tc * (lb - la) + la, 0, 1)
    dg = rng.normal(0, 1, 300)
    tg.backward(torch.tensor(dg))
    np.testing.assert_allclose(gate, tg.detach().numpy(), rtol=1e-14, atol=1e-15)
    ref = eo.concrete_gate_grad(dg, c.astype(np.float32), 0.5, -0.1, 1.1)
    inside = (tc.detach().numpy() * (lb - la) + la > 1e-6) & (tc.detach().numpy() * (lb - la) + la < 1 - 1e-6)
    np.testing.assert_allclose(ref[inside], tl.grad.numpy()[inside], rtol=1e-5)
    np.testing.assert_allclose(eo.concrete_gate_infer(loga), np.clip(1 / (1 + np.exp(-loga)) * (lb - la) + la, 0, 1))


def test_gather_and_reduce_max_oracles():
    rng = np.random.default_rng(4)
    x = rng.normal(0, 1, (3, 4, 5, 2))
    idx = np.array([[0, -3, 4, 5], [1, 2, 3, 0], [6, 4, -1, 2]])
    y = eo.fancy_gather(x, idx)
    for a in range(3):
        for b in range(4):
            i = max(idx[a, b], 0)
            np.testing.assert_array_equal(y[a, b], x[a, b, i] if i < 5 else 0)
    tx = torch.tensor(x, requires_grad=True)
    ti = torch.tensor(np.maximum(idx, 0))
    ok = torch.tensor(np.maximum(idx, 0) < 5)
    g = torch.gather(tx, 2, ti.clamp(max=4)[..., None, None].expand(3, 4, 1, 2))[:, :, 0] * ok[..., None]
    dy = rng.normal(0, 1, g.shape)
    g.backward(torch.tensor(dy))
    np.testing.assert_array_equal(eo.fancy_gather_grad(dy, idx, x.shape), tx.grad.numpy())
    # reduce_max: ties to the first, NaN never taken, -inf / NaN slices give (-FLT_MAX, 0)
    x = np.array([[1.0, 3.0, 3.0, np.nan], [np.nan, np.nan, np.nan, np.nan], [-np.inf, -np.inf, -np.inf, -np.inf],
                  [np.nan, -5.0, 2.0, 2.0]])
    m, a = eo.reduce_max(x, 1)
    np.testing.assert_array_equal(m, [3.0, -eo.FLT_MAX, -eo.FLT_MAX, 2.0])
    np.testing.assert_array_equal(a, [1, 0, 0, 2])
    x = rng.normal(0, 1, (3, 6, 4))
    for axis in range(3):
        m, a = eo.reduce_max(x, axis)
        np.testing.assert_array_equal(m, x.max(axis))
        np.testing.assert_array_equal(a, x.argmax(axis))
        tx = torch.tensor(x, requires_grad=True)
        dy = rng.normal(0, 1, m.shape)
        tx.amax(axis).backward(torch.tensor(dy))
        np.testing.assert_array_equal(eo.reduce_max_grad(dy, a, x.shape, axis), tx.grad.numpy())


def test_add_n_oracle_grouping():
    rng = np.random.default_rng(5)
    xs = [rng.normal(0, 1, 10).astype(np.float32) for _ in range(20)]
    got, exact = eo.add_n(xs, "float32")
    np.testing.assert_allclose(got, exact, rtol=0, atol=2e-5)
    # 20 tensors: groups x19..x12, then (s, x11..x5), then (s, x4..x0)
    s = np.zeros(10, np.float32)
    for x in xs[::-1][:8]:
        s = s + x
    for grp in (xs[::-1][8:15], xs[::-1][15:]):
        t = s.copy() * 0
        for x in [s] + grp:
            t = t + x
        s = t
    np.testing.assert_array_equal(got, s)
