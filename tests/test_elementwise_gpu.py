"""The elementwise ops on the GPU: every op and gradient elementwise against the float64 oracle with per-element bounds,
bit for bit where the result is a selection, a copy or a single correctly rounded operation, against the reference's own
kernels, in every execution context, past 2^31 element offsets, and in a two-step LSTM cell.

Bounds. The inputs are given to the oracle as the kernel reads them (16-bit values convert exactly), so every error is
formed on the device. Each fp32 quantity has a relative error of a few u = 2^-24: IEEE add, multiply, division and square
root 1/2 ulp, expf / logf / tanhf / expm1f within 2 ulp (CUDA C Programming Guide, mathematical functions). We allow
64 u times M, the magnitude of the terms that form the result (absolute values, so cancellation is covered, and the
argument of a tanh or sigmoid multiplied by its slope <= 1), then the one rounding to the output, u_out |ref|, plus half
the fp16 subnormal spacing.
"""
import threading

import numpy as np
import pytest
import torch

from blocksparse_b200 import bias_relu, elementwise as el, ewops as ew, fused_lstm_gates, get_entropy, set_entropy, split4
from oracle import elementwise_oracle as eo
from oracle import ref_elementwise as rew

gpu = pytest.mark.gpu
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
U32 = 2.0 ** -24
U_OUT = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
SIZES = [1, 3, 255, 256, 16383, 16384, 10 ** 6 + 3]
SLEEP_CYCLES = 1 << 22
ALPHA = {"elu": 0.7, "gelu": 0.044715, "swish": 1.702}
UNARY = ["negative", "reciprocal", "square", "sqrt", "exp", "log", "sigmoid", "tanh", "relu", "elu", "gelu", "swish"]
BINARY = ["add", "subtract", "multiply", "divide", "maximum", "minimum"]


def _np(t):
    return t.detach().double().cpu().numpy()


def _floor(dtype):
    return 1e-30 + (2.0 ** -25 if dtype == torch.float16 else 0.0)


def _check(got, ref, M, dtype, what, c=64):
    got = _np(got)
    ref = np.asarray(ref, np.float64)
    bound = c * U32 * np.abs(M) + U_OUT[dtype] * np.abs(ref) + _floor(dtype)
    with np.errstate(invalid="ignore"):
        bad = ~(np.abs(got - ref) <= bound) & ~(got == ref)
    assert not bad.any(), "%s: %d elements off, first at %d: got %r ref %r bound %r" % (
        what, bad.sum(), np.argmax(bad), got.reshape(-1)[np.argmax(bad)], ref.reshape(-1)[np.argmax(bad)],
        np.broadcast_to(bound, ref.shape).reshape(-1)[np.argmax(bad)])


def _same(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, what
    assert torch.equal(a.contiguous().view(-1).view(torch.uint8), b.contiguous().view(-1).view(torch.uint8)), what


def _input(op, n, dtype, rng, misaligned=False):
    x = rng.normal(0, 2, n)
    if op in ("sqrt", "log", "reciprocal"):
        x = np.abs(x) + 0.1
    x = np.clip(x, -10, 10)
    t = torch.empty(n + int(misaligned), dtype=dtype, device="cuda")
    t[int(misaligned):] = torch.as_tensor(x, dtype=torch.float32).to(dtype)
    return t[int(misaligned):]


def _unary_M(op, x, z, a):
    x, z = np.abs(x), np.abs(z)
    if op == "gelu":
        return x * (1 + eo.SQRT_2_PI * (x + a * x ** 3))
    if op == "swish":
        return x * (1 + abs(a) * x)
    return z


def _unary_grad_M(op, dz, s, a):
    dz, s = np.abs(dz), np.abs(s)
    if op == "sigmoid":
        return dz * (s + s * s)
    if op == "tanh":
        return dz * (1 + s * s)
    if op == "elu":
        return dz * abs(a) * (1 + np.exp(np.minimum(s, 0)) + np.abs(np.expm1(-s)))
    if op == "gelu":
        return dz * (1 + s * (1 + 3 * a * s * s)) * (1 + eo.SQRT_2_PI * (s + a * s ** 3))
    if op == "swish":
        return dz * (1 + abs(a) * s) ** 2
    return np.abs(eo.unary_grad(op, dz, s, **({"alpha": a} if a is not None else {})))


# ---- unary and binary ops ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("op", UNARY)
def test_unary_forward_and_gradient(op, dtype):
    rng = np.random.default_rng(UNARY.index(op))
    a = ALPHA.get(op)
    kw = {} if a is None else {"alpha": a}
    for n in SIZES:
        for mis in ((False, True) if n >= 16383 else (False,)):
            x = _input(op, n, dtype, rng, mis).requires_grad_()
            dz = _input("", n, dtype, rng, mis)
            z = getattr(ew, op)(x, **kw)
            z.backward(dz)
            xn, dzn = _np(x), _np(dz)
            ref = eo.unary(op, xn, **kw)
            what = "%s %s n=%d misaligned=%s" % (op, dtype, n, mis)
            _check(z, ref, _unary_M(op, xn, ref, a or 0), dtype, what)
            s = _np(z) if op in eo.Z_GRAD else xn
            gref = eo.unary_grad(op, dzn, s, **kw)
            _check(x.grad, gref, _unary_grad_M(op, dzn, s, a or 0), dtype, what + " grad")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("op", BINARY)
def test_binary_forward_and_gradient(op, dtype):
    rng = np.random.default_rng(100 + BINARY.index(op))
    for n in SIZES:
        for mis in ((False, True) if n >= 16383 else (False,)):
            x = _input("", n, dtype, rng, mis)
            y = _input("", n, dtype, rng, mis)
            if op == "divide":
                y = torch.where(y.abs() < 0.1, torch.full_like(y, 0.5), y)
            if op in ("maximum", "minimum"):
                y[::7] = x[::7]                          # ties
            x.requires_grad_()
            y.requires_grad_()
            dz = _input("", n, dtype, rng, mis)
            z = getattr(ew, op)(x, y)
            z.backward(dz)
            xn, yn, dzn = _np(x), _np(y), _np(dz)
            ref = eo.binary(op, xn, yn)
            what = "%s %s n=%d misaligned=%s" % (op, dtype, n, mis)
            _check(z, ref, ref, dtype, what, c=1)
            dxr, dyr = eo.binary_grad(op, dzn, xn, yn)
            _check(x.grad, dxr, dxr, dtype, what + " dx", c=4)
            _check(y.grad, dyr, dyr, dtype, what + " dy", c=4)


@gpu
def test_nan_and_inf_rules():
    x = torch.tensor([1.0, float("nan"), 2.0, float("nan"), -1.0], device="cuda")
    y = torch.tensor([float("nan"), 3.0, 2.0, float("nan"), 0.0], device="cuda")
    assert ew.maximum(x, y).tolist()[:3] == [1.0, 3.0, 2.0] and np.isnan(ew.maximum(x, y)[3].item())
    assert ew.minimum(x, y).tolist()[:3] == [1.0, 3.0, 2.0]
    assert ew.relu(torch.tensor([float("nan"), -0.0, 2.0], device="cuda")).tolist() == [0.0, 0.0, 2.0]


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_two_runs_are_bitwise_identical(dtype):
    rng = np.random.default_rng(7)
    x, dz = (_input("", 70007, dtype, rng) for _ in range(2))
    b = _input("", 70007 // 7, torch.float32, rng)
    outs = []
    for _ in range(2):
        xs = x.reshape(7, -1).clone().requires_grad_()
        bb = b.clone().requires_grad_()
        z = ew.multiply(ew.gelu(ew.add(xs, bb)), bb)
        z.backward(dz.reshape(7, -1))
        outs.append((z, xs.grad, bb.grad))
    for a, r in zip(*outs):
        _same(a, r, "rerun")


# ---- bias-add / gain-mul broadcasts -----------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("bdtype", DTYPES, ids=str)
def test_broadcast_add_and_multiply(dtype, bdtype):
    rng = np.random.default_rng(11)
    for shape, bshape, swap in [((64, 256), (256,), False), ((3, 5, 136), (1, 136), False), ((1000, 33), (33,), True),
                                ((7, 1), (1,), False), ((4096, 24), (1, 1, 24), True)]:
        K = shape[-1]
        N = int(np.prod(shape)) // K
        x = _input("", int(np.prod(shape)), dtype, rng).view(shape).requires_grad_()
        b = _input("", K, bdtype, rng).view(bshape).requires_grad_()
        dz = _input("", x.numel(), dtype, rng).view(shape)
        xn, bn, dzn = _np(x), _np(b), _np(dz)
        what = "%s %s %s b %s" % (shape, dtype, bdtype, bshape)
        # add: db is bitwise bias_relu's db for the same dz
        z = ew.add(b, x) if swap else ew.add(x, b)
        assert z.dtype == dtype and z.shape == x.shape
        z.backward(dz)
        ref = eo.bias_add(xn, bn)
        _check(z, ref, ref, dtype, what + " add", c=1)
        _same(x.grad, dz, what + " add dx")
        x2 = x.detach().clone().requires_grad_()
        b2 = b.detach().reshape(-1).clone().requires_grad_()
        bias_relu(x2, b2).backward(dz)
        _same(b.grad.reshape(-1), b2.grad, what + " db against bias_relu")
        _, dbr = eo.bias_add_grad(dzn, bn)
        _check(b.grad.reshape(-1), dbr, (N + 64) * np.abs(dzn).reshape(N, K).sum(0), bdtype, what + " db", c=1)
        # multiply
        x.grad = b.grad = None
        z = ew.multiply(b, x) if swap else ew.multiply(x, b)
        z.backward(dz)
        ref = eo.gain_mul(xn, bn)
        _check(z, ref, ref, dtype, what + " mul", c=1)
        dxr, dgr = eo.gain_mul_grad(dzn, xn, bn)
        _check(x.grad, dxr, dxr, dtype, what + " mul dx", c=1)
        _check(b.grad.reshape(-1), dgr, (N + 64) * np.abs(dzn * xn).reshape(N, K).sum(0), bdtype, what + " dg", c=2)


@gpu
def test_other_broadcasts_fall_back_to_torch_bitwise():
    rng = np.random.default_rng(12)
    for xs, ys in [((4, 1, 6), (5, 6)), ((4, 6), (4, 1)), ((3, 6), ()), ((2, 3, 6), (3, 6))]:
        x = torch.as_tensor(rng.normal(0, 1, xs), dtype=torch.float32, device="cuda").half()
        y = torch.as_tensor(rng.normal(0, 1, ys), dtype=torch.float32, device="cuda").half()
        for fn, tfn in ((ew.add, torch.add), (ew.multiply, torch.mul), (ew.subtract, torch.sub),
                        (ew.divide, torch.div), (ew.maximum, torch.fmax), (ew.minimum, torch.fmin)):
            _same(fn(x, y), tfn(x, y), "%s %s %s" % (fn.__name__, xs, ys))


# ---- float_cast / filter_tensor ---------------------------------------------------------------------------------------
@gpu
def test_float_cast_every_pair_and_every_16bit_code():
    rng = np.random.default_rng(13)
    wide = np.concatenate([rng.normal(0, 1, 100000) * np.exp2(rng.integers(-140, 120, 100000)),
                           [0.0, -0.0, np.inf, -np.inf, 65504.0, 65520.0, 1e-8, 3e38]]).astype(np.float32)
    codes = torch.arange(65536, dtype=torch.int32, device="cuda").to(torch.int16)
    srcs = {torch.float32: torch.as_tensor(wide, device="cuda"), torch.float16: codes.view(torch.float16),
            torch.bfloat16: codes.view(torch.bfloat16)}
    for sdt, x in srcs.items():
        for ddt in DTYPES:
            for mis in (0, 1):
                xv = x[mis:]
                y = ew.float_cast(xv, ddt)
                if sdt == ddt:
                    assert y is xv
                    continue
                ref = xv.float().to(ddt)                      # through fp32, round to nearest even
                nan = torch.isnan(ref)
                assert torch.equal(torch.isnan(y), nan), (sdt, ddt)
                _same(y[~nan], ref[~nan], "float_cast %s -> %s" % (sdt, ddt))
    x = torch.as_tensor(wide[:1000], device="cuda").requires_grad_()
    y = ew.float_cast(x, torch.float16)
    y.backward(torch.ones_like(y))
    assert x.grad.dtype == torch.float32 and bool((x.grad == 1).all())
    x = torch.as_tensor(wide[:1000], device="cuda").half().requires_grad_()
    y = ew.float_cast(x, torch.float32, dx_dtype=torch.bfloat16)
    dz = torch.as_tensor(rng.normal(0, 1, 1000).astype(np.float32), device="cuda")
    y.backward(dz)
    _same(x.grad, dz.bfloat16().half(), "float_cast dx through dx_dtype")


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_filter_tensor(dtype):
    rng = np.random.default_rng(14)
    base = rng.normal(0, 100, 5000)
    base[::17], base[1::17], base[2::17] = np.inf, -np.inf, np.nan
    x = torch.as_tensor(base, dtype=torch.float32, device="cuda").to(dtype)
    xn = _np(x)
    for kw in (dict(), dict(scale=0.5), dict(saturate=60.0), dict(zero_infs=True), dict(zero_nans=True),
               dict(scale=3.0, saturate=200.0, zero_infs=True, zero_nans=True), dict(saturate=80.0, zero_infs=True)):
        for use_t in (False, True):
            kk = dict(kw)
            if use_t and "scale" in kk:
                kk["scale"] = torch.tensor([kk["scale"]], device="cuda")
            xx = x.clone().requires_grad_()
            y = ew.filter_tensor(xx, **kk)
            ref = eo.filter_tensor(xn, **kw)
            g = _np(y)
            assert np.array_equal(np.isnan(g), np.isnan(ref)), kw
            fin = ~np.isnan(ref)
            assert np.array_equal(g[np.isinf(ref)], ref[np.isinf(ref)]), kw
            fin &= ~np.isinf(ref)
            _check(y[torch.as_tensor(fin, device="cuda")], ref[fin], ref[fin], dtype, "filter %s" % kw, c=1)
            y.backward(x)
            gg = _np(xx.grad)
            assert np.array_equal(np.isnan(gg), np.isnan(ref)) and np.array_equal(gg[fin], g[fin]), kw
    assert ew.scale_tensor(x, 2.0).dtype == dtype


# ---- add_n ------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_add_n_matches_the_reference_grouping(dtype):
    rng = np.random.default_rng(15)
    for count in range(1, 21):
        for n in (3, 4096, 100001):
            xs = [_input("", n, dtype, rng).requires_grad_() for _ in range(count)]
            y = ew.add_n(xs)
            ref, _ = eo.add_n([_np(t) for t in xs], str(dtype).replace("torch.", ""))
            _same(y.detach(), torch.as_tensor(ref, device="cuda").to(dtype), "add_n %d %s n=%d" % (count, dtype, n))
            dz = _input("", n, dtype, rng)
            y.backward(dz)
            for t in xs:
                _same(t.grad, dz, "add_n grad")
        if count <= 8:
            y8 = ew.add_n8(xs)
            ref8 = np.zeros(n, np.float32)
            for t in xs:
                ref8 = ref8 + _np(t).astype(np.float32)
            _same(y8.detach(), torch.as_tensor(ref8, device="cuda").to(dtype), "add_n8 %d" % count)


# ---- concrete gate ----------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_concrete_gate(dtype):
    rng = np.random.default_rng(16)
    n = 300001
    loga = _input("", n, dtype, rng).requires_grad_()
    t, la, lb = 0.5, -0.1, 1.1
    set_entropy(4321, device="cuda")
    g1 = ew.concrete_gate(loga, t, la, lb)
    assert get_entropy().tolist() == [4321, 1]
    g2 = ew.concrete_gate(loga, t, la, lb)
    assert get_entropy().tolist() == [4321, 2] and not torch.equal(g1, g2)
    set_entropy(4321, device="cuda")
    _same(ew.concrete_gate(loga, t, la, lb), g1, "concrete_gate from (seed, call)")
    set_entropy(4321, device="cuda")
    g = ew.concrete_gate(loga, t, la, lb)
    f = eo.concrete_uniform(4321, 0, n).astype(np.float64)
    ln = _np(loga)
    ref, c = eo.concrete_gate(ln, f, t, la, lb)
    rcp = float(np.float32(1) / np.float32(t))
    M = (np.abs(np.log(f)) + np.abs(np.log1p(-f)) + np.abs(ln)) * rcp * (lb - la) + 1
    _check(g, ref, M, dtype, "concrete_gate")
    dg = _input("", n, dtype, rng)
    g.backward(dg)
    st = eo._stretch32(c.astype(np.float32), la, lb).astype(np.float64)
    safe = (np.abs(st) > 1e-4) & (np.abs(st - 1) > 1e-4)
    gref = eo.concrete_gate_grad(_np(dg), c, t, la, lb)
    dgn = np.abs(_np(dg))
    Mg = dgn * (lb - la) * rcp * (c + c * c) * (1 + M)
    _check(loga.grad[torch.as_tensor(safe, device="cuda")], gref[safe], Mg[safe], dtype, "concrete_gate grad")
    inf = ew.concrete_gate_infer(loga.detach(), la, lb)
    iref = eo.concrete_gate_infer(ln, la, lb)
    _check(inf, iref, 1 + np.abs(ln), dtype, "concrete_gate_infer")


@gpu
def test_concrete_gate_statistics_fit_the_hard_concrete_distribution():
    set_entropy(99, device="cuda")
    n, beta, la, lb = 2 * 10 ** 6, 2.0 / 3.0, -0.1, 1.1
    for lv in (-1.0, 0.0, 1.5):
        g = ew.concrete_gate(torch.full((n,), lv, device="cuda"), beta, la, lb).double()
        logit = lambda p: np.log(p / (1 - p))  # noqa: E731
        p0 = 1 / (1 + np.exp(-(beta * logit(-la / (lb - la)) - lv)))
        p1 = 1 - 1 / (1 + np.exp(-(beta * logit((1 - la) / (lb - la)) - lv)))
        assert abs((g == 0).double().mean().item() - p0) < 3e-3, (lv, p0)
        assert abs((g == 1).double().mean().item() - p1) < 3e-3, (lv, p1)
        # the density between: P(gate <= 0.5) = P(concrete <= (0.5 - la) / (lb - la))
        ph = 1 / (1 + np.exp(-(beta * logit((0.5 - la) / (lb - la)) - lv)))
        assert abs((g <= 0.5).double().mean().item() - ph) < 3e-3, (lv, ph)


# ---- fancy_gather / reduce_max ----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dtype", DTYPES + [torch.int32], ids=str)
def test_fancy_gather(dtype):
    rng = np.random.default_rng(17)
    for xshape, r in [((4, 6, 9, 3), 2), ((50, 12), 1), ((5, 7, 2000), 1), ((3, 4, 5), 2)]:
        xv = rng.normal(0, 3, xshape)
        x = torch.as_tensor(xv, device="cuda").to(dtype)
        idx = torch.as_tensor(rng.integers(-2, xshape[r] + 2, xshape[:r]), dtype=torch.int32, device="cuda")
        y = ew.fancy_gather(x.requires_grad_() if dtype != torch.int32 else x, idx)
        ref = eo.fancy_gather(x.detach().cpu().numpy() if dtype != torch.bfloat16 else x.detach().float().cpu().numpy(),
                              idx.cpu().numpy())
        _same(y.detach(), torch.as_tensor(ref, device="cuda").to(dtype), "fancy_gather %s %s" % (xshape, dtype))
        if dtype == torch.int32:
            continue
        dy = torch.as_tensor(rng.normal(0, 1, y.shape), device="cuda").to(dtype)
        y.backward(dy)
        gref = eo.fancy_gather_grad(dy.float().cpu().numpy(), idx.cpu().numpy(), xshape)
        _same(x.grad, torch.as_tensor(gref, device="cuda").to(dtype), "fancy_gather grad %s" % (xshape,))


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_reduce_max_every_axis_ties_and_nan(dtype):
    rng = np.random.default_rng(18)
    xv = rng.integers(-20, 20, (6, 300, 5)).astype(np.float32)       # many ties
    xv[0, :, 0] = np.nan
    xv[1, 7:40, 2] = np.nan
    xv[2, :, :] = -np.inf
    xv[3, 5, 1] = np.inf
    x0 = torch.as_tensor(xv, device="cuda").to(dtype)
    for axis in (0, 1, 2, -1, -2):
        for keep in (False, True):
            x = x0.clone().requires_grad_()
            y = ew.reduce_max(x, axis, keepdims=keep)
            m, a = eo.reduce_max(_np(x0), axis, keepdims=keep)
            what = "reduce_max %s axis %d keep %s" % (dtype, axis, keep)
            _same(y.detach(), torch.as_tensor(m.astype(np.float32), device="cuda").to(dtype), what)
            dy = torch.as_tensor(rng.normal(0, 1, y.shape), device="cuda").to(dtype)
            y.backward(dy)
            gref = eo.reduce_max_grad(dy.float().cpu().numpy(), a, xv.shape, axis)
            _same(x.grad, torch.as_tensor(gref, device="cuda").to(dtype), what + " grad")
    # the index type follows the axis length: uint8 <= 256, uint16 <= 65536, int32 beyond
    assert el._rmax(x0, 6, 300, 5)[1].dtype == torch.uint16
    assert el._rmax(x0, 1800, 1, 5)[1].dtype == torch.uint8
    xl = torch.as_tensor(rng.normal(0, 1, (3, 70000)), device="cuda").to(dtype)
    xl[1, 69999] = 100
    yl = ew.reduce_max(xl.requires_grad_(), -1)
    _same(yl.detach(), xl.detach().float().amax(-1).to(dtype), "reduce_max 70000")
    assert el._rmax(xl.detach(), 3, 70000, 1)[1].dtype == torch.int32
    assert el._rmax(xl.detach(), 3, 70000, 1)[1][1].item() == 69999


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_assign_add(dtype):
    rng = np.random.default_rng(19)
    for n, mis in ((16384, False), (16383, True), (3, False)):
        y = _input("", n, dtype, rng, mis)
        x = _input("", n, dtype, rng, mis)
        ref = (y.float() + x.float()).to(dtype)
        v = y._version
        out = ew.assign_add(y, x)
        assert out is y and y._version > v
        _same(y, ref, "assign_add %s %d" % (dtype, n))


# ---- the reference's kernels ------------------------------------------------------------------------------------------
def _need_ref():
    why = rew.missing()
    if why:
        pytest.skip(why)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_against_the_reference_kernels(dtype):
    """The reference forms div, rcp, sqrt, exp, log and sigmoid with the PTX .approx instructions (relative errors up to
    about 2^-21, lg2 an absolute 2^-22) and its bf16 stores round ties away from zero; it is held to the oracle with
    bounds widened by 2^-18 M and 2^-20 absolute, and one output step more, while ours keeps its own bounds above."""
    _need_ref()
    rng = np.random.default_rng(20)
    for n in (4096, 1001, 20000):
        for op in UNARY + BINARY:
            a = ALPHA.get(op)
            kw = {} if a is None else {"alpha": a}
            x = _input(op, n, dtype, rng)
            y = _input("", n, dtype, rng)
            if op == "divide":
                y = torch.where(y.abs() < 0.1, torch.full_like(y, 0.5), y)
            dz = _input("", n, dtype, rng)
            xn, yn, dzn = _np(x), _np(y), _np(dz)
            what = "reference %s %s n=%d" % (op, dtype, n)
            if op in BINARY:
                z = rew.ew_forward(op, x, y)
                ref = eo.binary(op, xn, yn)
                M = np.abs(ref)
            else:
                z = rew.ew_forward(op, x, **kw)
                ref = eo.unary(op, xn, **kw)
                M = _unary_M(op, xn, ref, a or 0)
            _check(z, ref, 64 * M + 4 * np.abs(ref) * (2 if dtype == torch.bfloat16 else 0) + 16, dtype, what, c=2 ** 6)
            ours = getattr(ew, op)(x, y) if op in BINARY else getattr(ew, op)(x, **kw)
            assert float((ours.float() - z.float()).abs().max()) <= 2 ** -17 * float(np.abs(M).max() + 1) + \
                2 * U_OUT[dtype] * float(np.abs(ref).max()), what
            if op in ("add", "subtract", "negative"):
                continue
            if op in BINARY:
                dx, dy = rew.ew_backward(op, dz, x=x, y=y)
                dxr, dyr = eo.binary_grad(op, dzn, xn, yn)
                _check(dx, dxr, 64 * np.abs(dxr) + 16, dtype, what + " dx", c=64)
                _check(dy, dyr, 64 * np.abs(dyr) + 16, dtype, what + " dy", c=64)
            else:
                s = ours if op in eo.Z_GRAD else x
                sn = _np(s)
                dx = rew.ew_backward(op, dz, x=x, z=ours) if op in eo.Z_GRAD else rew.ew_backward(op, dz, x=x, **kw)
                gref = eo.unary_grad(op, dzn, sn, **kw)
                _check(dx, gref, 64 * _unary_grad_M(op, dzn, sn, a or 0) + 16 * np.abs(dzn), dtype, what + " dx",
                       c=64)
    # bias-add db and gain-mul dx / dg: fp32 vectors, as the ops are registered
    for N, K in ((512, 256), (40, 100)):
        x = _input("", N * K, dtype, rng).view(N, K)
        dz = _input("", N * K, dtype, rng).view(N, K)
        g = _input("", K, torch.float32, rng)
        db = rew.ew_backward("bias_add", dz)
        xx, gg = x.clone().requires_grad_(), g.clone().requires_grad_()
        ew.add(xx, gg).backward(dz)
        tot = (N + 64) * np.abs(_np(dz)).sum(0)
        _check(db, _np(gg.grad), tot, torch.float32, "reference bias-add db", c=2)
        rdx, rdg = rew.ew_backward("gain_mul", dz, x=x, g=g)
        xx.grad = gg.grad = None
        ew.multiply(xx, gg).backward(dz)
        _check(rdx, _np(xx.grad), _np(xx.grad), dtype, "reference gain-mul dx", c=4)
        _check(rdg, _np(gg.grad), (N + 64) * np.abs(_np(dz) * _np(x)).sum(0), torch.float32, "reference dg", c=2)


@gpu
def test_against_the_reference_casts_sums_gates_gathers_and_maxima():
    _need_ref()
    rng = np.random.default_rng(21)
    codes = torch.arange(65536, dtype=torch.int32, device="cuda").to(torch.int16)
    for dt in (torch.float16, torch.bfloat16):
        x = codes.view(dt)
        r = rew.float_cast(x, torch.float32)
        ok = ~torch.isnan(r)
        _same(ew.float_cast(x, torch.float32)[ok], r[ok], "reference upcast %s" % dt)
        w = torch.as_tensor(rng.normal(0, 1, 100000).astype(np.float32), device="cuda")
        r = rew.float_cast(w, dt)
        ours = ew.float_cast(w, dt)
        diff = ours != r
        if dt == torch.float16:
            assert not diff.any()
        else:       # the reference rounds bf16 ties away from zero: only exact ties may differ
            low = w[diff].view(torch.int32) & 0xFFFF
            assert bool((low == 0x8000).all())
    for dt in DTYPES:
        for count in (1, 3, 5, 8):
            xs = [_input("", 4099, dt, rng) for _ in range(count)]
            r = rew.add_n8(xs)
            ours = ew.add_n8(xs)
            diff = ours != r
            if dt == torch.bfloat16:    # its bf16 stores round ties away from zero: only exact ties of the sum differ
                acc = np.zeros(4099, np.float32)
                for t in xs:
                    acc = acc + _np(t).astype(np.float32)
                low = acc.view(np.int32)[diff.cpu().numpy()] & 0xFFFF
                assert (low == 0x8000).all(), "reference add_n8 %d bf16" % count
            else:
                assert not diff.any(), "reference add_n8 %d %s" % (count, dt)
        x = torch.as_tensor(rng.integers(-9, 9, (6, 300, 5)), dtype=torch.float32, device="cuda").to(dt)
        x[0, 3:9, 1] = float("nan")
        for axis in (0, 1, 2):
            ry, ra = rew.reduce_max(x, axis)
            y = ew.reduce_max(x, axis)
            _same(y.reshape(ry.shape), ry, "reference reduce_max %s axis %d" % (dt, axis))
            shape = tuple(x.shape)
            dims = (int(np.prod(shape[:axis])), shape[axis], int(np.prod(shape[axis + 1:])))
            _same(el._rmax(x, *dims)[1], ra, "reference argmax axis %d" % axis)
            dy = _input("", ry.numel(), dt, rng).view(ry.shape)
            xx = x.clone().requires_grad_()
            ew.reduce_max(xx, axis).backward(dy.view(y.shape))
            _same(xx.grad, rew.reduce_max_grad(dy, ra, shape, axis), "reference reduce_max grad axis %d" % axis)
        for xshape, r_ in [((4, 6, 9, 3), 2), ((50, 12), 1), ((5, 7, 700), 1)]:
            x = torch.as_tensor(rng.normal(0, 3, xshape), device="cuda").to(dt)
            idx = torch.as_tensor(rng.integers(-2, xshape[r_] + 2, xshape[:r_]), dtype=torch.int32, device="cuda")
            _same(ew.fancy_gather(x, idx), rew.fancy_gather(x, idx), "reference fancy_gather %s" % (xshape,))
            dy = torch.as_tensor(rng.normal(0, 1, tuple(idx.shape) + xshape[r_ + 1:]), device="cuda").to(dt)
            xx = x.clone().requires_grad_()
            ew.fancy_gather(xx, idx).backward(dy)
            _same(xx.grad, rew.fancy_gather_grad(dy, idx, xshape), "reference fancy_gather grad %s" % (xshape,))
    xi = torch.as_tensor(rng.integers(-100, 100, (8, 5, 3)), dtype=torch.int32, device="cuda")
    ii = torch.as_tensor(rng.integers(-1, 7, (8,)), dtype=torch.int32, device="cuda")
    _same(ew.fancy_gather(xi, ii), rew.fancy_gather(xi, ii), "reference fancy_gather int32")
    # concrete gate: the reference's uniforms are its own, so only the noise-free gate and the gradient compare
    loga = torch.as_tensor(rng.normal(0, 2, 100003).astype(np.float32), device="cuda")
    _check(ew.concrete_gate_infer(loga), _np(rew.concrete_gate_infer(loga)), 1.0, torch.float32,
           "reference concrete_gate_infer", c=2 ** 8)
    set_entropy(5, device="cuda")
    lg = loga.clone().requires_grad_()
    g = ew.concrete_gate(lg, 0.5)
    dg = torch.as_tensor(rng.normal(0, 1, 100003).astype(np.float32), device="cuda")
    g.backward(dg)
    # the concrete values, recovered as the kernel formed them, feed the reference's gradient
    f = eo.concrete_uniform(5, 0, 100003).astype(np.float64)
    _, c = eo.concrete_gate(_np(loga), f, 0.5)
    cf = torch.as_tensor(c.astype(np.float32), device="cuda")
    rd = rew.concrete_gate_grad(dg, cf, 0.5)
    st = eo._stretch32(c.astype(np.float32), -0.1, 1.1)
    safe = torch.as_tensor((np.abs(st) > 1e-4) & (np.abs(st - 1) > 1e-4), device="cuda")
    _check(lg.grad[safe], _np(rd[safe]), np.abs(_np(rd[safe])) + 1e-3 * np.abs(_np(dg[safe])), torch.float32,
           "reference concrete_gate grad", c=2 ** 12)


# ---- execution contexts -----------------------------------------------------------------------------------------------
def _make(seed, device):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(96, 72, generator=g).to(device=device, dtype=torch.bfloat16)
    b = torch.randn(72, generator=g).to(device)
    dz = torch.randn(96, 72, generator=g).to(device=device, dtype=torch.bfloat16)
    s = torch.rand(1, generator=g).to(device) + 0.5
    return x, b, dz, s


def _run_all(x, b, dz, s):
    xx, bb = x.detach().requires_grad_(), b.detach().requires_grad_()
    z = ew.sigmoid(ew.multiply(ew.add(xx, bb), bb))
    z = ew.filter_tensor(z, scale=s, saturate=0.75)
    z = ew.add_n([z, xx, z, xx, z, xx, z, xx, z, xx])
    m = ew.reduce_max(ew.float_cast(z, torch.float32), 0)
    torch.autograd.backward([z, m], [dz, dz[0].float()])
    return z.detach(), m.detach(), xx.grad, bb.grad, ew.concrete_gate_infer(x)


@gpu
def test_side_stream_with_inputs_still_being_written():
    staging = _make(7, "cuda")
    ref = _run_all(*staging)
    bufs = [torch.full_like(t, float("nan")) for t in staging]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for b, t in zip(bufs, staging):
            b.copy_(t)
        out = _run_all(*bufs)
    s.synchronize()
    for a, r in zip(out, ref):
        _same(a, r, "side stream")


@gpu
def test_graph_replay_with_new_inputs():
    static = _make(0, "cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _run_all(*static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = _run_all(*static)
    for i in range(1, 4):
        new = _make(i, "cuda")
        for t, n in zip(static, new):
            t.copy_(n)
        graph.replay()
        for a, r in zip(out, _run_all(*new)):
            _same(a, r, "replay %d" % i)


@gpu
def test_two_host_threads():
    ins = [_make(10 + i, "cuda") for i in range(2)]
    refs = [_run_all(*x) for x in ins]
    results, errors = [None, None], []

    def worker(i):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                for _ in range(3):
                    results[i] = _run_all(*ins[i])
                torch.cuda.current_stream().synchronize()
        except Exception as e:                       # noqa: BLE001  (re-raised in the main thread)
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for i in range(2):
        for a, r in zip(results[i], refs[i]):
            _same(a, r, "thread %d" % i)


@gpu
def test_second_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    ref = _run_all(*_make(5, "cuda:0"))
    out = _run_all(*_make(5, "cuda:1"))
    for a, r in zip(out, ref):
        assert a.device == torch.device("cuda:1")
        _same(a.to("cuda:0"), r, "cuda:1")
    set_entropy(3, device="cuda:1")
    g = ew.concrete_gate(torch.zeros(1000, device="cuda:1"))
    assert g.device == torch.device("cuda:1") and get_entropy("cuda:1").tolist() == [3, 1]


# ---- offsets past 2^31 ------------------------------------------------------------------------------------------------
@gpu
def test_offsets_past_2_31_on_bf16():
    n = 2 ** 31 + 4099
    x = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    x[:2 ** 20] = torch.randn(2 ** 20, device="cuda").bfloat16()
    x[-2 ** 20:] = torch.randn(2 ** 20, device="cuda").bfloat16()
    x[2 ** 20:-2 ** 20] = 0.25
    z = ew.sigmoid(x)
    for sl in (slice(0, 2 ** 20), slice(n - 2 ** 20, n)):
        _check(z[sl], eo.unary("sigmoid", _np(x[sl])), eo.unary("sigmoid", _np(x[sl])), torch.bfloat16, "2^31 sigmoid")
    dx = el._bwd(x, el.SIG_OP, z)          # dz = x, s = z
    sl = slice(n - 2 ** 20, n)
    ref = eo.unary_grad("sigmoid", _np(x[sl]), _np(z[sl]))
    _check(dx[sl], ref, np.abs(_np(x[sl])) * 2, torch.bfloat16, "2^31 sigmoid grad")
    del dx, z
    K = 4096
    xm = x[:(n // K) * K].view(-1, K)
    xm[-1, 1000] = 50.0
    y = ew.reduce_max(xm, -1)
    assert y[-1].item() == 50.0 and y[0].item() == xm[0].float().max().item()
    y = ew.add(xm, torch.ones(K, device="cuda"))
    _same(y[-3:], (xm[-3:].float() + 1).bfloat16(), "2^31 bias-add")


# ---- a two-step LSTM cell ---------------------------------------------------------------------------------------------
@gpu
def test_two_step_lstm_cell_against_fused_lstm_gates():
    rng = np.random.default_rng(22)
    N, K = 64, 96
    hs = [torch.as_tensor(rng.normal(0, 1.5, (N, 4 * K)).astype(np.float32), device="cuda") for _ in range(2)]
    b = torch.as_tensor(rng.normal(0, 0.5, 4 * K).astype(np.float32), device="cuda")
    c0 = torch.as_tensor(rng.normal(0, 1, (N, K)).astype(np.float32), device="cuda")
    ec = torch.as_tensor(rng.normal(0, 1, (N, K)).astype(np.float32), device="cuda")

    def composed(c, h, bias):
        i, u, f, o = split4(ew.add(h, bias))
        c = ew.add(ew.multiply(ew.sigmoid(f), c), ew.multiply(ew.sigmoid(i), ew.tanh(u)))
        return c, ew.multiply(ew.sigmoid(o), ew.tanh(c))

    outs = []
    for step in (composed, lambda c, h, bias: fused_lstm_gates(c, h, bias=bias, forget_bias=0.0)):
        ins = [t.clone().requires_grad_() for t in [c0, b] + hs]
        c, bb = ins[0], ins[1]
        for h in ins[2:]:
            c, hn = step(c, h, bb)
        torch.autograd.backward([c, hn], [ec, ec])
        outs.append([c.detach(), hn.detach()] + [t.grad for t in ins])
    for a, r, what in zip(outs[0], outs[1], ("c", "h", "dc0", "db", "dh0", "dh1")):
        err = float((a - r).abs().max())
        assert err <= 1e-5 * max(1.0, float(r.abs().max())), (what, err)
