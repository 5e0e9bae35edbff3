"""Elementwise math, casts, filters, sums, concrete gates, gathers and column maxima -- host side of the rest of the
reference's blocksparse/ewops.py (binary ops :69-95, unary ops :97-114, their gradients :116-156, filter_tensor /
scale_tensor :158-172, float_cast :178-204, concrete_gate :244-265, add_n8 / add_n :268-292, fancy_gather :352-386,
reduce_max :389-419, assign_add :423-424), on torch tensors, calling the sm_90a kernels of csrc/elementwise.cuh.

Every op takes CUDA tensors of fp32, fp16 or bf16 (fancy_gather also int32), forms its values in fp32 with accurate
math and rounds each output once; there is no CPU path. Argument errors raise ValueError before anything is launched.
The reference's replace_add_n / restore_add_n patch TensorFlow and are not carried here.
"""
import numbers

import numpy as np
import torch

from . import _lib
from .ewops import ACT_NONE, _br_bwd, get_entropy
from .transformer import _on_device_of

__all__ = ["add", "subtract", "multiply", "divide", "maximum", "minimum", "negative", "reciprocal", "square", "sqrt",
           "exp", "log", "sigmoid", "tanh", "relu", "elu", "gelu", "swish", "fast_gelu", "filter_tensor",
           "scale_tensor", "float_cast", "concrete_gate", "concrete_gate_infer", "add_n8", "add_n", "fancy_gather",
           "reduce_max", "assign_add"]

(ADD_OP, SUB_OP, MUL_OP, DIV_OP, MAXIMUM_OP, MINIMUM_OP, NEG_OP, RCP_OP, SQR_OP, SQRT_OP, EXP_OP, LOG_OP, SIG_OP,
 TANH_OP, RELU_OP, ELU_OP, GELU_OP, SWISH_OP, BIASADD_OP, GAINMUL_OP) = range(20)
_Z_GRAD_OPS = (SIG_OP, TANH_OP, RELU_OP)         # gradients formed from the output z (reference ewops.py:140)
_FLOATS = (torch.float32, torch.float16, torch.bfloat16)


def _dt(t):
    return _lib.dtype_code(t.dtype)


def _cuda(t, what, dtypes=_FLOATS):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise ValueError("%s needs CUDA tensors (there is no CPU path)" % what)
    if t.dtype not in dtypes:
        raise ValueError("%s: unsupported dtype %s (%s only)" % (what, t.dtype, ", ".join(str(d) for d in dtypes)))
    return t


def _same_device(what, *ts):
    for t in ts[1:]:
        if t.device != ts[0].device:
            raise ValueError("%s: operands live on different devices (%s and %s)" % (what, ts[0].device, t.device))


def _number(what, name, v):
    if not isinstance(v, numbers.Real) or isinstance(v, bool):
        raise ValueError("%s: %s must be a Python number, got %r" % (what, name, v))
    return float(v)


# ---- launches ---------------------------------------------------------------------------------------------------------
@_on_device_of
def _fwd(x, op, y=None, b=None, K=0, alpha=1.0, out=None):
    z = torch.empty_like(x) if out is None else out
    if x.numel():
        rc = _lib.load().bsmm_ew_forward(_dt(x), _lib.F32 if b is None else _dt(b), op, x.data_ptr(), _lib.ptr(y),
                                         _lib.ptr(b), z.data_ptr(), x.numel(), K, alpha, _lib.stream_ptr())
        _lib.check(rc, "bsmm_ew_forward")
    return z


@_on_device_of
def _bwd(dz, op, s, y=None, alpha=1.0):
    """dx, or (dx, dy) for the binary ops; s is x, or z for _Z_GRAD_OPS."""
    dx = torch.empty_like(dz)
    dy = torch.empty_like(dz) if y is not None else None
    if dz.numel():
        rc = _lib.load().bsmm_ew_backward(_dt(dz), op, dz.data_ptr(), s.data_ptr(), _lib.ptr(y), dx.data_ptr(),
                                          _lib.ptr(dy), dz.numel(), alpha, _lib.stream_ptr())
        _lib.check(rc, "bsmm_ew_backward")
    return dx if y is None else (dx, dy)


@_on_device_of
def _gain_mul_grad(dz, x, g, N, K):
    dx, dg = torch.empty_like(dz), torch.empty_like(g)
    if N == 0:
        return dx, dg.zero_()
    ws = torch.empty(_lib.load().bsmm_bias_grad_workspace_bytes(1, N, K) // 4, dtype=torch.float32, device=dz.device)
    rc = _lib.load().bsmm_gain_mul_grad(_dt(dz), _dt(g), dz.data_ptr(), x.data_ptr(), g.data_ptr(), dx.data_ptr(),
                                        dg.data_ptr(), ws.data_ptr(), N, K, _lib.stream_ptr())
    _lib.check(rc, "bsmm_gain_mul_grad")
    return dx, dg


@_on_device_of
def _cast(x, dtype):
    y = torch.empty(x.shape, dtype=dtype, device=x.device)
    if x.numel():
        rc = _lib.load().bsmm_float_cast(_dt(x), _lib.dtype_code(dtype), x.data_ptr(), y.data_ptr(), x.numel(),
                                         _lib.stream_ptr())
        _lib.check(rc, "bsmm_float_cast")
    return y


@_on_device_of
def _filter(x, scale, scale_t, saturate, zero_infs, zero_nans):
    y = torch.empty_like(x)
    if x.numel():
        rc = _lib.load().bsmm_filter_tensor(_dt(x), x.data_ptr(), y.data_ptr(), x.numel(), scale, _lib.ptr(scale_t),
                                            saturate, int(zero_infs), int(zero_nans), _lib.stream_ptr())
        _lib.check(rc, "bsmm_filter_tensor")
    return y


@_on_device_of
def _add_n(x0, xs):
    y = torch.empty_like(x0)
    if x0.numel():
        rc = _lib.load().bsmm_add_n(_dt(x0), _lib.ptr_array(xs), len(xs), y.data_ptr(), x0.numel(), _lib.stream_ptr())
        _lib.check(rc, "bsmm_add_n")
    return y


# ---- binary and unary ops ---------------------------------------------------------------------------------------------
class _BinaryFunction(torch.autograd.Function):
    """z = op(x, y), same shapes. add gives (dz, dz), sub (dz, -dz); the others read x and y (reference
    ewops.py:116-127)."""

    @staticmethod
    def forward(ctx, op, x, y):
        ctx.op = op
        if op not in (ADD_OP, SUB_OP):
            ctx.save_for_backward(x, y)
        return _fwd(x, op, y)

    @staticmethod
    def backward(ctx, dz):
        dz = dz.contiguous()
        if ctx.op == ADD_OP:
            return None, dz, dz
        if ctx.op == SUB_OP:
            return None, dz, _fwd(dz, NEG_OP)
        x, y = ctx.saved_tensors
        return (None,) + _bwd(dz, ctx.op, x, y)


class _BroadcastFunction(torch.autograd.Function):
    """z = x + b or x * g with a vector of x's last dim, read as fp32. db is bias_relu's fixed-order column sum of dz
    (bitwise its db); dg the same partition over dz * x (reference ewops.py:145-156)."""

    @staticmethod
    def forward(ctx, op, x, b):
        K = x.shape[-1]
        ctx.op, ctx.NK = op, (x.numel() // K if K else 0, K)
        ctx.save_for_backward(x if op == GAINMUL_OP else None, b)
        return _fwd(x, op, None, b.reshape(-1), K)

    @staticmethod
    def backward(ctx, dz):
        x, b = ctx.saved_tensors
        N, K = ctx.NK
        dz = dz.contiguous()
        bf = b.reshape(-1)
        if ctx.op == BIASADD_OP:
            if K == 0:
                return None, dz, torch.zeros_like(b)
            return None, dz, _br_bwd(dz.view(N, K), None, bf, 1, N, K, ACT_NONE)[1].view(b.shape)
        if K == 0:
            return None, torch.empty_like(dz), torch.zeros_like(b)
        dx, dg = _gain_mul_grad(dz, x, bf, N, K)
        return None, dx, dg.view(b.shape)


def _binary(x, y, op, bc_op, torch_op, what):
    for t in (x, y):
        _cuda(t, what)
    _same_device(what, x, y)
    if x.shape == y.shape:
        if x.dtype != y.dtype:
            raise ValueError("%s: x and y of one shape must share one dtype, got %s and %s" % (what, x.dtype, y.dtype))
        return _BinaryFunction.apply(op, x.contiguous(), y.contiguous())
    if bc_op is not None and x.dim() and y.dim() and x.shape[-1] == y.shape[-1] and x.shape[-1] < 2 ** 31:
        if y.numel() == y.shape[-1]:
            return _BroadcastFunction.apply(bc_op, x.contiguous(), y.contiguous())
        if x.numel() == x.shape[-1]:
            return _BroadcastFunction.apply(bc_op, y.contiguous(), x.contiguous())
    return torch_op(x, y)


_BINARY_DOC = """z = x {sym} y (reference ewops.py:{line}), differentiable in x and y.

    x and y: CUDA tensors of fp32 / fp16 / bf16 on one device. Of one shape (and then one dtype) they run one
    elementwise kernel, formed in fp32 and rounded once.{bcast} Any other pair of shapes falls back to torch.{torch}(x, y),
    as the reference falls back to TensorFlow. `name` is accepted and ignored."""
_BCAST_DOC = """ When one operand is a vector as long as the other's last dim (shape (K,),
    (1, K), ...), the {what} kernel adds it along that dim: the vector is read as fp32 in any of the three dtypes, z
    has the other operand's dtype, and the vector's gradient is a fixed-order column sum, bitwise reproducible{db}."""


def add(x, y, name=None):
    return _binary(x, y, ADD_OP, BIASADD_OP, torch.add, "add")


def multiply(x, y, name=None):
    return _binary(x, y, MUL_OP, GAINMUL_OP, torch.mul, "multiply")


def subtract(x, y, name=None):
    return _binary(x, y, SUB_OP, None, torch.sub, "subtract")


def divide(x, y, name=None):
    return _binary(x, y, DIV_OP, None, torch.div, "divide")


def maximum(x, y, name=None):
    return _binary(x, y, MAXIMUM_OP, None, torch.fmax, "maximum")


def minimum(x, y, name=None):
    return _binary(x, y, MINIMUM_OP, None, torch.fmin, "minimum")


add.__doc__ = _BINARY_DOC.format(sym="+", line=90, torch="add", bcast=_BCAST_DOC.format(
    what="bias-add", db=" and bitwise bias_relu's db for the same dz"))
multiply.__doc__ = _BINARY_DOC.format(sym="*", line=91, torch="mul", bcast=_BCAST_DOC.format(what="gain-mul", db=""))
subtract.__doc__ = _BINARY_DOC.format(sym="-", line=92, torch="sub", bcast="")
divide.__doc__ = _BINARY_DOC.format(sym="/", line=93, torch="div", bcast="") + """

    The quotient is an IEEE fp32 division (the reference multiplies by an approximate reciprocal)."""
maximum.__doc__ = """z = max(x, y) elementwise (reference ewops.py:94), as fmaxf: a NaN operand gives the other one. The
    gradient gives dz to every operand equal to z (both on a tie). Shapes, dtypes and the torch.fmax fallback as in
    subtract."""
minimum.__doc__ = """z = min(x, y) elementwise (reference ewops.py:95), as fminf; otherwise as maximum."""


class _UnaryFunction(torch.autograd.Function):
    """Saves z for sigmoid, tanh and relu, x for the others, nothing for negative (reference ewops.py:129-143)."""

    @staticmethod
    def forward(ctx, op, alpha, x):
        z = _fwd(x, op, None, None, 0, alpha)
        ctx.op, ctx.alpha = op, alpha
        if op != NEG_OP:
            ctx.save_for_backward(z if op in _Z_GRAD_OPS else x)
        return z

    @staticmethod
    def backward(ctx, dz):
        dz = dz.contiguous()
        if ctx.op == NEG_OP:
            return None, None, _fwd(dz, NEG_OP)
        s, = ctx.saved_tensors
        return None, None, _bwd(dz, ctx.op, s, None, ctx.alpha)


def _unary(x, op, what, alpha=1.0):
    _cuda(x, what)
    return _UnaryFunction.apply(op, _number(what, "alpha", alpha), x.contiguous())


def negative(x, name=None):
    """z = -x (reference ewops.py:97); its gradient is -dz."""
    return _unary(x, NEG_OP, "negative")


def reciprocal(x, name=None):
    """z = 1 / x as an IEEE fp32 division (reference ewops.py:98); dx = -dz / x^2."""
    return _unary(x, RCP_OP, "reciprocal")


def square(x, name=None):
    """z = x^2 (reference ewops.py:99); dx = 2 dz x."""
    return _unary(x, SQR_OP, "square")


def sqrt(x, name=None):
    """z = sqrt(x), IEEE fp32 (reference ewops.py:100); dx = dz / (2 sqrt(x))."""
    return _unary(x, SQRT_OP, "sqrt")


def exp(x, name=None):
    """z = exp(x) with expf (reference ewops.py:101); dx = dz exp(x), recomputed from x."""
    return _unary(x, EXP_OP, "exp")


def log(x, name=None):
    """z = log(x) with logf (reference ewops.py:102); dx = dz / x."""
    return _unary(x, LOG_OP, "log")


def sigmoid(x, name=None):
    """z = 1 / (1 + exp(-x)) (reference ewops.py:103); the gradient reads z: dx = dz (z - z^2)."""
    return _unary(x, SIG_OP, "sigmoid")


def tanh(x, name=None):
    """z = tanh(x) with tanhf (reference ewops.py:104); the gradient reads z: dx = dz (1 - z^2)."""
    return _unary(x, TANH_OP, "tanh")


def relu(x, name=None):
    """z = max(x, 0), a NaN giving 0 (reference ewops.py:105); the gradient reads z: dx = dz where z > 0, else 0."""
    return _unary(x, RELU_OP, "relu")


def elu(x, alpha=1.0, name=None):
    """z = x for x > 0, else alpha (exp(x) - 1), with expm1f (reference ewops.py:109); dx = dz, else dz alpha exp(x)."""
    return _unary(x, ELU_OP, "elu", alpha)


def gelu(x, alpha=0.044715, name=None):
    """z = x (1 + tanh(sqrt(2 / pi) (x + alpha x^3))) / 2 (reference ewops.py:110), and its exact derivative."""
    return _unary(x, GELU_OP, "gelu", alpha)


def swish(x, alpha=1.0, name=None):
    """z = x sigmoid(alpha x) (reference ewops.py:111); dx = dz (s + alpha x s (1 - s)), s = sigmoid(alpha x)."""
    return _unary(x, SWISH_OP, "swish", alpha)


def fast_gelu(x, name=None):
    """swish(x, alpha=1.702) (reference ewops.py:113-114)."""
    return swish(x, alpha=1.702, name=name)


# ---- filter_tensor / scale_tensor -------------------------------------------------------------------------------------
class _FilterFunction(torch.autograd.Function):
    """The gradient is the same filter applied to dy (reference ewops.py:170-172)."""

    @staticmethod
    def forward(ctx, x, scale, scale_t, saturate, zero_infs, zero_nans):
        ctx.args = (scale, saturate, zero_infs, zero_nans)
        ctx.save_for_backward(scale_t)
        return _filter(x, scale, scale_t, saturate, zero_infs, zero_nans)

    @staticmethod
    def backward(ctx, dy):
        scale, saturate, zero_infs, zero_nans = ctx.args
        scale_t, = ctx.saved_tensors
        return _filter(dy.contiguous(), scale, scale_t, saturate, zero_infs, zero_nans), None, None, None, None, None


def filter_tensor(x, scale=1.0, saturate=0.0, zero_infs=False, zero_nans=False):
    """y = saturate(scale * x) with infs and / or NaNs first set to 0 (reference ewops.py:158-164), in fp32 and rounded
    once; differentiable in x, whose gradient is the same filter applied to dy.

    scale: a Python number, or a one-element fp32 CUDA tensor on x's device, read on the device when the kernel runs (so
    a captured CUDA graph uses its value at replay). saturate: a Python number; nonzero clamps to [-saturate, saturate]
    with fminf / fmaxf, so a NaN that zero_nans did not remove becomes +saturate, as in the reference (65504 saturates
    fp16 infinities)."""
    _cuda(x, "filter_tensor")
    scale_t = None
    if torch.is_tensor(scale):
        if scale.dtype != torch.float32 or scale.numel() != 1 or scale.device != x.device:
            raise ValueError("filter_tensor: a tensor scale must be one fp32 element on %s, got %s %s on %s" %
                             (x.device, tuple(scale.shape), scale.dtype, scale.device))
        scale_t, scale = scale.reshape(1).contiguous(), 1.0
    else:
        scale = _number("filter_tensor", "scale", scale)
    saturate = _number("filter_tensor", "saturate", saturate)
    return _FilterFunction.apply(x.contiguous(), scale, scale_t, saturate, bool(zero_infs), bool(zero_nans))


def scale_tensor(x, scale=1.0):
    """filter_tensor(x, scale) (reference ewops.py:167-168)."""
    return filter_tensor(x, scale)


# ---- float_cast -------------------------------------------------------------------------------------------------------
class _FloatCastFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dtype, dx_dtype):
        ctx.dx_dtype = dx_dtype
        return _cast(x, dtype)

    @staticmethod
    def backward(ctx, dz):
        dz = dz.contiguous()
        return (dz if dz.dtype == ctx.dx_dtype else _cast(dz, ctx.dx_dtype)), None, None


def float_cast(x, dtype, dx_dtype=None, name=None):
    """x converted to `dtype` (reference ewops.py:178-204): any pair among fp32 / fp16 / bf16, through fp32 and rounded
    once to nearest even; x itself when it already has that dtype. The gradient is dz converted to dx_dtype (default:
    x's dtype), or dz itself when it has that dtype; torch autograd then hands x.grad over in x's dtype."""
    _cuda(x, "float_cast")
    if dtype not in _FLOATS:
        raise ValueError("float_cast: dtype must be float32, float16 or bfloat16, got %r" % (dtype,))
    if dx_dtype is not None and dx_dtype not in _FLOATS:
        raise ValueError("float_cast: dx_dtype must be float32, float16 or bfloat16, got %r" % (dx_dtype,))
    if dtype == x.dtype:
        return x
    return _FloatCastFunction.apply(x.contiguous(), dtype, x.dtype if dx_dtype is None else dx_dtype)


# ---- concrete gate ----------------------------------------------------------------------------------------------------
def _gate_limits(what, limit_a, limit_b):
    la, lb = _number(what, "limit_a", limit_a), _number(what, "limit_b", limit_b)
    if not np.float32(la) < np.float32(lb):
        raise ValueError("%s: limit_a %r must be below limit_b %r" % (what, limit_a, limit_b))
    return la, lb


@_on_device_of
def _gate_fwd(loga, rcp, la, lb, eps):
    gate = torch.empty_like(loga)
    concrete = torch.empty(loga.shape, dtype=torch.float32, device=loga.device)
    if loga.numel():
        state = get_entropy(loga.device)
        rc = _lib.load().bsmm_concrete_gate(_dt(loga), loga.data_ptr(), gate.data_ptr(), concrete.data_ptr(),
                                            loga.numel(), rcp, la, lb, eps, state.data_ptr(), _lib.stream_ptr())
        _lib.check(rc, "bsmm_concrete_gate")
    return gate, concrete


@_on_device_of
def _gate_bwd(dg, concrete, rcp, la, lb):
    dloga = torch.empty_like(dg)
    if dg.numel():
        rc = _lib.load().bsmm_concrete_gate_grad(_dt(dg), dg.data_ptr(), concrete.data_ptr(), dloga.data_ptr(),
                                                 dg.numel(), rcp, la, lb, _lib.stream_ptr())
        _lib.check(rc, "bsmm_concrete_gate_grad")
    return dloga


class _ConcreteGateFunction(torch.autograd.Function):
    """Saves the fp32 concrete values; the gradient flows through them (reference ewops.py:258-265)."""

    @staticmethod
    def forward(ctx, loga, rcp, la, lb, eps):
        gate, concrete = _gate_fwd(loga, rcp, la, lb, eps)
        ctx.args = (rcp, la, lb)
        ctx.save_for_backward(concrete)
        return gate

    @staticmethod
    def backward(ctx, dg):
        concrete, = ctx.saved_tensors
        return _gate_bwd(dg.contiguous(), concrete, *ctx.args), None, None, None, None


def concrete_gate(loga, tempurature=2.0 / 3.0, limit_a=-0.1, limit_b=1.1, epsilon=1e-6):
    """A hard-concrete (L0) gate sample per element of loga (reference ewops.py:250-253; the parameter keeps the
    reference's spelling), differentiable in loga:
        f = u (1 - 2 epsilon) + epsilon,  c = sigmoid((log f - log(1 - f) + loga) / tempurature),
        gate = clamp(c (limit_b - limit_a) + limit_a, 0, 1).
    u is uniform in [0, 1): word e % 4 of Philox4x32-10 keyed by this device's seed at counter (e / 4, call), the state
    dropout draws from (set_entropy / get_entropy); each call advances call by one on the device, so a sample depends on
    (seed, call, loga) only and a captured graph draws a new one at every replay. The reference draws from its own
    Tausworthe buffer instead, so its samples are not these. The gradient flows through c, saved in fp32:
    dloga = dgate (limit_b - limit_a) c (1 - c) / tempurature where the stretch lies in [0, 1], else 0.

    loga: CUDA, fp32 / fp16 / bf16 (the gate comes back in that dtype). The other arguments: Python numbers, with
    tempurature > 0, limit_a < limit_b and 0 <= epsilon < 0.5."""
    what = "concrete_gate"
    _cuda(loga, what)
    t = _number(what, "tempurature", tempurature)
    if not t > 0:
        raise ValueError("concrete_gate: tempurature must be positive, got %r" % (tempurature,))
    la, lb = _gate_limits(what, limit_a, limit_b)
    eps = _number(what, "epsilon", epsilon)
    if not 0 <= eps < 0.5:
        raise ValueError("concrete_gate: epsilon must be in [0, 0.5), got %r" % (epsilon,))
    rcp = float(np.float32(1) / np.float32(t))
    return _ConcreteGateFunction.apply(loga.contiguous(), rcp, la, lb, eps)


def concrete_gate_infer(loga, limit_a=-0.1, limit_b=1.1):
    """gate = clamp(sigmoid(loga) (limit_b - limit_a) + limit_a, 0, 1), the noise-free gate (reference
    ewops.py:255-256); not differentiable, as in the reference."""
    what = "concrete_gate_infer"
    _cuda(loga, what)
    la, lb = _gate_limits(what, limit_a, limit_b)
    loga = loga.contiguous()
    return _gate_infer(loga, la, lb)


@_on_device_of
def _gate_infer(loga, la, lb):
    gate = torch.empty_like(loga)
    if loga.numel():
        rc = _lib.load().bsmm_concrete_gate_infer(_dt(loga), loga.data_ptr(), gate.data_ptr(), loga.numel(), la, lb,
                                                  _lib.stream_ptr())
        _lib.check(rc, "bsmm_concrete_gate_infer")
    return gate


# ---- add_n8 / add_n ---------------------------------------------------------------------------------------------------
class _AddNFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *xs):
        ctx.n = len(xs)
        return _add_n(xs[0], xs)

    @staticmethod
    def backward(ctx, dz):
        return (dz,) * ctx.n


def add_n8(xs, name="AddN"):
    """The sum of 1 to 8 tensors of one shape, dtype and device in one launch (reference ewops.py:272-274): added in
    fp32 in list order, starting from +0, and rounded once. Every input receives dz."""
    xs = list(xs)
    if not 1 <= len(xs) <= 8:
        raise ValueError("add_n8 takes 1 to 8 tensors, got %d" % len(xs))
    for t in xs:
        _cuda(t, "add_n8")
    if any(t.shape != xs[0].shape or t.dtype != xs[0].dtype or t.device != xs[0].device for t in xs):
        raise ValueError("add_n8: the tensors must share one shape, dtype and device, got %s" %
                         [(tuple(t.shape), t.dtype, t.device) for t in xs])
    return _AddNFunction.apply(*[t.contiguous() for t in xs])


def add_n(xs, name="AddN"):
    """The sum of any number of tensors of one shape, dtype and device (reference ewops.py:276-292), grouped exactly as
    the reference groups them: one tensor is returned as it is; two are one add; more are taken from the end of the list,
    8 at a time, each group after the first led by the previous group's sum:
        add_n8([x[-1], ..., x[-8]]), then add_n8([s, x[-9], ..., x[-15]]), ...
    so the result is rounded to the dtype once per group of add_n8, at the points this grouping gives. Every input
    receives dz."""
    xs = list(xs)
    if not xs:
        raise ValueError("add_n needs at least one tensor")
    if len(xs) == 1:
        return xs[0]
    if len(xs) == 2:
        for t in xs:
            _cuda(t, "add_n")
        _same_device("add_n", *xs)
        if xs[0].shape != xs[1].shape or xs[0].dtype != xs[1].dtype:
            raise ValueError("add_n: the tensors must share one shape and dtype, got %s" %
                             [(tuple(t.shape), t.dtype) for t in xs])
        return _BinaryFunction.apply(ADD_OP, xs[0].contiguous(), xs[1].contiguous())
    rest = xs[::-1]                      # taken from the end of the list
    total = add_n8(rest[:8])
    for i in range(8, len(rest), 7):
        total = add_n8([total] + rest[i:i + 7])
    return total


# ---- fancy_gather -----------------------------------------------------------------------------------------------------
@_on_device_of
def _gather(x, idx, d0, d1, d2, out_shape):
    y = torch.empty(out_shape, dtype=x.dtype, device=x.device)
    if d0 * d2:
        rc = _lib.load().bsmm_fancy_gather(x.element_size(), x.data_ptr(), idx.data_ptr(), y.data_ptr(), d0, d1, d2,
                                           _lib.stream_ptr())
        _lib.check(rc, "bsmm_fancy_gather")
    return y


@_on_device_of
def _gather_grad(dy, idx, d0, d1, d2, x_shape):
    dx = torch.empty(x_shape, dtype=dy.dtype, device=dy.device)
    if d0 * d1 * d2:
        rc = _lib.load().bsmm_fancy_gather_grad(dy.element_size(), dy.data_ptr(), idx.data_ptr(), dx.data_ptr(), d0, d1,
                                                d2, _lib.stream_ptr())
        _lib.check(rc, "bsmm_fancy_gather_grad")
    return dx


class _FancyGatherFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, idx, dims, out_shape):
        ctx.args = (dims, tuple(x.shape))
        ctx.save_for_backward(idx)
        return _gather(x, idx, *dims, out_shape)

    @staticmethod
    def backward(ctx, dy):
        dims, x_shape = ctx.args
        idx, = ctx.saved_tensors
        return _gather_grad(dy.contiguous(), idx, *dims, x_shape), None, None, None


def fancy_gather(x, idx, use_tf=False):
    """y[i..., :] = x[i..., max(idx[i...], 0), :] (reference ewops.py:357-381): idx indexes the dim of x after idx's
    dims, whose leading dims it shares. A negative index reads row 0 and an index >= that dim reads 0, as the reference
    kernel does. y has shape idx.shape + x.shape[idx.dim() + 1:], and its values are x's bit for bit. Differentiable in
    x: dx holds dy at the gathered rows and 0 elsewhere.

    x: CUDA, fp32 / fp16 / bf16 / int32 (no gradient for int32), of higher rank than idx; any trailing size (the
    reference's kernel takes at most 1024). idx: CUDA int32. use_tf=True raises ValueError."""
    if use_tf:
        raise ValueError("fancy_gather: use_tf is a TensorFlow composition; there is none here")
    _cuda(x, "fancy_gather", _FLOATS + (torch.int32,))
    _cuda(idx, "fancy_gather", (torch.int32,))
    _same_device("fancy_gather", x, idx)
    r = idx.dim()
    if x.dim() <= r or tuple(x.shape[:r]) != tuple(idx.shape):
        raise ValueError("fancy_gather: x %s must extend idx's shape %s by at least one dim" %
                         (tuple(x.shape), tuple(idx.shape)))
    d0, d1 = idx.numel(), x.shape[r]
    d2 = x.numel() // (d0 * d1) if d0 * d1 else int(np.prod(x.shape[r + 1:], dtype=np.int64))
    out_shape = tuple(idx.shape) + tuple(x.shape[r + 1:])
    return _FancyGatherFunction.apply(x.contiguous(), idx.contiguous(), (d0, d1, d2), out_shape)


# ---- reduce_max -------------------------------------------------------------------------------------------------------
def _argmax_dtype(d1):
    if d1 <= 256:
        return torch.uint8, _lib.LABEL_U8
    if d1 <= 65536:
        return torch.uint16, _lib.LABEL_U16
    return torch.int32, _lib.LABEL_I32


@_on_device_of
def _rmax(x, d0, d1, d2):
    adt, code = _argmax_dtype(d1)
    y = torch.empty((d0, d2), dtype=x.dtype, device=x.device)
    a = torch.empty((d0, d2), dtype=adt, device=x.device)
    if d0 * d2:
        rc = _lib.load().bsmm_reduce_max(_dt(x), code, x.data_ptr(), y.data_ptr(), a.data_ptr(), d0, d1, d2,
                                         _lib.stream_ptr())
        _lib.check(rc, "bsmm_reduce_max")
    return y, a


@_on_device_of
def _rmax_grad(dy, a, d0, d1, d2):
    dx = torch.empty((d0, d1, d2), dtype=dy.dtype, device=dy.device)
    if d0 * d2:
        rc = _lib.load().bsmm_reduce_max_grad(_dt(dy), _argmax_dtype(d1)[1], dy.data_ptr(), a.data_ptr(),
                                              dx.data_ptr(), d0, d1, d2, _lib.stream_ptr())
        _lib.check(rc, "bsmm_reduce_max_grad")
    return dx


class _ReduceMaxFunction(torch.autograd.Function):
    """Saves only the argmax (uint8 / uint16 / int32); the gradient puts dy there (reference ewops.py:412-419)."""

    @staticmethod
    def forward(ctx, x, dims, y_shape):
        y, a = _rmax(x, *dims)
        ctx.args = (dims, tuple(x.shape))
        ctx.save_for_backward(a)
        ctx.mark_non_differentiable(a)
        return y.view(y_shape), a

    @staticmethod
    def backward(ctx, dy, _):
        dims, x_shape = ctx.args
        a, = ctx.saved_tensors
        return _rmax_grad(dy.contiguous().view(dims[0], dims[2]), a, *dims).view(x_shape), None, None


def reduce_max(x, axis, keepdims=False, use_tf=False):
    """The maximum of x along `axis` (reference ewops.py:394-410), differentiable in x: dx holds dy at the position the
    maximum was taken from and 0 elsewhere. The position is stored as uint8 when the axis has <= 256 entries, uint16
    when <= 65536, int32 beyond.

    Every axis, the last one included, runs on this package's kernel, with the reference kernel's rule: the first entry
    strictly greater than everything before it wins, starting from -FLT_MAX at index 0. So ties go to the first entry, a
    NaN is never taken, and a slice of NaNs or of -inf gives -FLT_MAX (-inf in fp16 / bf16, where it rounds so) at index
    0. This differs from torch.amax / torch.max, which propagate NaN.

    x: CUDA, fp32 / fp16 / bf16, rank >= 1, the axis non-empty. axis: a Python int. use_tf=True raises ValueError."""
    if use_tf:
        raise ValueError("reduce_max: use_tf is a TensorFlow composition; there is none here")
    _cuda(x, "reduce_max")
    if type(axis) is not int:
        raise ValueError("reduce_max: axis must be a Python int, got %r" % (axis,))
    nd = x.dim()
    if not -nd <= axis < nd:
        raise ValueError("reduce_max: axis %d out of range for a tensor of rank %d" % (axis, nd))
    axis %= nd
    shape = tuple(x.shape)
    d1 = shape[axis]
    if d1 == 0:
        raise ValueError("reduce_max: the reduced axis of shape %s is empty" % (shape,))
    d0, d2 = int(np.prod(shape[:axis], dtype=np.int64)), int(np.prod(shape[axis + 1:], dtype=np.int64))
    y_shape = shape[:axis] + ((1,) if keepdims else ()) + shape[axis + 1:]
    return _ReduceMaxFunction.apply(x.contiguous(), (d0, d1, d2), y_shape)[0]


# ---- assign_add -------------------------------------------------------------------------------------------------------
def assign_add(y, x, name=None):
    """y += x in place, formed in fp32 and rounded once, and returns y (reference ewops.py:423-424). Not differentiable;
    y's version counter is bumped so that autograd refuses a graph that saved y before. y and x: CUDA, one shape and
    dtype of fp32 / fp16 / bf16; y contiguous."""
    for t in (y, x):
        _cuda(t, "assign_add")
    _same_device("assign_add", y, x)
    if y.shape != x.shape or y.dtype != x.dtype:
        raise ValueError("assign_add: y and x must share one shape and dtype, got %s %s and %s %s" %
                         (tuple(y.shape), y.dtype, tuple(x.shape), x.dtype))
    if not y.is_contiguous():
        raise ValueError("assign_add: y must be contiguous (it is updated in place)")
    with torch.no_grad():
        _fwd(y, ADD_OP, x.contiguous(), None, 0, 1.0, y)
    torch.autograd.graph.increment_version(y)
    return y


# `from blocksparse_b200 import ewops as ew; ew.add(...)` reads as the reference does; ewops.__all__ is left as it is.
from . import ewops as _ewops  # noqa: E402

for _name in __all__:
    setattr(_ewops, _name, globals()[_name])
del _name
