"""Float64 oracle of the elementwise ops of blocksparse_b200.elementwise (the reference's blocksparse/ewops.py :69-424).

Every function takes NumPy arrays (any float dtype) and returns float64, except where the reference's selection or
rounding rule is itself the thing being checked: reduce_max's argmax, add_n's grouping and concrete_gate's uniforms,
which are replayed as the device forms them.
"""
import numpy as np

from .ewops_oracle import _LO, _u64, philox4x32_10

SQRT_2_PI = np.sqrt(2.0 / np.pi)
FLT_MAX = float(np.finfo(np.float32).max)


def _f(x):
    return np.asarray(x, np.float64)


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


# ---- binary ops (ewops.py:69-95) and their gradients (:116-127) --------------------------------------------------------
BINARY = {
    "add": lambda x, y: x + y,
    "subtract": lambda x, y: x - y,
    "multiply": lambda x, y: x * y,
    "divide": lambda x, y: x / y,
    "maximum": np.fmax,          # fmaxf / fminf: a NaN operand gives the other one
    "minimum": np.fmin,
}


def binary(op, x, y):
    with np.errstate(all="ignore"):
        return BINARY[op](_f(x), _f(y))


def binary_grad(op, dz, x, y):
    """(dx, dy); maximum / minimum give dz to every operand equal to the result (x >= y and y >= x)."""
    dz, x, y = _f(dz), _f(x), _f(y)
    with np.errstate(all="ignore"):
        if op == "add":
            return dz, dz
        if op == "subtract":
            return dz, -dz
        if op == "multiply":
            return dz * y, dz * x
        if op == "divide":
            return dz / y, -dz * x / (y * y)
        if op == "maximum":
            return np.where(x >= y, dz, 0.0), np.where(y >= x, dz, 0.0)
        if op == "minimum":
            return np.where(x <= y, dz, 0.0), np.where(y <= x, dz, 0.0)
    raise ValueError(op)


def bias_add(x, b):
    return _f(x) + _f(b).reshape(-1)


def gain_mul(x, g):
    return _f(x) * _f(g).reshape(-1)


def bias_add_grad(dz, b):
    """(dx, db): dx = dz, db = column sums of dz over every axis but the last."""
    dz = _f(dz)
    return dz, dz.reshape(-1, dz.shape[-1]).sum(0)


def gain_mul_grad(dz, x, g):
    dz, x = _f(dz), _f(x)
    return dz * _f(g).reshape(-1), (dz * x).reshape(-1, dz.shape[-1]).sum(0)


# ---- unary ops (ewops.py:97-114) and their gradients (:129-143) --------------------------------------------------------
def unary(op, x, alpha=1.0):
    x = _f(x)
    with np.errstate(all="ignore"):
        if op == "negative":
            return -x
        if op == "reciprocal":
            return 1.0 / x
        if op == "square":
            return x * x
        if op == "sqrt":
            return np.sqrt(x)
        if op == "exp":
            return np.exp(x)
        if op == "log":
            return np.log(x)
        if op == "sigmoid":
            return _sig(x)
        if op == "tanh":
            return np.tanh(x)
        if op == "relu":
            return np.where(x > 0, x, 0.0)
        if op == "elu":
            return np.where(x > 0, x, alpha * np.expm1(x))
        if op == "gelu":
            return 0.5 * x * (1.0 + np.tanh(SQRT_2_PI * (x + alpha * x ** 3)))
        if op == "swish":
            return x * _sig(alpha * x)
    raise ValueError(op)


Z_GRAD = ("sigmoid", "tanh", "relu")       # the gradients the reference forms from the output z


def unary_grad(op, dz, s, alpha=1.0):
    """dx from dz and s: the output z for sigmoid, tanh and relu, the input x otherwise."""
    dz, s = _f(dz), _f(s)
    with np.errstate(all="ignore"):
        if op == "negative":
            return -dz
        if op == "reciprocal":
            return -dz / (s * s)
        if op == "square":
            return 2.0 * dz * s
        if op == "sqrt":
            return 0.5 * dz / np.sqrt(s)
        if op == "exp":
            return dz * np.exp(s)
        if op == "log":
            return dz / s
        if op == "sigmoid":
            return dz * (s - s * s)
        if op == "tanh":
            return dz * (1.0 - s * s)
        if op == "relu":
            return np.where(s > 0, dz, 0.0)
        if op == "elu":
            return np.where(s > 0, dz, dz * alpha * np.exp(s))
        if op == "gelu":
            t = np.tanh(SQRT_2_PI * (s + alpha * s ** 3))
            return 0.5 * dz * (1 + t) + 0.5 * dz * s * (1 - t * t) * SQRT_2_PI * (1 + 3 * alpha * s * s)
        if op == "swish":
            g = _sig(alpha * s)
            return dz * (g + alpha * s * g * (1 - g))
    raise ValueError(op)


# ---- filter_tensor (ewops.py:158-172, ew_op_gpu.cu:820-841) ------------------------------------------------------------
def filter_tensor(x, scale=1.0, saturate=0.0, zero_infs=False, zero_nans=False):
    """saturate(scale * x) after zeroing infs / NaNs; the clamp is fmin / fmax, so a NaN left in becomes +saturate."""
    x = _f(x).copy()
    if zero_infs:
        x[np.isinf(x)] = 0.0
    if zero_nans:
        x[np.isnan(x)] = 0.0
    with np.errstate(all="ignore"):
        x = x * float(np.float32(scale))
    if saturate != 0.0:
        s = float(np.float32(saturate))
        x = np.fmax(np.fmin(x, s), -s)
    return x


# ---- add_n8 / add_n (ewops.py:268-292) ---------------------------------------------------------------------------------
def add_n8(xs):
    """float64: the exact sum (the device adds in fp32 in list order and rounds once)."""
    return sum(_f(x) for x in xs)


def add_n(xs, dtype):
    """The reference's grouping with each add_n8 (and the two-tensor add) rounded to `dtype` (a torch dtype name:
    'float32', 'float16' or 'bfloat16') through fp32, as the device does: returns the float64 of the rounded result,
    and the float64 exact sum for comparison."""
    import torch

    def rnd(v):
        return torch.as_tensor(np.asarray(v, np.float32)).to(getattr(torch, dtype)).double().numpy()

    xs = [rnd(x) for x in xs]
    exact = sum(xs)
    if len(xs) == 1:
        return xs[0], exact
    if len(xs) == 2:
        return rnd(np.float32(xs[0]) + np.float32(xs[1])), exact
    def group(ts):
        acc = np.zeros_like(np.asarray(ts[0], np.float32))
        for t in ts:
            acc = acc + np.asarray(t, np.float32)        # fp32, in list order, from +0
        return rnd(acc)

    rest = xs[::-1]
    total = group(rest[:8])
    for i in range(8, len(rest), 7):
        total = group([total] + rest[i:i + 7])
    return total, exact


# ---- concrete gate (ewops.py:244-265, ew_op_gpu.cu:578-685) ------------------------------------------------------------
def concrete_uniform(seed, call, n, epsilon=1e-6):
    """fp32 f of every element, replayed exactly as the device forms it: u from Philox4x32-10 as dropout's, then
    f = fp32(u) * fp32(2^-32 (1 - 2 eps)) + eps, every step rounded to fp32."""
    seed, call = _u64(seed), _u64(call)
    g = np.arange((n + 3) // 4, dtype=np.uint64)
    ctr = np.stack([g & _LO, g >> np.uint64(32), np.full_like(g, call & 0xFFFFFFFF), np.full_like(g, call >> 32)], -1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint32), (len(g), 2))
    u = philox4x32_10(ctr.astype(np.uint32), key).reshape(-1)[:n]
    eps = np.float32(epsilon)
    scale = np.float32(2.3283064365386962891e-10) * (np.float32(1) - np.float32(2) * eps)
    return u.astype(np.float32) * scale + eps


def _stretch32(c, limit_a, limit_b):
    la, lb = np.float32(limit_a), np.float32(limit_b)
    return np.asarray(c, np.float32) * (lb - la) + la


def concrete_gate(loga, f, tempurature=2.0 / 3.0, limit_a=-0.1, limit_b=1.1):
    """(gate, concrete) in float64 from the fp32 uniforms f (concrete_uniform)."""
    rcp = float(np.float32(1) / np.float32(tempurature))
    f = _f(f).reshape(np.shape(loga))
    c = _sig((np.log(f) - np.log1p(-f) + _f(loga)) * rcp)
    gate = np.clip(c * (float(np.float32(limit_b)) - float(np.float32(limit_a))) + float(np.float32(limit_a)), 0, 1)
    return gate, c


def concrete_gate_grad(dgate, concrete, tempurature=2.0 / 3.0, limit_a=-0.1, limit_b=1.1):
    """dloga from the stored fp32 concrete values; the [0, 1] test uses the fp32 stretch, as the device forms it."""
    rcp = float(np.float32(1) / np.float32(tempurature))
    st = _stretch32(concrete, limit_a, limit_b)
    c = _f(concrete)
    d = np.where((st >= 0) & (st <= 1), _f(dgate), 0.0)
    return d * (float(np.float32(limit_b)) - float(np.float32(limit_a))) * (c - c * c) * rcp


def concrete_gate_infer(loga, limit_a=-0.1, limit_b=1.1):
    la, lb = float(np.float32(limit_a)), float(np.float32(limit_b))
    return np.clip(_sig(_f(loga)) * (lb - la) + la, 0, 1)


# ---- fancy_gather (ewops.py:352-386, ew_op_gpu.cu:1434-1504) ----------------------------------------------------------
def fancy_gather(x, idx):
    """x[i..., max(idx, 0), ...], 0 where the index is >= the dim (values copied as they are)."""
    x = np.asarray(x)
    idx = np.asarray(idx).astype(np.int64)
    r = idx.ndim
    d1 = x.shape[r]
    xf = x.reshape((idx.size, d1, -1))
    i = np.maximum(idx.reshape(-1), 0)
    ok = i < d1
    out = np.zeros((idx.size, xf.shape[2]), x.dtype)
    out[ok] = xf[np.nonzero(ok)[0], i[ok]]
    return out.reshape(idx.shape + x.shape[r + 1:])


def fancy_gather_grad(dy, idx, x_shape):
    dy = np.asarray(dy)
    idx = np.asarray(idx).astype(np.int64)
    r = idx.ndim
    d1 = x_shape[r]
    dx = np.zeros((idx.size, d1, dy.size // max(idx.size, 1)), dy.dtype)
    i = np.maximum(idx.reshape(-1), 0)
    ok = i < d1
    dx[np.nonzero(ok)[0], i[ok]] = dy.reshape(idx.size, -1)[ok]
    return dx.reshape(x_shape)


# ---- reduce_max (ewops.py:389-419, ew_op_gpu.cu:1545-1602) -------------------------------------------------------------
def reduce_max(x, axis, keepdims=False):
    """(max, argmax) by the reference kernel's rule: start from (-FLT_MAX, 0), take an entry only when strictly greater,
    so the first maximum wins, NaN is never taken and a slice of NaNs or -inf gives (-FLT_MAX, 0)."""
    x = np.moveaxis(_f(x), axis, -1)
    valid = ~np.isnan(x) & (x > -FLT_MAX)
    xv = np.where(valid, x, -np.inf)
    m = xv.max(-1)
    am = np.argmax(xv == m[..., None], -1)          # the first entry equal to the maximum
    none = ~valid.any(-1)
    m = np.where(none, -FLT_MAX, m)
    am = np.where(none, 0, am)
    if keepdims:
        m, am = np.expand_dims(m, axis), np.expand_dims(am, axis)
    return m, am


def reduce_max_grad(dy, argmax, x_shape, axis):
    dy, am = _f(dy), np.asarray(argmax).astype(np.int64)
    axis %= len(x_shape)
    d1 = x_shape[axis]
    dy = dy.reshape(x_shape[:axis] + x_shape[axis + 1:])
    am = am.reshape(dy.shape)
    onehot = np.arange(d1) == am[..., None]
    return np.moveaxis(np.where(onehot, dy[..., None], 0.0), -1, axis)


# ---- float_cast (ewops.py:178-204) -------------------------------------------------------------------------------------
def float_cast(x):
    """The exact value; the device rounds it once to the destination dtype."""
    return _f(x)
