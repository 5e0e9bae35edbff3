"""ctypes binding of the elementwise entries in oracle/_ref/libbsref.so (oracle/ref/elementwise.cu): the reference's own
EW_Forward / EW_Backward, FloatCast, AddN, ConcreteGateGrad / ConcreteGateInfer, EW_Fancy_Gather(_Grad) and
EW_Reduce_Max(_Grad) launchers, built for sm_90a, with the argument checks of their ops (ew_op.cc), the limits of the
launchers (int / uint sizes) and the plumbing of oracle/ref_kernels.py, including its poisoned output guard. Only the
test suite imports this module."""
import ctypes

import torch

from . import ref_kernels as rk

_u, _i, _f, _p = ctypes.c_uint, ctypes.c_int, ctypes.c_float, ctypes.c_void_p
SIGNATURES = {
    "bsref_ew_forward": [_i, _p, _p, _p, _p, _f, _i, _i, _i, _p],
    "bsref_ew_backward": [_i, _p, _p, _p, _p, _p, _p, _p, _p, _f, _i, _i, _i, _p],
    "bsref_float_cast": [_i, _i, _p, _p, _i, _p],
    "bsref_add_n": [_i, _p, ctypes.POINTER(_p), _i, _u, _p],
    "bsref_concrete_gate_grad": [_p, _p, _p, _f, _f, _f, _u, _p],
    "bsref_concrete_gate_infer": [_p, _p, _f, _f, _u, _p],
    "bsref_fancy_gather": [_i, _i, _p, _p, _p, _u, _u, _u, _p],
    "bsref_reduce_max": [_i, _i, _i, _p, _p, _p, _u, _u, _u, _p],
}
OPS = ["add", "subtract", "multiply", "divide", "maximum", "minimum", "negative", "reciprocal", "square", "sqrt", "exp",
       "log", "sigmoid", "tanh", "relu", "elu", "gelu", "swish", "bias_add", "gain_mul"]

_FNS = {}


def missing():
    """Why the elementwise entries cannot be called here, or None when they can: the library may be absent (no reference
    checkout where it was built), or built by an oracle/ref without elementwise.cu."""
    if not rk.available():
        return "oracle/_ref/libbsref.so not built (no reference checkout)"
    if not all(hasattr(rk.load(), name) for name in SIGNATURES):
        return ("oracle/_ref/libbsref.so was built without oracle/ref/elementwise.cu and has no elementwise entries; "
                "rebuild it with make -C oracle/ref REF=<reference checkout>")
    return None


def available():
    return missing() is None


def _call(name, outs, *args):
    fn = _FNS.get(name)
    if fn is None:
        fn = _FNS[name] = getattr(rk.load(), name)
        fn.argtypes, fn.restype = SIGNATURES[name], _i
    rc = fn(*args, rk._stream())
    if rc != 0:
        raise RuntimeError("%s: CUDA error %d" % (name, rc))
    torch.cuda.current_stream().synchronize()
    return [o.check(name) for o in outs]


def ew_forward(op, x, y=None, b=None, alpha=1.0):
    """z of EwZXy (binary ops, x and y of one shape), EwZXa (unary) or EwZXb (bias_add / gain_mul: b fp32 of x's last
    dim)."""
    code = OPS.index(op)
    x, = rk._dev(x)
    y = None if y is None else rk._dev(y)[0]
    if code >= 18:
        b, = rk._dev(b)
        if b.dtype != torch.float32 or b.numel() != x.shape[-1]:
            raise ValueError("EwZXb: b must be fp32 of x's last dim")
        K = rk._i32("K", x.shape[-1])
        size, N = K, rk._i32("N", x.numel() // K)
        if N >= 65536:
            raise ValueError("EwZXb: N = %d overflows grid.y" % N)
    else:
        size, N = rk._i32("size", x.numel()), 0
    z = rk._Out(x.shape, x.dtype, x.device)
    return _call("bsref_ew_forward", [z], rk._dt(x), z.t.data_ptr(), x.data_ptr(), None if y is None else y.data_ptr(),
                 None if b is None else b.data_ptr(), float(alpha), size, N, code)[0]


def ew_backward(op, dz, x=None, y=None, z=None, g=None, alpha=1.0):
    """dx (unary), (dx, dy) (multiply / divide / maximum / minimum), db fp32 (bias_add) or (dx, dg fp32) (gain_mul)."""
    code = OPS.index(op)
    dz, = rk._dev(dz)
    x, y, z, g = (None if t is None else rk._dev(t)[0] for t in (x, y, z, g))
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    if code >= 18:
        K = rk._i32("K", dz.shape[-1])
        size, N = K, rk._i32("N", dz.numel() // K)
        db = rk._Out((K,), torch.float32, dz.device)
        if code == 18:
            return _call("bsref_ew_backward", [db], rk._dt(dz), None, None, db.t.data_ptr(), dz.data_ptr(), None, None,
                         None, None, 1.0, size, N, code)[0]
        dx = rk._Out(dz.shape, dz.dtype, dz.device)
        return _call("bsref_ew_backward", [dx, db], rk._dt(dz), dx.t.data_ptr(), None, db.t.data_ptr(), dz.data_ptr(),
                     x.data_ptr(), None, None, g.data_ptr(), 1.0, size, N, code)
    size = rk._i32("size", dz.numel())
    dx = rk._Out(dz.shape, dz.dtype, dz.device)
    if 2 <= code <= 5:
        dy = rk._Out(dz.shape, dz.dtype, dz.device)
        return _call("bsref_ew_backward", [dx, dy], rk._dt(dz), dx.t.data_ptr(), dy.t.data_ptr(), None, dz.data_ptr(),
                     x.data_ptr(), y.data_ptr(), None, None, float(alpha), size, 0, code)
    return _call("bsref_ew_backward", [dx], rk._dt(dz), dx.t.data_ptr(), None, None, dz.data_ptr(), ptr(x), None, ptr(z),
                 None, float(alpha), size, 0, code)[0]


def float_cast(x, dtype):
    x, = rk._dev(x)
    if (x.dtype == torch.float32) == (dtype == torch.float32):
        raise ValueError("FloatCast is registered for fp32 <-> fp16 / bf16 only")
    y = rk._Out(x.shape, dtype, x.device)
    return _call("bsref_float_cast", [y], rk.DT[dtype], rk._dt(x), y.t.data_ptr(), x.data_ptr(),
                 rk._i32("size", x.numel()))[0]


def add_n8(xs):
    xs = rk._dev(*xs)
    if not 1 <= len(xs) <= 9:
        raise ValueError("AddN8: only 8+1 inputs allowed")
    y = rk._Out(xs[0].shape, xs[0].dtype, xs[0].device)
    arr = (_p * len(xs))(*[t.data_ptr() for t in xs])
    return _call("bsref_add_n", [y], rk._dt(xs[0]), y.t.data_ptr(), arr, len(xs), rk._u32("size", xs[0].numel()))[0]


def concrete_gate_grad(dgate, concrete, tempurature=2.0 / 3.0, limit_a=-0.1, limit_b=1.1):
    dgate, concrete = rk._dev(dgate, concrete)
    if dgate.dtype != torch.float32 or concrete.dtype != torch.float32:
        raise ValueError("ConcreteGateGrad is registered for fp32 only")
    out = rk._Out(dgate.shape, torch.float32, dgate.device)
    rcp = float(torch.tensor(1.0, dtype=torch.float32) / torch.tensor(tempurature, dtype=torch.float32))
    return _call("bsref_concrete_gate_grad", [out], out.t.data_ptr(), dgate.data_ptr(), concrete.data_ptr(),
                 float(limit_a), float(limit_b), rcp, rk._u32("size", dgate.numel()))[0]


def concrete_gate_infer(loga, limit_a=-0.1, limit_b=1.1):
    loga, = rk._dev(loga)
    if loga.dtype != torch.float32:
        raise ValueError("ConcreteGateInfer is registered for fp32 only")
    out = rk._Out(loga.shape, torch.float32, loga.device)
    return _call("bsref_concrete_gate_infer", [out], out.t.data_ptr(), loga.data_ptr(), float(limit_a), float(limit_b),
                 rk._u32("size", loga.numel()))[0]


def _gather_dims(x_shape, idx):
    r = idx.dim()
    d0, d1 = idx.numel(), x_shape[r]
    d2 = 1
    for d in x_shape[r + 1:]:
        d2 *= d
    if d2 > 1024:
        raise ValueError("fancy_gather: the reference asserts a trailing size <= 1024")
    return rk._u32("d0", d0), rk._u32("d1", d1), d2


def fancy_gather(x, idx):
    x, idx = rk._dev(x, idx)
    if idx.dtype != torch.int32:
        raise ValueError("FancyGather takes int32 indices")
    d0, d1, d2 = _gather_dims(tuple(x.shape), idx)
    rk._u32("size", x.numel())
    y = rk._Out(tuple(idx.shape) + tuple(x.shape[idx.dim() + 1:]), x.dtype, x.device)
    dt = 3 if x.dtype == torch.int32 else rk._dt(x)
    return _call("bsref_fancy_gather", [y], dt, 0, y.t.data_ptr(), idx.data_ptr(), x.data_ptr(), d0, d1, d2)[0]


def fancy_gather_grad(dy, idx, x_shape):
    dy, idx = rk._dev(dy, idx)
    d0, d1, d2 = _gather_dims(tuple(x_shape), idx)
    if d2 == 1 and d1 > 1024:
        raise ValueError("FancyGatherGrad: dim1 = %d exceeds the 1024 threads of a CTA" % d1)
    rk._u32("size", d0 * d1 * d2)
    dx = rk._Out(tuple(x_shape), dy.dtype, dy.device)
    return _call("bsref_fancy_gather", [dx], rk._dt(dy), 1, dx.t.data_ptr(), idx.data_ptr(), dy.data_ptr(), d0, d1,
                 d2)[0]


def _rmax_dims(shape, axis):
    axis %= len(shape)
    d0 = d2 = 1
    for d in shape[:axis]:
        d0 *= d
    for d in shape[axis + 1:]:
        d2 *= d
    return rk._u32("d0", d0), rk._u32("d1", shape[axis]), rk._u32("d2", d2)


def reduce_max(x, axis):
    """(y, argmax) of ReduceMax with its index type (uint8 for <= 256 entries, uint16 beyond)."""
    x, = rk._dev(x)
    d0, d1, d2 = _rmax_dims(tuple(x.shape), axis)
    if d1 > 65536:
        raise ValueError("ReduceMax: %d entries do not fit uint16" % d1)
    rk._u32("size", x.numel())
    it, adt = (rk.IT[torch.uint8], torch.uint8) if d1 <= 256 else (rk.IT[torch.uint16], torch.uint16)
    y = rk._Out((d0, d2), x.dtype, x.device)
    a = rk._Out((d0, d2), adt, x.device)
    return _call("bsref_reduce_max", [y, a], rk._dt(x), it, 0, y.t.data_ptr(), a.t.data_ptr(), x.data_ptr(), d0, d1, d2)


def reduce_max_grad(dy, argmax, x_shape, axis):
    dy, argmax = rk._dev(dy, argmax)
    d0, d1, d2 = _rmax_dims(tuple(x_shape), axis)
    dx = rk._Out(tuple(x_shape), dy.dtype, dy.device)
    it = rk.IT[argmax.dtype]
    return _call("bsref_reduce_max", [dx], rk._dt(dy), it, 1, dx.t.data_ptr(), argmax.data_ptr(), dy.data_ptr(), d0, d1,
                 d2)[0]
