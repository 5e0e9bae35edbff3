"""ctypes binding of the LSTM entries in oracle/_ref/libbsref.so (oracle/ref/lstm.cu): the reference's own gate,
gate-gradient and sparse relu launchers, built for sm_90a, with the argument checks of their ops (lstm_op.cc), the
limits of the launchers (int offsets, N on grid.y or grid.x) and the plumbing of oracle/ref_kernels.py. Only the test
suite imports this module."""
import ctypes

import torch

from . import ref_kernels as rk

_u, _i, _f, _p = ctypes.c_uint, ctypes.c_int, ctypes.c_float, ctypes.c_void_p
SIGNATURES = {
    "bsref_lstm_gates": [_i, _p, _p, _p, _p, _p, _f, _i, _i, _p],
    "bsref_lstm_gates_grad": [_i, _p, _p, _p, _p, _p, _p, _p, _f, _i, _i, _p],
    "bsref_lstm_gates4": [_i, _p, _p, _p, _p, _p, _p, _p, _f, _i, _i, _p],
    "bsref_lstm_gates4_grad": [_i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _f, _i, _i, _p],
    "bsref_sparse_relu": [_i, _p, _p, _f, _u, _u, _p],
}

_FNS = {}


def missing():
    """Why the LSTM entries cannot be called here, or None when they can. The library may be absent (no reference
    checkout where it was built), or built by an oracle/ref that did not yet have lstm.cu: every other entry is then
    there and these are not."""
    if not rk.available():
        return "oracle/_ref/libbsref.so not built (no reference checkout)"
    if not all(hasattr(rk.load(), name) for name in SIGNATURES):
        return ("oracle/_ref/libbsref.so was built without oracle/ref/lstm.cu and has no LSTM entries; rebuild it with "
                "make -C oracle/ref REF=<reference checkout>")
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


def _rows(what, N, limit=65535):
    if not 0 <= N <= limit:
        raise ValueError("%s: %d rows exceed the launcher's grid (at most %d)" % (what, N, limit))


def lstm_gates(c, h, bias=None, forget_bias=1.0):
    """(c_next, h_next) of LSTMGates: c (N, K), h (N, 4K) of one dtype, bias None or 4K fp32 entries."""
    c, h = rk._dev(c, h)
    N, K = c.shape
    if h.shape != (N, 4 * K) or h.dtype != c.dtype or (bias is not None and (bias.dtype != torch.float32 or
                                                                              bias.numel() != 4 * K)):
        raise ValueError("LSTMGates: c (N, K), h (N, 4K) of one dtype, bias of 4K fp32 entries")
    _rows("LSTMGates", N)
    rk._i32("N * 4K", N * 4 * K)
    b = None if bias is None else rk._dev(bias)[0]
    outs = [rk._Out(c.shape, c.dtype, c.device) for _ in range(2)]
    return _call("bsref_lstm_gates", outs, rk._dt(c), outs[0].t.data_ptr(), outs[1].t.data_ptr(), c.data_ptr(),
                 h.data_ptr(), None if b is None else b.data_ptr(), float(forget_bias), N, 4 * K)


def lstm_gates_grad(c, h, eh, ec=None, bias=None, forget_bias=1.0):
    """(dc, dh) of LSTMGatesGrad; ec None is the op's grads list without ec."""
    c, h, eh = rk._dev(c, h, eh)
    N, K = c.shape
    _rows("LSTMGatesGrad", N)
    rk._i32("N * 4K", N * 4 * K)
    ec = None if ec is None else rk._dev(ec)[0]
    b = None if bias is None else rk._dev(bias)[0]
    outs = [rk._Out(c.shape, c.dtype, c.device), rk._Out(h.shape, h.dtype, h.device)]
    return _call("bsref_lstm_gates_grad", outs, rk._dt(c), outs[0].t.data_ptr(), outs[1].t.data_ptr(),
                 None if ec is None else ec.data_ptr(), eh.data_ptr(), c.data_ptr(), h.data_ptr(),
                 None if b is None else b.data_ptr(), float(forget_bias), N, 4 * K)


def lstm_gates4(c, i, u, f, o, forget_bias=1.0):
    """(c_next, h_next) of LSTMGates4, inputs in the op's order (c, i, u, f, o), each (N, K)."""
    ts = rk._dev(c, i, u, f, o)
    N, K = ts[0].shape
    rk._i32("N * K", N * K)
    outs = [rk._Out(ts[0].shape, ts[0].dtype, ts[0].device) for _ in range(2)]
    return _call("bsref_lstm_gates4", outs, rk._dt(ts[0]), outs[0].t.data_ptr(), outs[1].t.data_ptr(),
                 *[t.data_ptr() for t in ts], float(forget_bias), N, K)


def lstm_gates4_grad(c, i, u, f, o, eh, ec=None, forget_bias=1.0):
    """(dc, di, du, df, do) of LSTMGates4Grad."""
    ts = rk._dev(c, i, u, f, o, eh)
    N, K = ts[0].shape
    rk._i32("N * K", N * K)
    ec = None if ec is None else rk._dev(ec)[0]
    outs = [rk._Out(ts[0].shape, ts[0].dtype, ts[0].device) for _ in range(5)]
    return _call("bsref_lstm_gates4_grad", outs, rk._dt(ts[0]), *[o.t.data_ptr() for o in outs],
                 None if ec is None else ec.data_ptr(), ts[5].data_ptr(), *[t.data_ptr() for t in ts[:5]],
                 float(forget_bias), N, K)


def sparse_relu(x, alpha=1.0):
    """y of SparseRelu along the last axis."""
    x, = rk._dev(x)
    K = x.shape[-1]
    N = x.numel() // K
    rk._i32("N * K", N * K)
    y = rk._Out(x.shape, x.dtype, x.device)
    return _call("bsref_sparse_relu", [y], rk._dt(x), y.t.data_ptr(), x.data_ptr(), float(alpha), K, N)[0]
