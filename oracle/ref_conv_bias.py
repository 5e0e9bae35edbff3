"""ctypes binding of the edge bias and cwise_linear entries in oracle/_ref/libbsref.so (oracle/ref/conv_bias.cu,
oracle/ref/cwise_linear.cu): the reference's own EdgeBiasForward / EdgeBiasBackward and CWiseLinear_Forward /
CWiseLinear_Backward launchers, built for sm_90a, on the plumbing of oracle/ref_kernels.py. Their offsets are 32-bit
and their grids put N on grid.z (edge bias) or grid.y (cwise_linear forward), so shapes must stay inside those limits.
Only the test suite and scripts/conv_bias.py import this module."""
import ctypes

import numpy as np
import torch

from . import ref_kernels as rk

_i, _u, _p = ctypes.c_int, ctypes.c_uint, ctypes.c_void_p
SIGNATURES = {
    "bsref_edge_bias": [_i, _p, _p, _p, _p, _p, _u, _u, _u, _u, _i, _i, _p],
    "bsref_edge_bias_grad": [_i, _p, _p, _p, _p, _p, _p, _u, _u, _u, _u, _i, _p],
    "bsref_cwise_linear": [_i, _p, _p, _p, _p, _u, _u, _u, _i, _i, _p],
    "bsref_cwise_linear_grad": [_i, _p, _p, _p, _p, _p, _p, _p, _u, _u, _u, _i, _i, _p],
}
_FNS = {}


def missing():
    """Why the entries cannot be called here, or None when they can."""
    if not rk.available():
        return "oracle/_ref/libbsref.so not built (no reference checkout)"
    if not all(hasattr(rk.load(), name) for name in SIGNATURES):
        return ("oracle/_ref/libbsref.so was built without oracle/ref/conv_bias.cu and cwise_linear.cu; rebuild it "
                "with make -C oracle/ref REF=<reference checkout>")
    return None


def _fn(name):
    fn = _FNS.get(name)
    if fn is None:
        fn = _FNS[name] = getattr(rk.load(), name)
        fn.argtypes, fn.restype = SIGNATURES[name], _i
    return fn


def launcher(name, *args):
    """A zero-argument callable that enqueues one reference launch (for timing); raises on a launch error."""
    fn = _fn(name)

    def run():
        rc = fn(*args, rk._stream())
        if rc != 0:
            raise RuntimeError("%s: CUDA error %d" % (name, rc))
    return run


def edge_bias_args(op, x, g, b, y, lut, inference=False):
    N, MPQ = x.shape[0], int(np.prod(op.MPQ))
    rk._u32("N * K * MPQ", N * op.K * MPQ)
    return (rk._dt(x), y.data_ptr(), x.data_ptr(), g.data_ptr(), b.data_ptr(), lut.data_ptr(), op.edgeBiasDim, MPQ,
            op.K, N, op.layout, int(inference))


def edge_bias(op, x, g, b, inference=False):
    """y of the reference's EdgeBias on x (a copy of x is updated in place for inference)."""
    x, g, b = rk._dev(x, g.float(), b.float())
    lut = torch.as_tensor(op.edgeBiasLut).to(x.device)
    y = x.clone() if inference else torch.empty_like(x)
    src = y if inference else x
    launcher("bsref_edge_bias", *edge_bias_args(op, src, g, b, y, lut, inference))()
    torch.cuda.current_stream().synchronize()
    return y


def edge_bias_grad(op, dy, x, g):
    """(dx, dg, db) of the reference's EdgeBiasGrad; dx is a copy of dy scaled in place, as the op does."""
    dy, x, g = rk._dev(dy, x, g.float())
    lut = torch.as_tensor(op.edgeBiasLut).to(x.device)
    dx = dy.clone()
    dg = torch.empty(op.shape, dtype=torch.float32, device=x.device)
    db = torch.empty(op.shape, dtype=torch.float32, device=x.device)
    N, MPQ = x.shape[0], int(np.prod(op.MPQ))
    rk._u32("N * K * MPQ", N * op.K * MPQ)
    launcher("bsref_edge_bias_grad", rk._dt(x), dx.data_ptr(), dg.data_ptr(), db.data_ptr(), x.data_ptr(),
             g.data_ptr(), lut.data_ptr(), op.edgeBiasDim, MPQ, op.K, N, op.layout)()
    torch.cuda.current_stream().synchronize()
    return dx, dg, db


def _dims(x):
    N, C = x.shape[0], x.shape[1]
    DHW = int(np.prod(x.shape[2:])) if x.dim() > 2 else 1
    rk._u32("N * C * DHW", N * C * DHW)
    return N, C, DHW


def cwise_linear(x, a=None, b=None, relu=False, bias_first=False):
    x, = rk._dev(x)
    y = torch.empty_like(x)
    N, C, DHW = _dims(x)
    launcher("bsref_cwise_linear", rk._dt(x), y.data_ptr(), x.data_ptr(), None if a is None else a.data_ptr(),
             None if b is None else b.data_ptr(), N, C, DHW, int(relu), int(bias_first))()
    torch.cuda.current_stream().synchronize()
    return y


def cwise_linear_grad(dy, xy, a=None, b=None, relu=False, bias_first=False):
    """(dx, da, db) of the reference's CWiseLinearGrad: xy is x with a gain, y for relu without one; dx is dy itself
    without gain and relu, and da / db are None where a / b are."""
    dy, = rk._dev(dy)
    N, C, DHW = _dims(dy)
    rd = a is not None or relu
    dx = torch.empty_like(dy) if rd else dy
    da = torch.empty(C, dtype=torch.float32, device=dy.device) if a is not None else None
    db = torch.empty(C, dtype=torch.float32, device=dy.device) if b is not None else None
    p = lambda t: None if t is None else t.data_ptr()
    launcher("bsref_cwise_linear_grad", rk._dt(dy), p(dx) if rd else None, p(da), p(db), dy.data_ptr(), p(xy), p(a),
             p(b), N, C, DHW, int(relu), int(bias_first))()
    torch.cuda.current_stream().synchronize()
    return dx, da, db
