"""ctypes binding of the quantize entries in oracle/_ref/libbsref.so (oracle/ref/quantize.cu): the reference's own
Quantize and QuantizationStats launchers, built for sm_90a, given the rounding constants its QuantizeOp derives from the
spec and the exponent (oracle/quantize_oracle.fmt), with the launchers' 32-bit sizes and the plumbing of
oracle/ref_kernels.py. Only the test suite imports this module."""
import ctypes

import numpy as np
import torch

from . import quantize_oracle as qo
from . import ref_kernels as rk

_u, _i, _f, _p = ctypes.c_uint, ctypes.c_int, ctypes.c_float, ctypes.c_void_p
SIGNATURES = {
    "bsref_quantize": [_i, _p, _p, _p, _f, _u, _f, _f, _u, _u, _i, _p],
    "bsref_quantization_stats": [_i, _p, _p, _p, _f, _f, _u, _p],
}

_FNS = {}


def missing():
    """Why the quantize entries cannot be called here, or None when they can: the library may be absent (no reference
    checkout where it was built), or built by an oracle/ref without quantize.cu."""
    if not rk.available():
        return "oracle/_ref/libbsref.so not built (no reference checkout)"
    if not all(hasattr(rk.load(), name) for name in SIGNATURES):
        return ("oracle/_ref/libbsref.so was built without oracle/ref/quantize.cu and has no quantize entries; rebuild "
                "it with make -C oracle/ref REF=<reference checkout>")
    return None


def available():
    return missing() is None


def _fn(name):
    fn = _FNS.get(name)
    if fn is None:
        fn = _FNS[name] = getattr(rk.load(), name)
        fn.argtypes, fn.restype = SIGNATURES[name], _i
    return fn


def _bits_f32(b):
    return float(np.array([b], np.uint32).view(np.float32)[0])


def quantize(x, exp, ebits, fbits, denorm=True):
    """y of the reference kernel without stochastic rounding, x fp32 or bf16, at exponent record value exp (the
    QuantizeOp constants of UpdateExponent, with this port's clamp of the exponent at 254)."""
    x, = rk._dev(x)
    if x.dtype not in (torch.float32, torch.bfloat16):
        raise ValueError("Quantize is registered for fp32 and bf16 only")
    f = qo.fmt(exp, ebits, fbits, denorm)
    round_scale = _bits_f32((127 - fbits - 1) << 23)
    y = rk._Out(x.shape, x.dtype, x.device)
    rc = _fn("bsref_quantize")(rk._dt(x), y.t.data_ptr(), x.data_ptr(), None, round_scale, f["mask"],
                               _bits_f32(f["max_float"]), _bits_f32(f["min_float"]), f["exp_norm"],
                               rk._u32("size", x.numel()), 0, rk._stream())
    if rc != 0:
        raise RuntimeError("bsref_quantize: CUDA error %d" % rc)
    torch.cuda.current_stream().synchronize()
    return y.check("bsref_quantize")


def quantization_stats(x, max_float, ftz_float):
    """(mean |x|, stdv, sat %, ftz %, max |x|) from QuantizationStats, x fp32, fp16 or bf16."""
    x, = rk._dev(x)
    scratch = torch.zeros(8, dtype=torch.float32, device=x.device)
    out = (ctypes.c_float * 5)()
    rc = _fn("bsref_quantization_stats")(rk._dt(x), out, scratch.data_ptr(), x.data_ptr(), float(max_float),
                                         float(ftz_float), rk._u32("size", x.numel()), rk._stream())
    if rc != 0:
        raise RuntimeError("bsref_quantization_stats: CUDA error %d" % rc)
    return tuple(np.float32(v) for v in out)
