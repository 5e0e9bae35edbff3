"""ctypes binding of bsref_adafactor in oracle/_ref/libbsref.so (oracle/ref/adafactor.cu): the reference's own Adafactor
launcher, built for sm_90a, with the argument checks of Adafactor2dOp / Adafactor1dOp (optimize_op.cc) and the plumbing
of oracle/ref_kernels.py. Only the test suite imports this module."""
import ctypes

import torch

from . import ref_kernels as rk

_u, _i, _f, _p = ctypes.c_uint, ctypes.c_int, ctypes.c_float, ctypes.c_void_p
SIGNATURES = {"bsref_adafactor": [_i, _p, _p, _p, _p, _p, _p, _p, _f, _f, _f, _f, _f, _u, _u, _f, _i, _i, _p]}

_FN = None


def missing():
    """Why bsref_adafactor cannot be called here, or None when it can. The library may be absent (no reference checkout
    where it was built), or built by an oracle/ref that did not yet have adafactor.cu: every other entry is then there
    and this one is not."""
    if not rk.available():
        return "oracle/_ref/libbsref.so not built (no reference checkout)"
    if not hasattr(rk.load(), "bsref_adafactor"):
        return ("oracle/_ref/libbsref.so was built without oracle/ref/adafactor.cu and has no bsref_adafactor; rebuild it "
                "with make -C oracle/ref REF=<reference checkout>")
    return None


def available():
    return missing() is None


def _fn():
    global _FN
    if _FN is None:
        fn = rk.load().bsref_adafactor
        fn.argtypes = SIGNATURES["bsref_adafactor"]
        fn.restype = _i
        _FN = fn
    return _FN


def adafactor(grad, param, cv, rv, lr, decay, epsilon=1e-30, clip_thresh=1.0, grad_scale=1.0, norm_scale=None,
              saturate=0.0, zero_infs=False, zero_nans=False):
    """One step on clones: returns (param, cv, rv). param fp32 of rank 1 or 2; rv None for rank 1 and (1, K) params,
    else rv [C] and cv [K]. grad fp32, fp16 or bf16. norm_scale: None or a 1-element fp32 CUDA tensor."""
    grad, param, cv = rk._dev(grad, param, cv)
    if param.dtype != torch.float32 or cv.dtype != torch.float32 or grad.shape != param.shape:
        raise ValueError("Adafactor: fp32 param and cv, grad of the param's shape")
    factored = param.dim() == 2 and param.shape[0] > 1
    if factored != (rv is not None) or param.dim() not in (1, 2):
        raise ValueError("Adafactor2d takes a (C > 1, K) param with rv; Adafactor1d a rank-1 or (1, K) one without")
    C, K = (param.shape[0], param.shape[1]) if factored else (1, param.numel())
    if cv.numel() != K or (factored and rv.numel() != C):
        raise ValueError("bad cv / rv shape")
    rk._u32("C * K", C * K)
    outs = [rk._Out(t.shape, torch.float32, param.device) for t in ((param, cv, rv) if factored else (param, cv))]
    for o, t in zip(outs, (param, cv, rv)):
        o.t.copy_(t)
    if C * K == 0:
        return [o.t for o in outs] + ([] if factored else [None])
    x = torch.empty(C * K, dtype=torch.float32, device=param.device)
    means = torch.empty(2, dtype=torch.float32, device=param.device)
    ns = None if norm_scale is None else rk._dev(norm_scale)[0].data_ptr()
    rc = _fn()(rk._dt(grad), outs[0].t.data_ptr(), outs[1].t.data_ptr(), outs[2].t.data_ptr() if factored else None,
               x.data_ptr(), means.data_ptr(), grad.data_ptr(), ns, float(grad_scale), float(lr), float(decay),
               float(epsilon), float(clip_thresh), C, K, float(saturate), int(bool(zero_infs)), int(bool(zero_nans)),
               rk._stream())
    if rc != 0:
        raise RuntimeError("bsref_adafactor: CUDA error %d" % rc)
    torch.cuda.current_stream().synchronize()
    res = [o.check("bsref_adafactor") for o in outs]
    return res if factored else res + [None]
