"""ctypes binding of bsref_dw_matmul_large_n in oracle/_ref/libbsref.so (oracle/ref/matmul.cu): the reference's own
Gemm_TN launcher behind dw_matmul_large_n, built for sm_90a, with the argument checks of DwMatmulLargeNOp (matmul_op.cc)
and the plumbing of oracle/ref_kernels.py. Only the test suite imports this module."""
import ctypes
import math

import torch

from . import ref_kernels as rk

_u, _i, _p = ctypes.c_uint, ctypes.c_int, ctypes.c_void_p
SIGNATURES = {"bsref_dw_matmul_large_n": [_i, _p, _p, _p, _u, _u, _u, _p]}

_FN = None


def missing():
    """Why bsref_dw_matmul_large_n cannot be called here, or None when it can: the library may be absent (no reference
    checkout where it was built) or built by an oracle/ref that did not yet have matmul.cu."""
    if not rk.available():
        return "oracle/_ref/libbsref.so not built (no reference checkout)"
    if not hasattr(rk.load(), "bsref_dw_matmul_large_n"):
        return ("oracle/_ref/libbsref.so was built without oracle/ref/matmul.cu and has no bsref_dw_matmul_large_n; "
                "rebuild it with make -C oracle/ref REF=<reference checkout>")
    return None


def available():
    return missing() is None


def _fn():
    global _FN
    if _FN is None:
        fn = rk.load().bsref_dw_matmul_large_n
        fn.argtypes = SIGNATURES["bsref_dw_matmul_large_n"]
        fn.restype = _i
        _FN = fn
    return _FN


def dw_matmul_large_n(x, e):
    """U (fp32 [C, K]) = x^T e over the leading dims, fp32 or fp16, as the reference's op computes it: C and K multiples
    of 4, N a multiple of 32, and the launcher's 32-bit offsets."""
    x, e = rk._dev(x, e)
    if x.dtype != e.dtype or x.dtype not in (torch.float32, torch.float16):
        raise ValueError("DwMatmulLargeN takes x and e of one dtype, float or half")
    if x.dim() != e.dim() or x.shape[:-1] != e.shape[:-1]:
        raise ValueError("Mismatched Shapes")
    C, K, N = x.shape[-1], e.shape[-1], math.prod(x.shape[:-1])
    if C % 4 or K % 4:
        raise ValueError("Channel dims must be multiple of 4")
    if N % 32:
        raise ValueError("Minibatch dim must be multiple of 32")
    rk._u32("N * C", N * C)
    rk._u32("N * K", N * K)
    rk._u32("C * K", C * K)
    out = rk._Out((C, K), torch.float32, x.device)
    rc = _fn()(rk._dt(x), out.t.data_ptr(), x.data_ptr(), e.data_ptr(), C, K, N, rk._stream())
    if rc != 0:
        raise RuntimeError("bsref_dw_matmul_large_n: CUDA error %d" % rc)
    torch.cuda.current_stream().synchronize()
    return out.check("bsref_dw_matmul_large_n")
