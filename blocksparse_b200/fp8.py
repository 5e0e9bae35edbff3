"""fp8 block-sparse matmul on the H100's fp8 tensor cores.

  quantize_fp8(x, dtype=torch.float8_e4m3fn) -> (q, scale_inv)
        per-tensor quantisation with the current amax: q = fp8(x * FP8_MAX / amax), scale_inv = amax / FP8_MAX, so that
        x ~= q * scale_inv (bsmm_fp8_quantize; the exact rounding and special cases are in include/bsmm_b200.h).
  quantize_fp8_weights(bsmm, w, dtype=torch.float8_e4m3fn) -> (wq, wq_t, scale_inv)
        the same over a (blocks, bs, bs) weight tensor: wq holds the blocks as stored, wq_t each block transposed.
  xprop_fp8(bsmm, x, w, x_scale_inv, w_scale_inv, bprop=False, out_dtype=torch.bfloat16) -> y
        fprop (x = quantised activations, w = wq_t) or bprop (x = quantised output gradient, w = wq) of the
        BlocksparseMatMul `bsmm`, y = (x . w) * x_scale_inv * w_scale_inv in fp16 / bf16.

BlocksparseMatMul.matmul_fp8(I, W) is the autograd op built from these. Feature axis 1 and block sizes 32 / 64 only.
scale_inv stays on the device, so nothing here synchronises the host and every call is CUDA-graph capturable.
See DESIGN.md 6e.
"""
import torch

from . import _lib

__all__ = ["quantize_fp8", "quantize_fp8_weights", "xprop_fp8"]

FP8_DTYPES = (torch.float8_e4m3fn, torch.float8_e5m2)
FP8_MAX = {torch.float8_e4m3fn: 448.0, torch.float8_e5m2: 57344.0}
_SRC_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def _check_src(t, what):
    if not torch.is_tensor(t):
        raise ValueError("%s takes a tensor, got %r" % (what, type(t)))
    if t.dtype not in _SRC_DTYPES:
        raise ValueError("%s takes float32, float16 or bfloat16, got %s" % (what, t.dtype))
    if not t.is_cuda:
        raise _lib.BsmmError("%s needs CUDA tensors (no CPU path)" % what)


def quantize_fp8(x, dtype=torch.float8_e4m3fn):
    """(q, scale_inv): x cast to fp8 `dtype` (same shape, contiguous) with one scale for the whole tensor, and the fp32
    scale_inv (shape (1,), on x's device) that dequantises it."""
    code = _lib.fp8_code(dtype)
    _check_src(x, "quantize_fp8")
    x = x.detach().contiguous()
    q = torch.empty(x.shape, dtype=dtype, device=x.device)
    scales = torch.empty(2, dtype=torch.float32, device=x.device)      # amax, scale_inv
    with torch.cuda.device(x.device):
        rc = _lib.load().bsmm_fp8_quantize(_lib.dtype_code(x.dtype), code, x.data_ptr(), x.numel(), scales.data_ptr(),
                                           scales.data_ptr() + 4, q.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "bsmm_fp8_quantize")
    return q, scales[1:]


def quantize_fp8_weights(bsmm, w, dtype=torch.float8_e4m3fn):
    """(wq, wq_t, scale_inv) of the (blocks, bs, bs) weights `w` of `bsmm`: wq the blocks as stored (bprop reads
    them), wq_t each block transposed (fprop reads them), both fp8 `dtype`, and the fp32 scale_inv of shape (1,)."""
    code = _lib.fp8_code(dtype)
    if bsmm.bsize not in (32, 64):
        raise ValueError("fp8 weights need block size 32 or 64, got %d" % bsmm.bsize)
    _check_src(w, "quantize_fp8_weights")
    if tuple(w.shape) != bsmm.w_shape:
        raise ValueError("w must have shape %s, got %s" % (bsmm.w_shape, tuple(w.shape)))
    w = w.detach().contiguous()
    wq = torch.empty(bsmm.w_shape, dtype=dtype, device=w.device)
    wq_t = torch.empty(bsmm.w_shape, dtype=dtype, device=w.device)
    scales = torch.empty(2, dtype=torch.float32, device=w.device)
    with torch.cuda.device(w.device):
        rc = _lib.load().bsmm_fp8_weights(_lib.dtype_code(w.dtype), code, bsmm.bsize, bsmm.blocks, w.data_ptr(),
                                          scales.data_ptr(), scales.data_ptr() + 4, wq.data_ptr(), wq_t.data_ptr(),
                                          _lib.stream_ptr())
    _lib.check(rc, "bsmm_fp8_weights")
    return wq, wq_t, scales[1:]


def check_config(bsmm):
    if bsmm.axis != 1:
        raise ValueError("the fp8 path needs feature_axis 1 (its activations must be K-major), got 0")
    if bsmm.bsize not in (32, 64):
        raise ValueError("the fp8 path needs block size 32 or 64, got %d" % bsmm.bsize)


def xprop_fp8(bsmm, x, w, x_scale_inv, w_scale_inv, bprop=False, out_dtype=torch.bfloat16):
    """fprop (bprop=False: x (..., C), w = wq_t) or bprop (bprop=True: x (..., K), w = wq) of `bsmm` on fp8 operands;
    returns y (..., K) or (..., C) in `out_dtype` (float16 or bfloat16), scaled by x_scale_inv * w_scale_inv."""
    check_config(bsmm)
    if x.dtype not in FP8_DTYPES or w.dtype not in FP8_DTYPES:
        raise ValueError("xprop_fp8 takes float8_e4m3fn / float8_e5m2 x and w, got %s and %s" % (x.dtype, w.dtype))
    if out_dtype not in (torch.float16, torch.bfloat16):
        raise ValueError("xprop_fp8 writes float16 or bfloat16, not %s" % (out_dtype,))
    if not x.is_cuda:
        raise _lib.BsmmError("xprop_fp8 needs CUDA tensors (no CPU path)")
    feat_in, feat_out = (bsmm.K, bsmm.C) if bprop else (bsmm.C, bsmm.K)
    if x.dim() < 1 or x.shape[-1] != feat_in:
        raise ValueError("expected feature dim %d on the last axis, got shape %s" % (feat_in, tuple(x.shape)))
    if tuple(w.shape) != bsmm.w_shape:
        raise ValueError("w must have shape %s, got %s" % (bsmm.w_shape, tuple(w.shape)))
    for t in (w, x_scale_inv, w_scale_inv):
        if t.device != x.device:
            raise ValueError("xprop_fp8: operands live on %s and %s" % (x.device, t.device))
    for t in (x_scale_inv, w_scale_inv):
        if t.dtype != torch.float32 or t.numel() < 1:
            raise ValueError("scale_inv must be a float32 tensor with one element")
    x2 = x.reshape(-1, feat_in).contiguous()
    w = w.contiguous()
    N = x2.shape[0]
    y = torch.empty((N, feat_out), dtype=out_dtype, device=x.device)
    d = bsmm._device_luts(x.device)
    n_in, n_out = (bsmm.KB, bsmm.CB) if bprop else (bsmm.CB, bsmm.KB)
    with torch.cuda.device(x.device):
        rc = _lib.load().bsmm_xprop_fp8(_lib.fp8_code(x.dtype), _lib.fp8_code(w.dtype), _lib.dtype_code(out_dtype), 1,
                                        bsmm.bsize, int(bool(bprop)), d["bprop" if bprop else "fprop"].data_ptr(), n_out,
                                        n_in, bsmm.blocks, x2.data_ptr(), w.data_ptr(), y.data_ptr(), N,
                                        x_scale_inv.data_ptr(), w_scale_inv.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "bsmm_xprop_fp8")
    return y.reshape(tuple(x.shape[:-1]) + (feat_out,))
