"""fp8 block-sparse matmul on the H100's fp8 tensor cores.

  quantize_fp8(x, dtype=torch.float8_e4m3fn) -> (q, scale_inv)
        per-tensor quantisation with the current amax: q = fp8(x * FP8_MAX / amax), scale_inv = amax / FP8_MAX, so that
        x ~= q * scale_inv (bsmm_fp8_quantize; the exact rounding and special cases are in include/bsmm_b200.h).
  quantize_fp8_weights(bsmm, w, dtype=torch.float8_e4m3fn) -> (wq, wq_t, scale_inv)
        the same over a (blocks, bs, bs) weight tensor: wq holds the blocks as stored, wq_t each block transposed.
  quantize_fp8_t(x, dtype=torch.float8_e4m3fn, with_rows=True) -> (q or None, q_t, scale_inv)
        quantize_fp8 of a 2-D (rows, cols) tensor that also writes the transpose q_t (cols, pitch), pitch = rows
        rounded up to 16, zero past `rows`: the feature-major operand updat_fp8 reads. q is quantize_fp8's output
        byte for byte (None with with_rows=False) and q_t[:, :rows] is q.T.
  xprop_fp8(bsmm, x, w, x_scale_inv, w_scale_inv, bprop=False, out_dtype=torch.bfloat16) -> y
        fprop (x = quantised activations, w = wq_t) or bprop (x = quantised output gradient, w = wq) of the
        BlocksparseMatMul `bsmm`, y = (x . w) * x_scale_inv * w_scale_inv in fp16 / bf16.
  updat_fp8(bsmm, xts, dyts, x_scale_invs, dy_scale_invs, N, dw=None, dw_dtype=torch.bfloat16) -> dw
        weight gradient of `bsmm` from 1..8 pairs of feature-major fp8 operands (quantize_fp8_t's q_t of x and dy),
        dw = sum_p (xt_p . dyt_p^T) * x_scale_inv_p * dy_scale_inv_p over the first N columns (+ dw when given).

BlocksparseMatMul.matmul_fp8(I, W, fp8_dw=False) is the autograd op built from these. Feature axis 1 and block sizes
32 / 64 only. scale_inv stays on the device, so nothing here synchronises the host and every call is CUDA-graph
capturable. See DESIGN.md 6e and 6f.
"""
import torch

from . import _lib

__all__ = ["quantize_fp8", "quantize_fp8_t", "quantize_fp8_weights", "xprop_fp8", "updat_fp8"]

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


def t_pitch(rows):
    """Row pitch of quantize_fp8_t's q_t: rows rounded up to 16 (TMA needs 16-byte row strides)."""
    return (int(rows) + 15) // 16 * 16


def quantize_fp8_t(x, dtype=torch.float8_e4m3fn, with_rows=True):
    """(q, q_t, scale_inv) of a 2-D tensor x (rows, cols): q (rows, cols) is quantize_fp8(x, dtype)'s q byte for byte
    (None with with_rows=False), q_t (cols, pitch) holds q.T in its first `rows` columns and zeros after them, and
    scale_inv is the fp32 (1,) tensor that dequantises both. One amax pass and one cast pass write q and q_t."""
    code = _lib.fp8_code(dtype)
    if torch.is_tensor(x) and x.dim() != 2:
        raise ValueError("quantize_fp8_t takes a 2-D (rows, cols) tensor, got shape %s" % (tuple(x.shape),))
    _check_src(x, "quantize_fp8_t")
    x = x.detach().contiguous()
    rows, cols = x.shape
    pitch = t_pitch(rows)
    q = torch.empty((rows, cols), dtype=dtype, device=x.device) if with_rows else None
    # at least 16 bytes, so that the call has an output to write even when there are no elements
    buf = torch.empty(max(cols * pitch, 16), dtype=dtype, device=x.device)
    q_t = buf[:cols * pitch].view(cols, pitch)
    scales = torch.empty(2, dtype=torch.float32, device=x.device)      # amax, scale_inv
    with torch.cuda.device(x.device):
        rc = _lib.load().bsmm_fp8_quantize_t(_lib.dtype_code(x.dtype), code, x.data_ptr(), rows, cols, scales.data_ptr(),
                                             scales.data_ptr() + 4, _lib.ptr(q), buf.data_ptr(), pitch, _lib.stream_ptr())
    _lib.check(rc, "bsmm_fp8_quantize_t")
    return q, q_t, scales[1:]


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


def _as_list(t):
    return [t] if torch.is_tensor(t) else list(t)


def updat_fp8(bsmm, xts, dyts, x_scale_invs, dy_scale_invs, N, dw=None, dw_dtype=torch.bfloat16):
    """Weight gradient of `bsmm` on fp8 tensor cores: dw[w] = sum_p xt_p[c-blk] . dyt_p[k-blk]^T * x_scale_inv_p *
    dy_scale_inv_p over the first N columns, added to `dw` in place when it is given (else a new `dw_dtype` tensor).

    xts[p] (C, pitch) and dyts[p] (K, pitch) are feature-major fp8 operands (quantize_fp8_t's q_t of x (N, C) and of
    dy (N, K)), all with one pitch (a multiple of 16, at least N); 1..8 pairs, each with its own fp32 scale_inv
    tensors. The operands carry the feature axis themselves, so bsmm.axis is not read. Block sizes 32 / 64 only."""
    if bsmm.bsize not in (32, 64):
        raise ValueError("updat_fp8 needs block size 32 or 64, got %d" % bsmm.bsize)
    xts, dyts = _as_list(xts), _as_list(dyts)
    xsi, dsi = _as_list(x_scale_invs), _as_list(dy_scale_invs)
    if not 1 <= len(xts) <= _lib.MAX_PAIRS or not len(xts) == len(dyts) == len(xsi) == len(dsi):
        raise ValueError("updat_fp8 takes 1..%d pairs with one x and one dy scale_inv each, got %d xts, %d dyts, %d and "
                         "%d scales" % (_lib.MAX_PAIRS, len(xts), len(dyts), len(xsi), len(dsi)))
    for t in xts + dyts + xsi + dsi:
        if not torch.is_tensor(t):
            raise ValueError("updat_fp8 takes tensors, got %r" % (type(t),))
    x0 = xts[0]
    if x0.dim() != 2:
        raise ValueError("xts must be 2-D (C, pitch), got shape %s" % (tuple(x0.shape),))
    pitch = x0.shape[1]
    N = int(N)
    if N < 0:
        raise ValueError("N must be >= 0, got %d" % N)
    if pitch % 16 or pitch < N:
        raise ValueError("the operands' pitch must be a multiple of 16 and at least N = %d, got %d" % (N, pitch))
    for ts, feat, what in ((xts, bsmm.C, "xts"), (dyts, bsmm.K, "dyts")):
        for t in ts:
            if t.dtype not in FP8_DTYPES:
                raise ValueError("%s must be float8_e4m3fn / float8_e5m2, got %s" % (what, t.dtype))
            if t.dtype != ts[0].dtype:
                raise ValueError("all %s must share one dtype" % what)
            if tuple(t.shape) != (feat, pitch) or not t.is_contiguous():
                raise ValueError("%s must be contiguous (%d, %d) tensors, got %s" % (what, feat, pitch, tuple(t.shape)))
    for t in xsi + dsi:
        if t.dtype != torch.float32 or t.numel() < 1:
            raise ValueError("scale_inv must be a float32 tensor with one element")
    if dw is not None:
        if tuple(dw.shape) != bsmm.w_shape or not dw.is_contiguous() or dw.dtype not in _SRC_DTYPES:
            raise ValueError("dw must be a contiguous float32 / float16 / bfloat16 tensor of shape %s" % (bsmm.w_shape,))
    elif dw_dtype not in _SRC_DTYPES:
        raise ValueError("updat_fp8 writes float32, float16 or bfloat16, not %s" % (dw_dtype,))
    if not x0.is_cuda:
        raise _lib.BsmmError("updat_fp8 needs CUDA tensors (no CPU path)")
    for t in xts + dyts + xsi + dsi + ([dw] if dw is not None else []):
        if t.device != x0.device:
            raise ValueError("updat_fp8: operands live on %s and %s" % (x0.device, t.device))
    beta = 0.0 if dw is None else 1.0
    if dw is None:
        dw = torch.empty(bsmm.w_shape, dtype=dw_dtype, device=x0.device)
    d = bsmm._device_luts(x0.device)
    with torch.cuda.device(x0.device):
        rc = _lib.load().bsmm_updat_fp8(_lib.fp8_code(x0.dtype), _lib.fp8_code(dyts[0].dtype), _lib.dtype_code(dw.dtype),
                                        bsmm.bsize, bsmm.blocks, bsmm.CB, bsmm.KB, _lib.ptr_array(xts),
                                        _lib.ptr_array(dyts), _lib.ptr_array(xsi), _lib.ptr_array(dsi), len(xts),
                                        dw.data_ptr(), N, pitch, beta, d["updat_sched"].data_ptr(), d["updat_tiles"],
                                        d["updat_kt"], _lib.stream_ptr())
    _lib.check(rc, "bsmm_updat_fp8")
    return dw
