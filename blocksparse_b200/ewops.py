"""Bias + activation and dropout -- host side of the reference's blocksparse/ewops.py (bias_relu :307-350, dropout
:207-242) and of its entropy state (blocksparse/utils.py:21-39), on torch tensors, calling the sm_90a kernels of
csrc/ewops.cuh through bsmm_bias_relu / bsmm_bias_relu_grad / bsmm_dropout_mask / bsmm_dropout_apply.

The reference's other elementwise ops (add, multiply, sigmoid, float_cast, filter_tensor, add_n, concrete_gate,
fancy_gather, reduce_max, assign_add, ...) live in blocksparse_b200/elementwise.py, which also sets them as attributes of
this module, so that `from blocksparse_b200 import ewops as ew; ew.add(x, b)` reads as the reference does; they are not
listed in this module's __all__.
"""
import ctypes
import math

import torch

from . import _lib
from .transformer import _dense_bench, _on_device_of

__all__ = ["bias_relu", "dropout", "set_entropy", "get_entropy"]

ACT_NONE, ACT_RELU, ACT_FAST_GELU = 0, 1, 2
MAX_DIMS = 8                                  # DROP_MAX_DIMS of csrc/ewops.cuh


# ---- bias_relu --------------------------------------------------------------------------------------------------------
def _layout(x, axis):
    """(axis code of the C entry, N, K): 1 for the feature axis last (x viewed as (N, K)), 0 for the feature axis first
    (x viewed as (K, N)). Any other axis raises."""
    nd = x.dim()
    if not -nd <= axis < nd:
        raise ValueError("bias_relu: axis %d out of range for a tensor of rank %d" % (axis, nd))
    axis = axis % nd
    K = x.shape[axis]
    N = x.numel() // K if K else 0
    if axis == nd - 1:
        return 1, N, K
    if axis == 0:
        return 0, N, K
    raise ValueError("bias_relu: the feature axis must be 0 or the last one, got %d for shape %s" % (axis, tuple(x.shape)))


@_on_device_of
def _br_fwd(x, b, axis, N, K, act):
    y = torch.empty_like(x)
    if N == 0 or K == 0:
        return y
    rc = _lib.load().bsmm_bias_relu(_lib.dtype_code(x.dtype), _lib.dtype_code(b.dtype), axis, x.data_ptr(), b.data_ptr(),
                                    y.data_ptr(), N, K, act, _lib.stream_ptr())
    _lib.check(rc, "bsmm_bias_relu")
    return y


@_on_device_of
def _br_bwd(dy, src, b, axis, N, K, act):
    """(dx, db); without an activation dx is dy itself."""
    dx = dy if act == ACT_NONE else torch.empty_like(dy)
    db = torch.empty_like(b)
    if N == 0 or K == 0:
        return dx, db.zero_()
    ws = torch.empty(_lib.load().bsmm_bias_grad_workspace_bytes(axis, N, K) // 4, dtype=torch.float32, device=dy.device)
    rc = _lib.load().bsmm_bias_relu_grad(_lib.dtype_code(dy.dtype), _lib.dtype_code(b.dtype), axis, dy.data_ptr(),
                                         _lib.ptr(src), b.data_ptr(), None if act == ACT_NONE else dx.data_ptr(),
                                         db.data_ptr(), ws.data_ptr(), N, K, act, _lib.stream_ptr())
    _lib.check(rc, "bsmm_bias_relu_grad")
    return dx, db


def _br_tag(x, axis, act):
    return "bias_relu %s %s axis %d%s" % (tuple(x.shape), str(x.dtype).replace("torch.", ""), axis,
                                          ["", " relu", " fast_gelu"][act])


class _BiasReluFunction(torch.autograd.Function):
    """Saves y for relu and x for fast_gelu, nothing else for the identity (reference ewops.py:335-350)."""

    @staticmethod
    def forward(ctx, x, b, axis, N, K, act, bench):
        y = _br_fwd(x, b, axis, N, K, act)
        ctx.args = (axis, N, K, act)
        ctx.bench = bench
        ctx.save_for_backward(y if act == ACT_RELU else x if act == ACT_FAST_GELU else None, b)
        return y

    @staticmethod
    def backward(ctx, dy):
        src, b = ctx.saved_tensors
        dy = dy.contiguous()
        if ctx.bench:
            axis, N, K, act = ctx.args
            _dense_bench(_br_tag(dy, axis, act) + " grad", lambda: _br_bwd(dy, src, b, *ctx.args),
                         (1 if act == ACT_NONE else 3) * dy.numel() * dy.element_size(), ctx.bench)
        dx, db = _br_bwd(dy, src, b, *ctx.args)
        return dx, db, None, None, None, None, None


def bias_relu(x, b, axis=-1, relu=False, fast_gelu=False, atomics=True, bench=0, use_tf=False):
    """y = act(x + b) with b broadcast along `axis` (reference ewops.py:307-331); act is relu, fast_gelu
    z * sigmoid(1.702 z), or the identity. Returns y, differentiable in x and b.

    x: CUDA, fp32 / fp16 / bf16, with the feature axis last (any rank) or first (x viewed as (K, N), the layout of
    BlocksparseMatMul(feature_axis=0)); any other axis raises ValueError. b: K entries, fp32 / fp16 / bf16, read as fp32;
    db comes back in b's dtype. y is formed in fp32 and rounded once. db is reduced in a fixed order, so it is bitwise
    reproducible; `atomics` is accepted for compatibility and has no effect. bench > 0 times that many launches of the
    forward (and of the gradient, in the backward) and prints one line each. relu with fast_gelu, or use_tf=True, raises
    ValueError."""
    if relu and fast_gelu:
        raise ValueError("relu and fast_gelu can not both be enabled.")
    if use_tf:
        raise ValueError("bias_relu: use_tf is a TensorFlow composition; there is none here")
    if not torch.is_tensor(x) or not x.is_cuda:
        raise ValueError("bias_relu needs a CUDA tensor (there is no CPU path)")
    if x.dim() < 1:
        raise ValueError("bias_relu needs a tensor of rank >= 1")
    _lib.dtype_code(x.dtype)
    ax, N, K = _layout(x, int(axis))
    if K >= 2 ** 31:
        raise ValueError("bias_relu: the feature axis has %d entries, at most 2^31 - 1 are supported" % K)
    if not torch.is_tensor(b) or b.device != x.device:
        raise ValueError("bias_relu: b must be a tensor on x's device %s" % x.device)
    _lib.dtype_code(b.dtype)
    if b.numel() != K:
        raise ValueError("bias_relu: b has %d entries, the feature axis %d" % (b.numel(), K))
    b = b.contiguous().view(-1)
    x = x.contiguous()
    act = ACT_RELU if relu else ACT_FAST_GELU if fast_gelu else ACT_NONE
    if bench:
        _dense_bench(_br_tag(x, ax, act), lambda: _br_fwd(x, b, ax, N, K, act), 2 * x.numel() * x.element_size(), bench)
    return _BiasReluFunction.apply(x, b, ax, N, K, act, int(bench))


# ---- entropy ----------------------------------------------------------------------------------------------------------
_ENTROPY = {}                                  # device index -> int64 [seed, call] on that device


def _cuda_device(device):
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise ValueError("the dropout state lives on a CUDA device, got %s" % dev)
    return dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())


def set_entropy(init=None, device=None):
    """Seed the dropout state of `device` (default: the current one): an int64 tensor [seed, call] in device memory.
    init=None draws the seed from torch's default CPU generator, so torch.manual_seed makes runs reproducible. Each mask
    drawn advances call by one on the device; a mask depends on (seed, call, its size) only. Returns the state.

    Dropout calls that share a device's state must be stream-ordered, like any other in-place write. Not allowed during
    CUDA graph capture (ValueError); a captured dropout reads and advances the state each replay."""
    dev = _cuda_device(device)
    if torch.cuda.is_current_stream_capturing():
        raise ValueError("set_entropy: the dropout state cannot be created or reseeded during CUDA graph capture")
    if init is None:
        init = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64).item())
    seed = (int(init) + 2 ** 63) % 2 ** 64 - 2 ** 63
    host = torch.tensor([seed, 0], dtype=torch.int64)
    state = _ENTROPY.get(dev.index)
    if state is None:
        state = _ENTROPY[dev.index] = host.to(dev)
    else:
        state.copy_(host)                      # in place: graphs that captured the state keep reading it
    return state


def get_entropy(device=None):
    """The dropout state of `device` (default: the current one), created by set_entropy() on first use. Clone it to
    checkpoint the random stream and copy_ the clone back to restore it."""
    dev = _cuda_device(device)
    state = _ENTROPY.get(dev.index)
    return set_entropy(None, dev) if state is None else state


# ---- dropout ----------------------------------------------------------------------------------------------------------
def _mask_strides(x, mask_shape):
    """Row-major strides of mask_shape, 0 on the dims the mask broadcasts over."""
    strides, s = [0] * len(mask_shape), 1
    for d in reversed(range(len(mask_shape))):
        strides[d] = s if mask_shape[d] != 1 else 0
        s *= mask_shape[d]
    return strides


@_on_device_of
def _gen_mask(x, M, keep_prob):
    mask = torch.empty((M + 31) // 32, dtype=torch.int32, device=x.device)
    if M:
        state = get_entropy(x.device)
        rc = _lib.load().bsmm_dropout_mask(mask.data_ptr(), M, keep_prob, state.data_ptr(), _lib.stream_ptr())
        _lib.check(rc, "bsmm_dropout_mask")
    return mask


@_on_device_of
def _mask_at(x, M, keep_prob, state):
    """The mask _gen_mask would draw for M elements if the device state held `state` (int64 [seed, call] on x's device).
    It is drawn from a copy, so neither `state` nor the device state moves: a backward or a recomputation redraws the
    mask of its forward from a snapshot."""
    mask = torch.empty((M + 31) // 32, dtype=torch.int32, device=x.device)
    if M:
        rc = _lib.load().bsmm_dropout_mask(mask.data_ptr(), M, keep_prob, state.clone().data_ptr(), _lib.stream_ptr())
        _lib.check(rc, "bsmm_dropout_mask")
    return mask


@_on_device_of
def _apply_mask(x, mask, shape, strides, keep_prob):
    y = torch.empty_like(x)
    if x.numel() == 0:
        return y
    nd = len(shape)
    arr = ctypes.c_longlong * max(nd, 1)
    rc = _lib.load().bsmm_dropout_apply(_lib.dtype_code(x.dtype), x.data_ptr(), mask.data_ptr(), y.data_ptr(), nd,
                                        arr(*shape), arr(*strides), mask.numel(), keep_prob, _lib.stream_ptr())
    _lib.check(rc, "bsmm_dropout_apply")
    return y


class _DropoutFunction(torch.autograd.Function):
    """The backward applies the same mask to dy (reference ewops.py:236-242)."""

    @staticmethod
    def forward(ctx, x, mask, shape, strides, keep_prob):
        ctx.args = (shape, strides, keep_prob)
        ctx.save_for_backward(mask)
        return _apply_mask(x, mask, *ctx.args)

    @staticmethod
    def backward(ctx, dy):
        mask, = ctx.saved_tensors
        return _apply_mask(dy.contiguous(), mask, *ctx.args), None, None, None, None


def dropout(x, keep_prob, mask=None, mask_shape=None):
    """(y, mask): y = x * (1 / keep_prob) where the mask keeps an element, +0 where it drops it (reference
    ewops.py:214-234); differentiable in x, with the same mask applied to the gradient.

    x: CUDA, fp32 / fp16 / bf16, rank <= 8. keep_prob: a Python float in (0, 1] (ValueError otherwise). The mask is the
    reference's format: a 1-D int32 tensor of ceil(M / 32) words, bit e % 32 of word e / 32 set = keep element e of the
    mask flattened in row-major order, M = prod(mask_shape) (x.numel() without one). mask_shape has x's rank and each of
    its dims is 1 (broadcast) or x's. Without `mask` a new one is drawn from this device's state (see set_entropy):
    element e is kept iff its Philox4x32-10 word is below floor(keep_prob * 2^32). A given `mask` is checked (int32,
    x's device, ceil(M / 32) words) and applied as it is, so a recomputed block reuses its forward's mask. Kept values
    are round(fp32(x) * fp32(1 / keep_prob))."""
    if not isinstance(keep_prob, (int, float)) or isinstance(keep_prob, bool):
        raise ValueError("dropout: keep_prob must be a Python float, got %r" % (keep_prob,))
    kp = float(keep_prob)
    if not 0.0 < kp <= 1.0:
        raise ValueError("dropout: keep_prob must be in (0, 1], got %r" % (keep_prob,))
    if not torch.is_tensor(x) or not x.is_cuda:
        raise ValueError("dropout needs a CUDA tensor (there is no CPU path)")
    _lib.dtype_code(x.dtype)
    if x.dim() > MAX_DIMS:
        raise ValueError("dropout: x has rank %d, at most %d is supported" % (x.dim(), MAX_DIMS))
    shape = tuple(x.shape)
    if mask_shape is not None and len(mask_shape) > 0:
        ms = tuple(int(d) for d in mask_shape)
        if len(ms) != len(shape) or any(m != 1 and m != s for m, s in zip(ms, shape)):
            raise ValueError("dropout: incompatible mask_shape %s for x of shape %s" % (ms, shape))
    else:
        ms = shape
    M = math.prod(ms)
    words = (M + 31) // 32
    if mask is None:
        mask = _gen_mask(x, M, kp)
    elif not torch.is_tensor(mask) or mask.dtype != torch.int32 or mask.device != x.device or mask.dim() != 1 \
            or mask.numel() != words:
        raise ValueError("dropout: mask must be a 1-D int32 tensor of %d words on %s, got %s" % (
            words, x.device, (mask.dtype, mask.device, tuple(mask.shape)) if torch.is_tensor(mask) else type(mask)))
    y = _DropoutFunction.apply(x.contiguous(), mask.contiguous(), shape, _mask_strides(x, ms), kp)
    return y, mask
