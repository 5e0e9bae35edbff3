"""Layer norm -- host side of the reference's blocksparse/norms.py (layer_norm :23-67 and its gradient), on torch tensors,
calling the sm_90a kernels of csrc/layer_norm.cuh through bsmm_layer_norm / bsmm_layer_norm_grad.

The reference's batch_norm ops are NCDHW kernels of its conv module and are not carried here.
"""
import torch

from . import _lib
from .checkers import layer_norm_grad_test, layer_norm_test  # noqa: F401  (the reference defines them in norms.py)
from .transformer import _dense_bench, _on_device_of


def _layout(x, axis):
    """(axis code of the C entry, N, K): 1 for the feature axis last (x viewed as (N, K)), 0 for the feature axis first
    (x viewed as (K, N)). Any other axis raises: the reference would run its axis-0 kernel on it as if x were (K, N)."""
    nd = x.dim()
    if not -nd <= axis < nd:
        raise ValueError("layer_norm: axis %d out of range for a tensor of rank %d" % (axis, nd))
    axis = axis % nd
    K = x.shape[axis]
    N = x.numel() // K if K else 0
    if axis == nd - 1:
        return 1, N, K
    if axis == 0:
        return 0, N, K
    raise ValueError("layer_norm: the feature axis must be 0 or the last one, got %d for shape %s" % (axis, tuple(x.shape)))


def _param(p, K, x, what):
    if not torch.is_tensor(p) or p.device != x.device:
        raise ValueError("layer_norm: %s must be a tensor on x's device %s" % (what, x.device))
    _lib.dtype_code(p.dtype)
    if p.numel() != K:
        raise ValueError("layer_norm: %s has %d entries, the feature axis %d" % (what, p.numel(), K))
    return p.contiguous().view(-1)


def _workspace(axis, N, K, S, device):
    n = _lib.load().bsmm_layer_norm_workspace_bytes(axis, N, K, S) // 4
    return torch.empty(max(n, 1), dtype=torch.float32, device=device)


@_on_device_of
def _ln_fwd(x, g, b, axis, N, K, S, eps, relu):
    y = torch.empty_like(x)
    stats = N * S if axis else N
    mean = torch.empty(stats, dtype=torch.float32, device=x.device)
    rstd = torch.empty_like(mean)
    if N == 0:
        return y, mean, rstd
    ws = _workspace(axis, N, K, S, x.device) if axis == 0 else None
    rc = _lib.load().bsmm_layer_norm(_lib.dtype_code(x.dtype), _lib.dtype_code(g.dtype), axis, x.data_ptr(), g.data_ptr(),
                                     b.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(), _lib.ptr(ws), N, K, S,
                                     float(eps), int(relu), _lib.stream_ptr())
    _lib.check(rc, "bsmm_layer_norm")
    return y, mean, rstd


@_on_device_of
def _ln_bwd(x, dy, g, b, mean, rstd, axis, N, K, S, eps, relu):
    dy = dy.to(x.dtype).contiguous()
    dx = torch.empty_like(x)
    dg, db = torch.empty_like(g), torch.empty_like(b)
    if N == 0:
        return dx, dg.zero_(), db.zero_()
    ws = _workspace(axis, N, K, S, x.device)
    rc = _lib.load().bsmm_layer_norm_grad(_lib.dtype_code(x.dtype), _lib.dtype_code(g.dtype), axis, dy.data_ptr(),
                                          x.data_ptr(), g.data_ptr(), b.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                          dx.data_ptr(), dg.data_ptr(), db.data_ptr(), ws.data_ptr(), N, K, S, float(eps),
                                          int(relu), _lib.stream_ptr())
    _lib.check(rc, "bsmm_layer_norm_grad")
    return dx, dg, db


def _tag(x, axis, S, relu):
    return "layer_norm %s %s axis %d segments %d%s" % (tuple(x.shape), str(x.dtype).replace("torch.", ""), axis, S,
                                                        " relu" if relu else "")


class _LayerNormFunction(torch.autograd.Function):
    """Saves x, g, b and the fp32 mean / rstd (one per segment and row); the backward recomputes xhat and, with relu,
    the fp32 pre-activation for the mask (reference norms.py:56-67, 156-168)."""

    @staticmethod
    def forward(ctx, x, g, b, axis, N, K, S, eps, relu, bench):
        y, mean, rstd = _ln_fwd(x, g, b, axis, N, K, S, eps, relu)
        ctx.args = (axis, N, K, S, eps, relu)
        ctx.bench = bench
        ctx.save_for_backward(x, g, b, mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, g, b, mean, rstd = ctx.saved_tensors
        if ctx.bench:
            axis, N, K, S, eps, relu = ctx.args
            _dense_bench(_tag(x, axis, S, relu) + " grad", lambda: _ln_bwd(x, dy, g, b, mean, rstd, *ctx.args),
                         3 * x.numel() * x.element_size(), ctx.bench)
        dx, dg, db = _ln_bwd(x, dy, g, b, mean, rstd, *ctx.args)
        return dx, dg, db, None, None, None, None, None, None, None


def layer_norm(x, g, b, axis=1, segments=1, epsilon=1e-6, relu=False, atomics=True, bench=0, use_tf=False):
    """y = relu?((x - mean) * rsqrt(var + epsilon) * g + b), the statistics taken along `axis` per segment of
    K / segments features (reference norms.py:23-53). Returns y, differentiable in x, g and b.

    x: CUDA, fp32 / fp16 / bf16, with the feature axis last (any rank) or first (x viewed as (K, N), the layout of
    BlocksparseMatMul(feature_axis=0)); any other axis raises ValueError. g, b: K entries each, fp32 / fp16 / bf16, read
    as fp32; dg and db come back in their dtypes. segments needs the last axis. Mean and variance are formed in fp32
    without E[x^2] - E[x]^2, and dg / db are reduced in a fixed order, so results are bitwise reproducible; `atomics` is
    accepted for compatibility and has no effect. bench > 0 times that many launches of the forward (and of the
    gradient, in the backward) and prints one line each. use_tf=True raises ValueError."""
    if use_tf:
        raise ValueError("layer_norm: use_tf is a TensorFlow composition; there is none here")
    if not torch.is_tensor(x) or not x.is_cuda:
        raise ValueError("layer_norm needs a CUDA tensor (there is no CPU path)")
    if x.dim() < 1:
        raise ValueError("layer_norm needs a tensor of rank >= 1")
    _lib.dtype_code(x.dtype)
    ax, N, K = _layout(x, int(axis))
    S = int(segments)
    if K == 0 or S < 1 or K % S:
        raise ValueError("layer_norm: %d features do not split into %d segments" % (K, S))
    if ax == 0 and S != 1:
        raise ValueError("layer_norm: segments need the feature axis last")
    g, b = _param(g, K, x, "g"), _param(b, K, x, "b")
    if g.dtype != b.dtype:
        raise ValueError("layer_norm: g and b must share a dtype, got %s and %s" % (g.dtype, b.dtype))
    x = x.contiguous()
    if bench:
        _dense_bench(_tag(x, ax, S, relu), lambda: _ln_fwd(x, g, b, ax, N, K, S, epsilon, relu),
                     2 * x.numel() * x.element_size(), bench)
    return _LayerNormFunction.apply(x, g, b, ax, N, K, S, float(epsilon), bool(relu), int(bench))
