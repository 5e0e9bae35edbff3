"""LSTM gates, split4 / concat4 and sparse relu -- host side of the reference's blocksparse/lstm.py (fused_lstm_gates
:22-69, split4 / concat4 :72-91, sparse_relu :94-117), on torch tensors, calling the sm_90a kernels of csrc/lstm.cuh
through bsmm_lstm_gates / bsmm_lstm_gates_grad / bsmm_sparse_relu / bsmm_relu_mask_grad.

The reference's grouped_lstm and FusedBasicLSTMCell live in lstm_layer.py and are reachable here too (not listed in
__all__). Its group_lstm_grads is TensorFlow graph surgery and is not carried: grouped_lstm's backward forms the
kernel's gradient as one dw_matmul_large_n over all steps, the work that rewrite does.
"""
import numbers

import torch

from . import _lib
from .checkers import sparse_relu_test  # noqa: F401  (the reference defines it in lstm.py)
from .ewops import ACT_NONE, _br_bwd
from .transformer import _on_device_of, _transpose_0213

__all__ = ["fused_lstm_gates", "split4", "concat4", "sparse_relu"]


def _dt(t):
    return _lib.dtype_code(t.dtype)


def _gate_ptrs(gates, K):
    """(i, u, f, o pointers, row stride): the four column blocks of one (N, 4K) tensor, or four (N, K) tensors."""
    if len(gates) == 1:
        p, es = gates[0].data_ptr(), gates[0].element_size()
        return [p + j * K * es for j in range(4)], 4 * K
    return [g.data_ptr() for g in gates], K


# ---- fused_lstm_gates -------------------------------------------------------------------------------------------------
@_on_device_of
def _gates_fwd(c, gates, bias, N, K, forget_bias):
    c_next, h_next = torch.empty_like(c), torch.empty_like(c)
    if N == 0:
        return c_next, h_next
    ptrs, stride = _gate_ptrs(gates, K)
    rc = _lib.load().bsmm_lstm_gates(_dt(c), _lib.F32 if bias is None else _dt(bias), c.data_ptr(), *ptrs, stride,
                                     _lib.ptr(bias), c_next.data_ptr(), h_next.data_ptr(), N, K, forget_bias,
                                     _lib.stream_ptr())
    _lib.check(rc, "bsmm_lstm_gates")
    return c_next, h_next


@_on_device_of
def _gates_bwd(c, gates, bias, ec, eh, N, K, forget_bias):
    """(dc, [dh] or [di, du, df, do]); ec / eh None read as zero."""
    dc = torch.empty_like(c)
    dg = [torch.empty_like(g) for g in gates]
    if N == 0:
        return dc.zero_(), [d.zero_() for d in dg]
    ptrs, stride = _gate_ptrs(gates, K)
    dptrs, _ = _gate_ptrs(dg, K)
    rc = _lib.load().bsmm_lstm_gates_grad(_dt(c), _lib.F32 if bias is None else _dt(bias), c.data_ptr(), *ptrs, stride,
                                          _lib.ptr(bias), _lib.ptr(ec), _lib.ptr(eh), dc.data_ptr(), *dptrs, N, K,
                                          forget_bias, _lib.stream_ptr())
    _lib.check(rc, "bsmm_lstm_gates_grad")
    return dc, dg


class _LstmGatesFunction(torch.autograd.Function):
    """Saves the inputs only; the backward recomputes the gates (reference lstm_op_gpu.cu LSTM_Backward). Inputs after
    the constants: c, the gate tensor(s), then the bias when there is one."""

    @staticmethod
    def forward(ctx, N, K, forget_bias, has_bias, c, *rest):
        gates, bias = (rest[:-1], rest[-1]) if has_bias else (rest, None)
        ctx.set_materialize_grads(False)
        ctx.args = (N, K, forget_bias, has_bias)
        ctx.save_for_backward(c, *rest)
        return _gates_fwd(c, gates, bias, N, K, forget_bias)

    @staticmethod
    def backward(ctx, ec, eh):
        N, K, forget_bias, has_bias = ctx.args
        c, *rest = ctx.saved_tensors
        gates, bias = (rest[:-1], rest[-1]) if has_bias else (rest, None)
        if ec is None and eh is None:
            return (None,) * (5 + len(rest))
        ec = None if ec is None else ec.to(c.dtype).contiguous()
        eh = None if eh is None else eh.to(c.dtype).contiguous()
        dc, dg = _gates_bwd(c, gates, bias, ec, eh, N, K, forget_bias)
        db = None
        if has_bias and ctx.needs_input_grad[-1]:
            # the column sums of dh as stored, in bias_relu's fixed order: bitwise its db for the same dh
            db = _br_bwd(dg[0].view(N, 4 * K), None, bias, 1, N, 4 * K, ACT_NONE)[1]
        return (None, None, None, None, dc) + tuple(dg) + ((db,) if has_bias else ())


def _cuda(t, what):
    if not torch.is_tensor(t) or not t.is_cuda:
        raise ValueError("%s needs CUDA tensors (there is no CPU path)" % what)
    _lib.dtype_code(t.dtype)
    return t


def fused_lstm_gates(c, *args, bias=None, forget_bias=1.0, name=None):
    """(c_next, h_next) of one LSTM cell step (reference lstm.py:22-45), differentiable in every tensor input:
        c_next = sigmoid(f + b_f + forget_bias) * c + sigmoid(i + b_i) * tanh(u + b_u)
        h_next = sigmoid(o + b_o) * tanh(c_next)
    formed in fp32 with accurate expf / tanhf, each output rounded once.

    fused_lstm_gates(c, h, bias=None): h is (..., 4K) with the column blocks i, u, f, o in that order (the reference's
    LSTM_Forward layout, TF BasicLSTMCell's i, j, f, o); c is (..., K) with the same leading dims. bias is None or 4K
    entries in fp32, fp16 or bf16, read as fp32; db comes back in its dtype, the column sum of dh as stored, bitwise
    equal to bias_relu's db for that dh.

    fused_lstm_gates(c, i, u, f, o): five tensors of one shape, any rank, purely elementwise; the gates are positional
    in the op's input order (sigmoid input gate, tanh update, forget, output). The reference example's call
    fused_lstm_gates(c, i, f, o, u) (examples/lstm/layers.py:539) gets exactly these positional semantics, so there f
    is the tanh update and u the output gate. A bias in this form raises ValueError, as the reference asserts.

    c and the gates: CUDA, one dtype of fp32 / fp16 / bf16; non-contiguous inputs are made contiguous. The backward
    recomputes the gates from the inputs, as the reference's does, and saves no activations; a missing gradient of
    c_next or h_next is read as zero without being materialised. `name` is accepted and ignored."""
    if len(args) not in (1, 4):
        raise ValueError("fused_lstm_gates takes c and either h or i, u, f, o; got %d tensors after c" % len(args))
    if len(args) == 4 and bias is not None:
        raise ValueError("fused_lstm_gates: bias is not enabled in the four-tensor form (c, i, u, f, o)")
    if not isinstance(forget_bias, numbers.Real) or isinstance(forget_bias, bool):
        raise ValueError("fused_lstm_gates: forget_bias must be a Python number, got %r" % (forget_bias,))
    c = _cuda(c, "fused_lstm_gates")
    gates = [_cuda(g, "fused_lstm_gates") for g in args]
    for t in gates + ([bias] if bias is not None else []):
        if t.device != c.device:
            raise ValueError("fused_lstm_gates: operands live on different devices (%s and %s)" % (c.device, t.device))
    if any(g.dtype != c.dtype for g in gates):
        raise ValueError("fused_lstm_gates: c and the gates must share one dtype, got %s" %
                         sorted({str(t.dtype) for t in [c] + gates}))
    if c.dim() < 1:
        raise ValueError("fused_lstm_gates needs tensors of rank >= 1")
    K = c.shape[-1]
    if len(args) == 1:
        h = gates[0]
        if h.shape[:-1] != c.shape[:-1] or h.shape[-1] != 4 * K:
            raise ValueError("fused_lstm_gates: h must be c's shape with 4x its last dim, got c %s and h %s" %
                             (tuple(c.shape), tuple(h.shape)))
        if bias is not None:
            _cuda(bias, "fused_lstm_gates")
            if bias.numel() != 4 * K:
                raise ValueError("fused_lstm_gates: bias has %d entries, h's last dim %d" % (bias.numel(), 4 * K))
    elif any(g.shape != c.shape for g in gates):
        raise ValueError("fused_lstm_gates: c, i, u, f and o must share one shape, got %s" %
                         [tuple(t.shape) for t in [c] + gates])
    if (4 * K if len(args) == 1 else K) >= 2 ** 31:
        raise ValueError("fused_lstm_gates: the gates' last dim has %d entries, at most 2^31 - 1 are supported" %
                         (4 * K if len(args) == 1 else K))
    N = c.numel() // K if K else 0
    c = c.contiguous()
    gates = [g.contiguous() for g in gates]
    extra = [bias.contiguous()] if bias is not None else []
    return _LstmGatesFunction.apply(N, max(K, 1), float(forget_bias), bias is not None, c, *gates, *extra)


# ---- split4 / concat4 -------------------------------------------------------------------------------------------------
def _split4(x):
    K = x.shape[-1] // 4
    N = x.numel() // (4 * K) if K else 0
    buf = _transpose_0213(x.contiguous(), 1, N, 4, K)             # (1, 4, N, K)
    return tuple(buf[0, j].view(x.shape[:-1] + (K,)) for j in range(4))


def _concat4(zs):
    return torch.cat([z.contiguous() for z in zs], dim=-1)


class _Split4Function(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return _split4(x)

    @staticmethod
    def backward(ctx, *dz):
        return _concat4(dz)


class _Concat4Function(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *zs):
        return _concat4(zs)

    @staticmethod
    def backward(ctx, dx):
        return _split4(dx)


def split4(x):
    """The four (..., K) column blocks of x (..., 4K) as contiguous tensors (reference lstm.py:75-76), bit for bit; its
    gradient is concat4. The blocks are the slices of one (4, N, K) buffer that transpose_0213 of x viewed as
    (1, N, 4, K) writes."""
    x = _cuda(x, "split4")
    if x.dim() < 1 or x.shape[-1] % 4:
        raise ValueError("split4: the last dim must be a multiple of 4, got shape %s" % (tuple(x.shape),))
    return _Split4Function.apply(x)


def concat4(z0, z1, z2, z3):
    """x (..., 4K) from its four (..., K) column blocks, bit for bit (reference lstm.py:78-79); the inverse of split4
    and its gradient."""
    zs = [_cuda(z, "concat4") for z in (z0, z1, z2, z3)]
    if any(z.shape != zs[0].shape or z.dtype != zs[0].dtype or z.device != zs[0].device for z in zs) or zs[0].dim() < 1:
        raise ValueError("concat4 takes four tensors of one shape, dtype and device, got %s" %
                         [(tuple(z.shape), z.dtype, z.device) for z in zs])
    return _Concat4Function.apply(*zs)


# ---- sparse_relu ------------------------------------------------------------------------------------------------------
@_on_device_of
def _srelu_fwd(x, N, K, alpha):
    y = torch.empty_like(x)
    if N == 0:
        return y
    rc = _lib.load().bsmm_sparse_relu(_dt(x), x.data_ptr(), y.data_ptr(), N, K, alpha, _lib.stream_ptr())
    _lib.check(rc, "bsmm_sparse_relu")
    return y


@_on_device_of
def _relu_mask_grad(dy, y):
    dx = torch.empty_like(y)
    if y.numel() == 0:
        return dx
    rc = _lib.load().bsmm_relu_mask_grad(_dt(y), dy.data_ptr(), y.data_ptr(), dx.data_ptr(), y.numel(),
                                         _lib.stream_ptr())
    _lib.check(rc, "bsmm_relu_mask_grad")
    return dx


class _SparseReluFunction(torch.autograd.Function):
    """Saves y; the gradient is relu's on it (reference lstm.py:106-109)."""

    @staticmethod
    def forward(ctx, x, N, K, alpha):
        y = _srelu_fwd(x, N, K, alpha)
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        y, = ctx.saved_tensors
        return _relu_mask_grad(dy.to(y.dtype).contiguous(), y), None, None, None


def sparse_relu(x, alpha=1.0):
    """y = max(x - (mean + alpha * std), 0) along the last axis (reference lstm.py:97-98), std the population standard
    deviation; differentiable in x.

    x: CUDA, fp32 / fp16 / bf16, any rank >= 1, rows of any length K >= 1. alpha: a Python number (ValueError
    otherwise). mean and std are formed in fp32 in two passes in a fixed order, never as E[x^2] - E[x]^2 (which the
    reference uses, lstm_op_gpu.cu:620, and which cancels when the mean is large against the spread); y is rounded
    once and bitwise reproducible. A row of one entry, or of equal entries, gives zeros. The gradient is relu's on the
    output, dx = dy where y > 0 and 0 elsewhere, as in the reference: it deliberately ignores how mean and std depend
    on x."""
    if not isinstance(alpha, numbers.Real) or isinstance(alpha, bool):
        raise ValueError("sparse_relu: alpha must be a Python number, got %r" % (alpha,))
    x = _cuda(x, "sparse_relu")
    if x.dim() < 1:
        raise ValueError("sparse_relu needs a tensor of rank >= 1")
    K = x.shape[-1]
    if K >= 2 ** 31:
        raise ValueError("sparse_relu: the last dim has %d entries, at most 2^31 - 1 are supported" % K)
    N = x.numel() // K if K else 0
    return _SparseReluFunction.apply(x.contiguous(), N, max(K, 1), float(alpha))


# the reference's lstm module also holds these; they live in lstm_layer.py and are reachable here too
from .lstm_layer import FusedBasicLSTMCell, grouped_lstm  # noqa: E402,F401
