"""Embedding lookup -- host side of the reference's blocksparse/embed.py, on torch tensors, calling the sm_90a kernels
of csrc/embed.cuh through bsmm_embedding_lookup / bsmm_embedding_grad.
"""
import torch

from . import _lib
from .transformer import _dense_bench, _on_device_of

__all__ = ["embedding_lookup"]


@_on_device_of
def _emb_fwd(emb, idx):
    C, K = emb.shape
    y = torch.empty(tuple(idx.shape) + (K,), dtype=emb.dtype, device=emb.device)
    if y.numel() == 0:
        return y
    rc = _lib.load().bsmm_embedding_lookup(_lib.dtype_code(emb.dtype), _lib.label_code(idx.dtype), emb.data_ptr(),
                                           idx.data_ptr(), y.data_ptr(), idx.numel(), C, K, _lib.stream_ptr())
    _lib.check(rc, "bsmm_embedding_lookup")
    return y


@_on_device_of
def _emb_bwd(dy, idx, C, K):
    n = idx.numel()
    if n == 0 or C == 0 or K == 0:
        return torch.zeros((C, K), dtype=dy.dtype, device=dy.device)
    dw = torch.empty((C, K), dtype=dy.dtype, device=dy.device)
    ws = torch.empty(_lib.load().bsmm_embedding_grad_workspace_bytes(n, C, K), dtype=torch.uint8, device=dy.device)
    rc = _lib.load().bsmm_embedding_grad(_lib.dtype_code(dy.dtype), _lib.label_code(idx.dtype), dy.data_ptr(),
                                         idx.data_ptr(), dw.data_ptr(), ws.data_ptr(), n, C, K, _lib.stream_ptr())
    _lib.check(rc, "bsmm_embedding_grad")
    return dw


def _tag(emb, idx):
    return "embedding_lookup nIdx %d C %d K %d %s" % (idx.numel(), emb.shape[0], emb.shape[1],
                                                        str(emb.dtype).replace("torch.", ""))


class _EmbeddingFunction(torch.autograd.Function):
    """Saves idx; dw is summed per row in fp32 in index order and rounded once to emb's dtype (reference
    embed.py:26-35)."""

    @staticmethod
    def forward(ctx, emb, idx, bench):
        ctx.C, ctx.K = emb.shape
        ctx.bench = bench
        ctx.save_for_backward(idx)
        return _emb_fwd(emb, idx)

    @staticmethod
    def backward(ctx, dy):
        idx, = ctx.saved_tensors
        dy = dy.contiguous()
        if ctx.bench:
            _dense_bench("embedding_lookup_grad nIdx %d C %d K %d" % (idx.numel(), ctx.C, ctx.K),
                         lambda: _emb_bwd(dy, idx, ctx.C, ctx.K), 2 * dy.numel() * dy.element_size(), ctx.bench)
        return _emb_bwd(dy, idx, ctx.C, ctx.K), None, None


def embedding_lookup(emb, idx, sort_grad=True, bench=0, use_tf=False):
    """y = emb[idx]: y has shape idx.shape + (K,) and holds bit copies of the rows of emb (C, K); an index < 0 or >= C
    gives a zero row and adds nothing to the gradient (reference embed.py:15-24). Differentiable in emb.

    emb: CUDA, fp32 / fp16 / bf16, 2-D. idx: any shape, uint8 / uint16 / int32 / int64, on emb's device. The gradient
    dw (C, K) in emb's dtype is summed per row in fp32 in index order and rounded once, without atomics, so it is
    bitwise reproducible; rows no index hits are 0. `sort_grad` is accepted for compatibility and has no effect (the
    gradient always sorts). bench > 0 times that many launches of the lookup (and of the gradient) and prints one line
    each. use_tf=True raises ValueError."""
    if use_tf:
        raise ValueError("embedding_lookup: use_tf is a TensorFlow composition; there is none here")
    if not torch.is_tensor(emb) or not emb.is_cuda or emb.dim() != 2:
        raise ValueError("embedding_lookup needs a 2-D CUDA tensor emb (there is no CPU path)")
    _lib.dtype_code(emb.dtype)
    if not torch.is_tensor(idx) or idx.device != emb.device:
        raise ValueError("embedding_lookup: idx must be a tensor on emb's device %s" % emb.device)
    _lib.label_code(idx.dtype)
    if emb.shape[0] >= 2 ** 31 - 1 or emb.shape[1] >= 2 ** 31:
        raise ValueError("embedding_lookup: emb of shape %s is too large" % (tuple(emb.shape),))
    emb, idx = emb.contiguous(), idx.contiguous()
    if bench:
        _dense_bench(_tag(emb, idx), lambda: _emb_fwd(emb, idx), 2 * idx.numel() * emb.shape[1] * emb.element_size(),
                     bench)
    return _EmbeddingFunction.apply(emb, idx, int(bench))
