"""ctypes binding of oracle/_ref/libbsref.so: the reference's own CUDA kernels (openai/blocksparse src/*_op_gpu.cu) built
for sm_90a by oracle/ref/Makefile, so that tests can run them next to ours on the same inputs.

Each function takes CUDA torch tensors, applies the argument checks of the reference op (its *_op.cc) and the limits of
its launcher (32-bit sizes, grid.y / grid.z below 65536, aligned vector widths), raising ValueError before anything is
launched, and returns new tensors. 16-bit data goes in and comes out as the raw bits of torch.float16 (the reference's
ehalf) or torch.bfloat16 (bhalf). Every output is allocated with a poisoned guard region after its end, checked after
the launch, so a write past the end raises instead of passing unseen.

Only the test suite imports this module; the package, bench.py and smoke() do not.
"""
import ctypes
import math
import os

import torch

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libbsref.so")
DT = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
IT = {torch.int32: 0, torch.uint8: 2}
if hasattr(torch, "uint16"):
    IT[torch.uint16] = 1
GUARD = 256                                    # bytes of poison after every output
POISON = 0x5A

_u, _i, _f, _p = ctypes.c_uint, ctypes.c_int, ctypes.c_float, ctypes.c_void_p
_ll = ctypes.POINTER(ctypes.c_longlong)
SIGNATURES = {
    "bsref_bias_relu": [_i, _p, _p, _p, _u, _u, _u, _u, _p],
    "bsref_bias_relu_grad_partials": [_u, _u, _u, _i],
    "bsref_bias_relu_grad": [_i, _p, _p, _p, _p, _p, _p, _u, _u, _u, _u, _i, _p],
    "bsref_dropout_apply": [_i, _p, _p, _p, _f, _i, _ll, _i, _ll, _p],
    "bsref_filter_tensor": [_i, _p, _p, _u, _f, _f, _i, _i, _p],
    "bsref_embedding_lookup": [_i, _i, _p, _p, _p, _i, _i, _i, _p],
    "bsref_embedding_grad": [_i, _i, _p, _p, _p, _i, _i, _i, _i, _p],
    "bsref_transpose_2d": [_i, _p, _p, _u, _u, _p],
    "bsref_transpose_0213": [_i, _p, _p, _u, _u, _u, _u, _p],
    "bsref_apply_adam": [_i, _p, _p, _p, _p, _p, _f, _f, _f, _f, _f, _f, _u, _f, _i, _i, _p],
}
RESTYPES = {"bsref_bias_relu_grad_partials": _u}

_LIB = None


def available():
    return os.path.exists(LIB_PATH)


def load():
    global _LIB
    if _LIB is None:
        lib = ctypes.CDLL(LIB_PATH)
        for name, args in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.argtypes = args
            fn.restype = RESTYPES.get(name, _i)
        _LIB = lib
    return _LIB


# ---- plumbing ---------------------------------------------------------------------------------------------------------
def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dt(t):
    if t.dtype not in DT:
        raise ValueError("the reference kernels take fp32, fp16 or bf16, got %s" % t.dtype)
    return DT[t.dtype]


def _dev(*ts):
    for t in ts:
        if not torch.is_tensor(t) or not t.is_cuda:
            raise ValueError("the reference kernels take CUDA tensors")
    return [t.contiguous() for t in ts]


def _u32(what, v):
    if not 0 <= v < 2 ** 32:
        raise ValueError("%s = %d does not fit the launcher's 32-bit uint" % (what, v))
    return v


def _i32(what, v):
    if not 0 <= v < 2 ** 31:
        raise ValueError("%s = %d does not fit the launcher's 32-bit int" % (what, v))
    return v


class _Out:
    """An output tensor followed by GUARD bytes of POISON; check() raises if the kernel wrote into them."""

    def __init__(self, shape, dtype, device):
        n = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
        self.raw = torch.full((n + GUARD,), POISON, dtype=torch.uint8, device=device)
        self.t = self.raw[:n].view(dtype).view(shape)

    def check(self, what):
        if not bool((self.raw[-GUARD:] == POISON).all()):
            raise AssertionError("%s wrote past the end of its output" % what)
        return self.t


def _call(name, outs, *args):
    rc = getattr(load(), name)(*args, _stream())
    if rc != 0:
        raise RuntimeError("%s: CUDA error %d" % (name, rc))
    torch.cuda.current_stream().synchronize()
    return [o.check(name) for o in outs]


# ---- bias + activation (ew_op.cc BiasReluOp / BiasReluGradOp) ---------------------------------------------------------
def _bias_layout(x, b, axis):
    if b.dtype != torch.float32:
        raise ValueError("BiasRelu takes b in fp32 only")
    nd = x.dim()
    axis = axis + nd if axis < 0 else axis
    if not (axis < nd and (axis == 0 or axis == nd - 1)):
        raise ValueError("BiasRelu bad axis")
    K = x.shape[axis]
    N = x.numel() // K if K else 0
    if K != b.numel():
        raise ValueError("BiasRelu missmatched channels")
    _u32("N * K", N * K)
    return (0 if axis == 0 else 1), N, K


def bias_relu(x, b, axis=-1, relu=0):
    """y = act(x + b); relu 0 none, 1 relu, 2 fast_gelu."""
    x, b = _dev(x, b)
    ax, N, K = _bias_layout(x, b, axis)
    y = _Out(x.shape, x.dtype, x.device)
    return _call("bsref_bias_relu", [y], _dt(x), y.t.data_ptr(), x.data_ptr(), b.data_ptr(), ax, N, K, relu)[0]


def bias_relu_grad(dy, src, b, axis=-1, relu=0, atomics=True):
    """(dx, db): src is y for relu and x for fast_gelu. Without an activation the kernel leaves dx unwritten and the
    reference's Python returns dy, so dx is dy here."""
    dy, src, b = _dev(dy, src, b)
    ax, N, K = _bias_layout(dy, b, axis)
    words = load().bsref_bias_relu_grad_partials(ax, N, K, int(bool(atomics)))
    part = torch.empty(max(words, 1), dtype=torch.float32, device=dy.device)
    dx = _Out(dy.shape, dy.dtype, dy.device)
    db = _Out((K,), torch.float32, dy.device)
    dxp, dbp = _call("bsref_bias_relu_grad", [dx, db], _dt(dy), db.t.data_ptr(), part.data_ptr() if words else None,
                     dx.t.data_ptr(), dy.data_ptr(), src.data_ptr(), b.data_ptr(), ax, N, K, relu, int(bool(atomics)))
    return (dy if relu == 0 else dxp), dbp


# ---- dropout (ew_op.cc ApplyDropoutMaskOp) ----------------------------------------------------------------------------
def apply_dropout_mask(x, mask, keep_prob, mask_shape=None):
    """x * (1 / keep_prob) where the mask bit is set, 0 elsewhere; mask: int32 words, mask_shape None for a flat mask
    over x, else x's rank with dims equal to x's or 1."""
    x, mask = _dev(x, mask)
    if mask.dtype != torch.int32:
        raise ValueError("ApplyDropoutMask takes an int32 mask")
    size = _u32("size", x.numel())
    if mask_shape is None or len(mask_shape) == 0:
        ms = ()
        msize = size
    else:
        ms = tuple(int(d) for d in mask_shape)
        if len(ms) > 5 or x.dim() != len(ms) or not 1 <= x.dim() <= 5:
            raise ValueError("ApplyDropoutMaskOp: bad mask shape (rank)")
        if any(m != s and m != 1 for m, s in zip(ms, x.shape)):
            raise ValueError("ApplyDropoutMaskOp: bad mask shape (dims)")
        if len(ms) == 1 and ms[0] == 1 and x.shape[0] != 1:
            # at rank 1 the launcher takes 4- or 8-wide vector loads, which test bits shift + i of one word: with a
            # broadcast stride of 0 they read bits 0..7 instead of bit 0
            raise ValueError("ApplyDropoutMask: a rank-1 mask of one element broadcast over x is read wrongly")
        msize = math.prod(ms)
    if mask.numel() != (msize + 31) // 32:
        raise ValueError("ApplyDropoutMaskOp: bad mask shape (size)")
    y = _Out(x.shape, x.dtype, x.device)
    if size == 0:
        return y.t
    arr = ctypes.c_longlong * 5
    return _call("bsref_dropout_apply", [y], _dt(x), y.t.data_ptr(), x.data_ptr(), mask.data_ptr(), float(keep_prob),
                 x.dim(), arr(*x.shape), len(ms), arr(*ms))[0]


# ---- grad filter (ew_op.cc FilterTensorOp) ----------------------------------------------------------------------------
def filter_tensor(x, scale=1.0, saturate=0.0, zero_infs=False, zero_nans=False):
    x, = _dev(x)
    y = _Out(x.shape, x.dtype, x.device)
    size = _u32("size", x.numel())
    if size == 0:
        return y.t
    return _call("bsref_filter_tensor", [y], _dt(x), y.t.data_ptr(), x.data_ptr(), size, float(scale), float(saturate),
                 int(bool(zero_infs)), int(bool(zero_nans)))[0]


# ---- embedding (embedding_op.cc EmbeddingLookupOp / EmbeddingLookupGradOp) --------------------------------------------
def _emb_args(idx, C, K):
    if idx.dtype not in IT:
        raise ValueError("EmbeddingLookup takes int32, uint16 or uint8 indices, got %s" % idx.dtype)
    # the launchers form nIdx * K, C * K and row * K + k from int operands
    nIdx = _i32("nIdx", idx.numel())
    _i32("C", C)
    _i32("nIdx * K", nIdx * K)
    _i32("C * K", C * K)
    return IT[idx.dtype], nIdx


def embedding_lookup(emb, idx):
    emb, idx = _dev(emb, idx)
    if emb.dim() != 2:
        raise ValueError("EmbeddingLookup takes a 2-D emb")
    C, K = emb.shape
    it, nIdx = _emb_args(idx, C, K)
    y = _Out(tuple(idx.shape) + (K,), emb.dtype, emb.device)
    if nIdx * K == 0:
        return y.t
    return _call("bsref_embedding_lookup", [y], it, _dt(emb), y.t.data_ptr(), idx.data_ptr(), emb.data_ptr(), nIdx, C,
                 K)[0]


def embedding_grad(dy, idx, C, sorted=True):
    """dw (C, K) in fp32, as the op returns it."""
    dy, idx = _dev(dy, idx)
    K = dy.shape[-1]
    it, nIdx = _emb_args(idx, C, K)
    if dy.numel() != nIdx * K:
        raise ValueError("EmbeddingLookupGrad: dy does not match idx")
    if sorted and -(-K // 256) >= 65536:
        raise ValueError("EmbeddingLookupGrad: K = %d overflows grid.y of the sorted kernel" % K)
    dw = _Out((C, K), torch.float32, dy.device)
    if C * K == 0:
        return dw.t
    return _call("bsref_embedding_grad", [dw], it, _dt(dy), dw.t.data_ptr(), idx.data_ptr(), dy.data_ptr(), nIdx, C, K,
                 int(bool(sorted)))[0]


# ---- transposes (transformer_op.cc Transpose2DOp / Transpose0213Op) ---------------------------------------------------
def transpose_2d(x):
    x, = _dev(x)
    if x.dim() != 2:
        raise ValueError("Transpose2D: x.dims() == 2")
    D0, D1 = (_u32("D", d) for d in x.shape)
    if D0 % 4 or D1 % 4:
        # each thread moves a 4 x 4 tile with 4-wide vector accesses and checks only the tile's first row and column,
        # so other sizes read and write past the rows (the op does not check; its kernel's comment asks for it)
        raise ValueError("Transpose_2D: both dims must be multiples of 4, got %s" % (tuple(x.shape),))
    if -(-D0 // 64) >= 65536:
        raise ValueError("Transpose_2D: D0 = %d overflows grid.y" % D0)
    y = _Out((D1, D0), x.dtype, x.device)
    if x.numel() == 0:
        return y.t
    return _call("bsref_transpose_2d", [y], _dt(x), y.t.data_ptr(), x.data_ptr(), D0, D1)[0]


def transpose_0213(x):
    x, = _dev(x)
    if x.dim() != 4:
        raise ValueError("Transpose0213: x.dims() == 4")
    D0, D1, D2, D3 = x.shape
    if D0 >= 65536 or D1 >= 65536:
        raise ValueError("Transpose0213: D0 and D1 must be < 65536, got %s" % (tuple(x.shape),))
    _u32("size", x.numel())
    y = _Out((D0, D2, D1, D3), x.dtype, x.device)
    if x.numel() == 0:
        return y.t
    return _call("bsref_transpose_0213", [y], _dt(x), y.t.data_ptr(), x.data_ptr(), D0, D1, D2, D3)[0]


# ---- Adam (optimize_op.cc ApplyAdamOp, dense, no lazy_emb, no gate) ---------------------------------------------------
def apply_adam(grad, param, mean, var, lr, beta1, beta2, epsilon, grad_scale=1.0, clip_sigma=0.0, norm_scale=None,
               saturate=0.0, zero_infs=False, zero_nans=False):
    """One step in place on clones: returns (param, mean, var). grad and param fp32; mean and var both fp32, or both
    int16 holding the 16-bit mean / variance codes. norm_scale: None or a 1-element fp32 CUDA tensor."""
    grad, param, mean, var = _dev(grad, param, mean, var)
    if grad.dtype != torch.float32 or param.dtype != torch.float32:
        raise ValueError("ApplyAdam is bound for fp32 grad and param")
    if not grad.shape == param.shape == mean.shape == var.shape:
        raise ValueError("ApplyAdam: grad, param, mean and var must have one shape")
    if mean.dtype != var.dtype or mean.dtype not in (torch.float32, torch.int16):
        raise ValueError("ApplyAdam: mean and var are both fp32 or both 16-bit codes")
    size = _u32("size", param.numel())
    outs = [_Out(t.shape, t.dtype, t.device) for t in (param, mean, var)]
    for o, t in zip(outs, (param, mean, var)):
        o.t.copy_(t)
    if size == 0:
        return [o.t for o in outs]
    ns = None if norm_scale is None else _dev(norm_scale)[0].data_ptr()
    return _call("bsref_apply_adam", outs, int(mean.dtype == torch.int16), grad.data_ptr(), ns, outs[0].t.data_ptr(),
                 outs[1].t.data_ptr(), outs[2].t.data_ptr(), float(lr), float(beta1), float(beta2), float(epsilon),
                 float(grad_scale), float(clip_sigma), size, float(saturate), int(bool(zero_infs)),
                 int(bool(zero_nans)))
