"""CPU restatement of the reference's dense softmax and top-k ops in float64 -- TEST INFRASTRUCTURE ONLY (see
oracle/__init__.py: only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this package).

Each function follows the reference (file:line relative to the openai/blocksparse source tree):
  masked_softmax       blocksparse/transformer.py:609-625 (masked_softmax_test)
  masked_top_k_softmax blocksparse/transformer.py:627-649 (masked_top_k_softmax_test)
  masked_softmax_grad  blocksparse/transformer.py:651-656 (masked_softmax_grad_test)
  rectified_top_k      blocksparse/transformer.py:536-549 (rectified_top_k_test)
  top_k                src/transformer_op.cc:58-92 (values and indices of the k largest entries; no NumPy checker)
Parity status: pinned to the reference's own NumPy checkers on seeded inputs (tests/golden/dense_*.npz), for the mask
shapes those checkers get right. Recorded differences, where this restatement follows the documented behaviour of the
ops rather than the reference:
  * the mask broadcasts by NumPy rules, so a (D1, 1, D3) mask is applied to the rows it names; the reference's checker
    flattens the mask (transformer.py:613) and its kernel derives the dim-1 stride from x (transformer_op.cc:184-185);
  * ties rank by index ascending (a stable sort on the value descending); the reference uses NumPy's unstable argsort.
The masked values v are formed as the ops form them, x * m * scale; pass `values` = float32 to rank on the fp32 values
the kernels compare.
"""
import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)


def masked_values(x, mask=None, scale=1.0, dtype=np.float64):
    """v = x * m * scale where m != 0, -FLT_MAX where m == 0 (transformer.py:612-619), broadcast to x's shape."""
    x = np.asarray(x, dtype=dtype)
    if mask is None:
        return x * dtype(scale)
    m = np.broadcast_to(np.asarray(mask, dtype=dtype), x.shape)
    return np.where(m != 0, x * m * dtype(scale), dtype(-FLT_MAX))


def rank(v):
    """Column order of each row of v (..., D3): value descending, then index ascending."""
    return np.argsort(-np.asarray(v), axis=-1, kind="stable")


def masked_softmax(x, mask=None, scale=1.0):
    y = masked_values(x, mask, scale)
    e = np.exp(y - y.max(axis=-1, keepdims=True))                       # transformer.py:622-623
    return e / e.sum(axis=-1, keepdims=True)


def masked_top_k_softmax(x, k, mask=None, scale=1.0, order_values=None):
    """order_values: the values whose rank picks the support (default: v in float64)."""
    y = masked_values(x, mask, scale)
    top = rank(y if order_values is None else order_values)[..., :k]    # transformer.py:641
    v = np.take_along_axis(y, top, axis=-1)
    e = np.exp(v - v.max(axis=-1, keepdims=True))                       # transformer.py:645-647
    z = np.zeros(y.shape)
    np.put_along_axis(z, top, e / e.sum(axis=-1, keepdims=True), axis=-1)
    return z


def masked_softmax_grad(dy, y, mask=None, scale=1.0):
    dy, y = np.asarray(dy, dtype=np.float64), np.asarray(y, dtype=np.float64)
    m = 1.0 if mask is None else np.asarray(mask, dtype=np.float64)
    return (dy - np.sum(dy * y, axis=-1, keepdims=True)) * y * m * scale    # transformer.py:656


def top_k(x, k):
    x = np.asarray(x)
    idx = rank(x.astype(np.float64))[..., :k]
    return np.take_along_axis(x, idx, axis=-1), idx.astype(np.int32)


def rectified_top_k(x, k, rebase=True):
    x = np.asarray(x, dtype=np.float64)
    top = rank(x)[..., :k]                                              # transformer.py:538
    v = np.take_along_axis(x, top, axis=-1)
    base = np.maximum(v[..., k - 1:k], 0.0) if rebase else np.zeros_like(v[..., :1])   # transformer.py:543
    y = np.zeros(x.shape)
    np.put_along_axis(y, top, np.maximum(v, base) - base, axis=-1)      # transformer.py:547
    return y
