"""Float64 NumPy oracle of softmax_cross_entropy, its gradient and the two transposes (reference
blocksparse/transformer.py:664-700). The reference checks these ops against TensorFlow only, so there is no reference
NumPy checker to pin them to; tests/test_xent_oracle.py checks this module against scipy and torch instead.

Semantics beyond the reference, shared with the kernels:
  * a label outside [0, K) gives NaN for its row's loss, lse and gradient;
  * -inf logits get probability 0; a label at a -inf entry gives +inf; a row of -inf only gives lse -inf, loss NaN.
"""
import numpy as np


def _rows(x, labels):
    x = np.asarray(x, dtype=np.float64)
    K = x.shape[-1]
    xr = x.reshape(-1, K)
    lab = np.asarray(labels).reshape(-1).astype(np.int64)
    if lab.size != xr.shape[0]:
        raise ValueError("%d labels for %d rows" % (lab.size, xr.shape[0]))
    return x, xr, lab, (lab >= 0) & (lab < K)


def _lse(xr):
    m = xr.max(axis=-1, keepdims=True)
    with np.errstate(invalid="ignore", divide="ignore"):
        ms = np.where(np.isneginf(m), 0.0, m)             # an all -inf row: sum 0, lse -inf
        return (ms + np.log(np.exp(xr - ms).sum(axis=-1, keepdims=True)))[:, 0]


def softmax_cross_entropy(x, labels):
    """(loss, lse), float64 of x.shape[:-1]: lse = logsumexp(x[n]), loss = lse - x[n, labels[n]]."""
    x, xr, lab, ok = _rows(x, labels)
    lse = _lse(xr)
    picked = xr[np.arange(xr.shape[0]), np.where(ok, lab, 0)]
    with np.errstate(invalid="ignore"):
        loss = np.where(ok, lse - picked, np.nan)
    lse = np.where(ok, lse, np.nan)
    return loss.reshape(x.shape[:-1]), lse.reshape(x.shape[:-1])


def softmax_cross_entropy_grad(x, labels, dy):
    """dx = dy[n] * (softmax(x[n]) - onehot(labels[n])), float64 of x's shape."""
    x, xr, lab, ok = _rows(x, labels)
    _, lse = softmax_cross_entropy(xr, lab)
    dyr = np.asarray(dy, dtype=np.float64).reshape(-1)
    with np.errstate(invalid="ignore", over="ignore"):
        p = np.exp(xr - lse.reshape(-1, 1))
        onehot = np.zeros_like(xr)
        onehot[np.nonzero(ok)[0], lab[ok]] = 1.0
        dx = dyr[:, None] * (p - onehot)
    return dx.reshape(x.shape)


def transpose_0213(x):
    x = np.asarray(x)
    if x.ndim != 4:
        raise ValueError("transpose_0213 needs rank 4")
    return np.ascontiguousarray(x.transpose(0, 2, 1, 3))


def transpose_2d(x):
    x = np.asarray(x)
    if x.ndim != 2:
        raise ValueError("transpose_2d needs rank 2")
    return np.ascontiguousarray(x.T)
