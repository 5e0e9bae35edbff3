"""Float64 oracle of layer norm and its gradient (reference blocksparse/norms.py: layer_norm :23-53, the gradient its
LayerNormGrad op computes, checked by layer_norm_grad_test :129-170).

Every function works on float64 copies of its inputs. x has the feature axis last or first (axis 0: x is viewed as
(K, N)); each row of K features is split into `segments` segments of L = K / segments that are normalised apart, with
gain and bias g[s*L:(s+1)*L], b[...]. The variance is the biased one, formed from centred values.
"""
import numpy as np


def _rows(a, axis, segments):
    """(rows, segments, L) float64 view of a with the feature axis `axis` (0 or last)."""
    a = np.asarray(a, dtype=np.float64)
    K = a.shape[axis]
    a2 = np.ascontiguousarray(a.reshape(K, -1).T) if axis == 0 else a.reshape(-1, K)
    return a2.reshape(a2.shape[0], segments, K // segments)


def _unrows(v, shape, axis):
    v = v.reshape(v.shape[0], -1)
    return (v.T if axis == 0 else v).reshape(shape)


def _axis(x, axis):
    axis = axis % np.ndim(x)
    if axis not in (0, np.ndim(x) - 1):
        raise ValueError("feature axis must be 0 or last")
    return 0 if axis == 0 and np.ndim(x) > 1 else -1


def statistics(x, axis=-1, segments=1, epsilon=1e-6):
    """(mean, rstd), float64 of shape (rows, segments)."""
    xs = _rows(x, _axis(x, axis), segments)
    mean = xs.mean(axis=2)
    var = np.square(xs - mean[..., None]).mean(axis=2)
    return mean, 1.0 / np.sqrt(var + epsilon)


def layer_norm(x, g, b, axis=-1, segments=1, epsilon=1e-6, relu=False):
    ax = _axis(x, axis)
    xs = _rows(x, ax, segments)
    mean, rstd = statistics(x, axis, segments, epsilon)
    gs = np.asarray(g, dtype=np.float64).reshape(1, segments, -1)
    bs = np.asarray(b, dtype=np.float64).reshape(1, segments, -1)
    y = (xs - mean[..., None]) * rstd[..., None] * gs + bs
    if relu:
        y = np.maximum(y, 0.0)
    return _unrows(y, np.shape(x), ax)


def layer_norm_grad(dy, x, g, b, axis=-1, segments=1, epsilon=1e-6, relu=False):
    """(dx of x's shape, dg, db of K entries)."""
    ax = _axis(x, axis)
    xs, dys = _rows(x, ax, segments), _rows(dy, ax, segments)
    mean, rstd = statistics(x, axis, segments, epsilon)
    gs = np.asarray(g, dtype=np.float64).reshape(1, segments, -1)
    bs = np.asarray(b, dtype=np.float64).reshape(1, segments, -1)
    xhat = (xs - mean[..., None]) * rstd[..., None]
    if relu:
        dys = np.where(xhat * gs + bs > 0, dys, 0.0)
    dg = np.einsum("rsl,rsl->sl", dys, xhat).reshape(-1)
    db = dys.sum(axis=0).reshape(-1)
    dyg = dys * gs
    L = xs.shape[2]
    s1 = np.einsum("rsl,rsl->rs", dyg, xhat)[..., None]
    s2 = dyg.sum(axis=2, keepdims=True)
    dx = rstd[..., None] * (dyg - (xhat * s1 + s2) / L)
    return _unrows(dx, np.shape(x), ax), dg, db
