"""Float64 NumPy oracle of the lstm module: the LSTM gate nonlinearity in both gate layouts with its gradient, and
sparse_relu with its gradient. Arrays of any float dtype go in; everything is computed in float64."""
import numpy as np


def _sig(z):
    """1 / (1 + e^-z) without overflow, and without the cancellation of 0.5 (1 + tanh(z / 2)) for z << 0."""
    e = np.exp(-np.abs(z))
    return np.where(np.asarray(z) >= 0, 1.0 / (1.0 + e), e / (1.0 + e))


def _split(h):
    K = h.shape[-1] // 4
    return [h[..., j * K:(j + 1) * K] for j in range(4)]


def _bias(bias, K):
    if bias is None:
        return [0.0] * 4
    b = np.asarray(bias, np.float64).reshape(-1)
    return [b[j * K:(j + 1) * K] for j in range(4)]


def _gates(c, i, u, f, o, bias, forget_bias):
    c, i, u, f, o = (np.asarray(t, np.float64) for t in (c, i, u, f, o))
    bi, bu, bf, bo = _bias(bias, c.shape[-1])
    si, tu, sf, so = _sig(i + bi), np.tanh(u + bu), _sig(f + bf + forget_bias), _sig(o + bo)
    cn = sf * c + si * tu
    return c, si, tu, sf, so, cn, np.tanh(cn)


def lstm_gates(c, i, u, f, o, bias=None, forget_bias=1.0):
    """(c_next, h_next) of the four-tensor form; bias None or 4K entries in the i, u, f, o blocks."""
    _, _, _, _, so, cn, tc = _gates(c, i, u, f, o, bias, forget_bias)
    return cn, so * tc


def lstm_gates_grad(c, i, u, f, o, ec=None, eh=None, bias=None, forget_bias=1.0):
    """(dc, di, du, df, do) of lstm_gates given the gradients ec of c_next and eh of h_next (None = 0)."""
    c, si, tu, sf, so, cn, tc = _gates(c, i, u, f, o, bias, forget_bias)
    ec = 0.0 if ec is None else np.asarray(ec, np.float64)
    eh = 0.0 if eh is None else np.asarray(eh, np.float64)
    dcn = ec + eh * so * (1.0 - tc * tc)
    di = dcn * tu * si * (1.0 - si)
    du = dcn * si * (1.0 - tu * tu)
    df = dcn * c * sf * (1.0 - sf)
    do = eh * tc * so * (1.0 - so)
    zero = np.zeros_like(cn)
    return tuple(zero + d for d in (dcn * sf, di, du, df, do))


def lstm_gates_fused(c, h, bias=None, forget_bias=1.0):
    """(c_next, h_next) of the fused form: h (..., 4K) with the column blocks i, u, f, o."""
    return lstm_gates(c, *_split(np.asarray(h)), bias=bias, forget_bias=forget_bias)


def lstm_gates_fused_grad(c, h, ec=None, eh=None, bias=None, forget_bias=1.0):
    """(dc, dh, db): dh (..., 4K) in the i, u, f, o blocks, db its column sums (None without a bias)."""
    dc, *dg = lstm_gates_grad(c, *_split(np.asarray(h)), ec=ec, eh=eh, bias=bias, forget_bias=forget_bias)
    dh = np.concatenate(dg, axis=-1)
    return dc, dh, (None if bias is None else dh.reshape(-1, dh.shape[-1]).sum(axis=0))


def sparse_relu(x, alpha=1.0):
    """max(x - (mean + alpha std), 0) along the last axis, std the population standard deviation."""
    x = np.asarray(x, np.float64)
    cutoff = x.mean(axis=-1, keepdims=True) + alpha * x.std(axis=-1, keepdims=True)
    return np.maximum(x - cutoff, 0.0)


def sparse_relu_grad(dy, y):
    """relu's gradient on the output: dy where y > 0, else 0."""
    return np.where(np.asarray(y) > 0, np.asarray(dy, np.float64), 0.0)
