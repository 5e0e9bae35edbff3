"""Float64 NumPy oracle of the LSTM layers: grouped_lstm (forward and BPTT, with and without the 4-segment layer norm)
and one FusedBasicLSTMCell step. Arrays of any float dtype go in; everything is computed in float64."""
import numpy as np

from .lstm_oracle import lstm_gates_fused, lstm_gates_fused_grad

LN_EPS = 1e-6


def _f64(a):
    return None if a is None else np.asarray(a, np.float64)


def _ln4(z, g, b, eps):
    """(v, xhat, rstd) of layer_norm(z, g, b, axis=1, segments=4): per row and segment of z (N, 4K)."""
    N, K4 = z.shape
    zs = z.reshape(N, 4, K4 // 4)
    mean = zs.mean(axis=2, keepdims=True)
    rstd = 1.0 / np.sqrt(((zs - mean) ** 2).mean(axis=2, keepdims=True) + eps)
    xh = ((zs - mean) * rstd).reshape(N, K4)
    return xh * g + b, xh, rstd


def _ln4_grad(dv, xh, rstd, g):
    """(dz, dg, db) of _ln4 given the gradient dv of its output."""
    N, K4 = dv.shape
    dxh = (dv * g).reshape(N, 4, K4 // 4)
    x3 = xh.reshape(N, 4, K4 // 4)
    dz = rstd * (dxh - dxh.mean(axis=2, keepdims=True) - x3 * (dxh * x3).mean(axis=2, keepdims=True))
    return dz.reshape(N, K4), (dv * xh).sum(axis=0), dv.sum(axis=0)


def _steps(x, c0, h0, kernel, bias, gain, layernorm, eps):
    x, c, h, kernel, bias, gain = (_f64(a) for a in (x, c0, h0, kernel, bias, gain))
    if x.ndim == 2:
        x = x[:, None, :]
    saved = []
    outs = []
    for t in range(x.shape[1]):
        xh = np.concatenate([x[:, t], h], axis=1)
        z = xh @ kernel
        if layernorm:
            v, xhat, rstd = _ln4(z, gain, bias, eps)
            c_new, h = lstm_gates_fused(c, v, forget_bias=1.0)
        else:
            v, xhat, rstd = z, None, None
            c_new, h = lstm_gates_fused(c, z, bias=bias, forget_bias=1.0)
        saved.append((xh, c, v, xhat, rstd))
        c = c_new
        outs.append(h)
    return np.stack(outs, axis=1), c, h, saved


def grouped_lstm(x, c0, h0, kernel, bias, gain=None, layernorm=True, eps=LN_EPS):
    """(output (N, T, W), c_T, h_T); x is (N, T, in) or (N, in)."""
    out, c, h, _ = _steps(x, c0, h0, kernel, bias, gain, layernorm, eps)
    return out, c, h


def grouped_lstm_grad(x, c0, h0, kernel, bias, gain, layernorm, d_out=None, d_c=None, d_h=None, eps=LN_EPS):
    """(dx (x's shape), dc0, dh0, dkernel, dbias, dgain or None) given the gradients of output, c_T and h_T (None = 0)."""
    x64 = _f64(x)
    _, _, _, saved = _steps(x, c0, h0, kernel, bias, gain, layernorm, eps)
    kernel, bias, gain = _f64(kernel), _f64(bias), _f64(gain)
    T = len(saved)
    N, W = saved[0][1].shape
    In = kernel.shape[0] - W
    d_out = np.zeros((N, T, W)) if d_out is None else _f64(d_out).reshape(N, T, W)
    dc = np.zeros((N, W)) if d_c is None else _f64(d_c)
    dh = np.zeros((N, W)) if d_h is None else _f64(d_h)
    dx = np.zeros((N, T, In))
    dk = np.zeros_like(kernel)
    db = np.zeros(4 * W)
    dg = np.zeros(4 * W) if layernorm else None
    for t in range(T - 1, -1, -1):
        xh, c, v, xhat, rstd = saved[t]
        eh = dh + d_out[:, t]
        if layernorm:
            dc, dv, _ = lstm_gates_fused_grad(c, v, ec=dc, eh=eh, forget_bias=1.0)
            dz, dgt, dbt = _ln4_grad(dv, xhat, rstd, gain)
            dg += dgt
            db += dbt
        else:
            dc, dz, dbt = lstm_gates_fused_grad(c, v, ec=dc, eh=eh, bias=bias, forget_bias=1.0)
            db += dbt
        dk += xh.T @ dz
        dxh = dz @ kernel.T
        dx[:, t] = dxh[:, :In]
        dh = dxh[:, In:]
    return dx.reshape(x64.shape), dc, dh, dk, db, dg


def cell_step(x, c, h, kernel, bias, forget_bias=1.0):
    """(h_next, c_next) of one FusedBasicLSTMCell step."""
    z = np.concatenate([_f64(x), _f64(h)], axis=1) @ _f64(kernel)
    c_next, h_next = lstm_gates_fused(_f64(c), z, bias=bias, forget_bias=forget_bias)
    return h_next, c_next


def cell_step_grad(x, c, h, kernel, bias, d_h=None, d_c=None, forget_bias=1.0):
    """(dx, dc, dh, dkernel, dbias) of cell_step given the gradients of h_next and c_next (None = 0)."""
    x, c, h, kernel = _f64(x), _f64(c), _f64(h), _f64(kernel)
    xh = np.concatenate([x, h], axis=1)
    z = xh @ kernel
    dc, dz, db = lstm_gates_fused_grad(c, z, ec=d_c, eh=d_h, bias=bias, forget_bias=forget_bias)
    dxh = dz @ kernel.T
    return dxh[:, :x.shape[1]], dc, dxh[:, x.shape[1]:], xh.T @ dz, db
