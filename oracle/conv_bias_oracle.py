"""float64 restatement of the reference's conv edge bias and cwise_linear (blocksparse/conv.py:55-219, 960-998), in
plain loops: the edge table builder, edge_bias_test / edge_bias_grad_test, cwise_linear_test / cwise_linear_grad_test,
and the bias_first (swap) gradient, which only the reference's kernel has (src/cwise_linear_op_gpu.cu:41-44).

undilated_pad=True reproduces the reference's SAME padding, which ignores the dilation; the default is TensorFlow's,
with the dilated filter extent. The two agree at dilation 1."""
import itertools

import numpy as np


def _expand(d, v=1):
    return [v] * (3 - len(d)) + list(d)


def _fprop_taps(q, X, S, pad, stride, dilate):
    out = []
    for s in range(S):
        x = q * stride - pad + s * dilate
        out.append(x if 0 <= x < X else -1)
    return out


def _bprop_taps(x, Q, S, pad, stride, dilate):
    out = []
    for s in reversed(range(S)):
        q = x - ((S - 1) * dilate - pad) + s * dilate
        if q % stride:
            out.append(-2)
        else:
            out.append(q // stride if 0 <= q // stride < Q else -1)
    return out


class EdgeBias(object):
    def __init__(self, y_shape, x_shape, w_shape, strides=None, padding="SAME", data_format="NHWC", dilations=None,
                 deconv=False, undilated_pad=False):
        self.layout = 0 if data_format in ("NCW", "NCHW", "NCDHW") else 1
        sdim, cdim = (slice(1, -1), -1) if self.layout else (slice(2, None), 1)
        C, K = x_shape[cdim], y_shape[cdim]
        MPQ, DHW, TRS = _expand(y_shape[sdim]), _expand(x_shape[sdim]), _expand(w_shape[:-2])
        st = [1, 1, 1] if strides is None else _expand(list(strides)[sdim])
        dl = [1, 1, 1] if dilations is None else _expand(list(dilations)[sdim])
        if padding.upper() == "VALID":
            pad = [0, 0, 0]
        else:
            pad = []
            for S, Q, W, s, d in zip(TRS, MPQ, DHW, st, dl):
                extent = S if undilated_pad else (S - 1) * d + 1
                pad.append(max((Q - 1) * s + extent - W, 0) // 2)
        self.padding = pad
        fn = _fprop_taps
        if deconv:
            fn, MPQ, DHW, K = _bprop_taps, DHW, MPQ, C
        self.MPQ, self.K = MPQ, K
        luts = [[fn(m, DHW[i], TRS[i], pad[i], st[i], dl[i]) for m in range(MPQ[i])] for i in range(3)]
        groups = {}
        for m, p, q in itertools.product(*[range(n) for n in MPQ]):
            key = tuple((a, b, c) for (a, d), (b, h), (c, w) in itertools.product(
                enumerate(luts[0][m]), enumerate(luts[1][p]), enumerate(luts[2][q])) if -1 in (d, h, w))
            if key:
                groups.setdefault(key, []).append((m * MPQ[1] + p) * MPQ[2] + q)
        self.edgeBiasMap = sorted(groups.values(), key=lambda v: v[0])
        self.edgeBiasDim = len(self.edgeBiasMap)
        self.edgeEntries = sum(len(v) for v in self.edgeBiasMap)
        self.shape = (self.edgeBiasDim, K) if self.layout else (K, self.edgeBiasDim)

    def lut(self):
        """The reference's int32 table: (offset, count) per edge, the positions, zeros to a multiple of 4."""
        head, data, off = [], [], 2 * self.edgeBiasDim
        for v in self.edgeBiasMap:
            head += [off, len(v)]
            data += v
            off += len(v)
        return np.array(head + data + [0] * ((4 - len(data) % 4) % 4), np.int32)

    def _view(self, a):
        a = np.asarray(a, np.float64)
        N, P = a.shape[0], int(np.prod(self.MPQ))
        return a.reshape(N, P, a.shape[-1]) if self.layout else np.swapaxes(a.reshape(N, a.shape[1], P), 1, 2)

    def _param(self, p, e):
        p = np.asarray(p, np.float64)
        return p[e, :] if self.layout else p[:, e]

    def _unview(self, v, shape):
        return (v if self.layout else np.swapaxes(v, 1, 2)).reshape(shape)

    def edge_bias(self, x, g, b):
        """y: x * g + b at the positions of each edge, x elsewhere; (N, positions, K) views in both layouts."""
        y = self._view(x).copy()
        for e, pos in enumerate(self.edgeBiasMap):
            y[:, pos, :] = y[:, pos, :] * self._param(g, e) + self._param(b, e)
        return self._unview(y, np.shape(x))

    def edge_bias_grad(self, dy, x, g):
        """(dx, dg, db): dx = g * dy at edge positions, dg = sum(dy * x), db = sum(dy) over N and the edge's positions."""
        d, xv = self._view(dy), self._view(x)
        dx = d.copy()
        dg, db = np.zeros(self.shape), np.zeros(self.shape)
        for e, pos in enumerate(self.edgeBiasMap):
            dx[:, pos, :] *= self._param(g, e)
            sg, sb = (d[:, pos, :] * xv[:, pos, :]).sum(axis=(0, 1)), d[:, pos, :].sum(axis=(0, 1))
            if self.layout:
                dg[e, :], db[e, :] = sg, sb
            else:
                dg[:, e], db[:, e] = sg, sb
        return self._unview(dx, np.shape(dy)), dg, db


def _bcast(x, v):
    shape = [1] * np.ndim(x)
    shape[1] = np.shape(x)[1]
    return np.asarray(v, np.float64).reshape(shape)


def cwise_linear(x, a=None, b=None, relu=False, bias_first=False):
    x = np.asarray(x, np.float64)
    a = 1.0 if a is None else _bcast(x, a)
    b = 0.0 if b is None else _bcast(x, b)
    y = a * (x + b) if bias_first else a * x + b
    return np.maximum(y, 0.0) if relu else y


def cwise_linear_grad(dy, x, a=None, b=None, relu=False, bias_first=False):
    """(dx, da, db) over axis 1. bias_first: da = sum dy * (x + b), db = sum dy * a (cwise_linear_op_gpu.cu:41-44)."""
    dy, x = np.asarray(dy, np.float64), np.asarray(x, np.float64)
    A = 1.0 if a is None else _bcast(x, a)
    B = 0.0 if b is None else _bcast(x, b)
    axes = tuple(i for i in range(dy.ndim) if i != 1)
    if relu:
        dy = dy * ((A * (x + B) if bias_first else A * x + B) > 0)
    dx = A * dy
    if bias_first:
        return dx, np.sum(dy * (x + B), axis=axes), np.sum(dx, axis=axes)
    return dx, np.sum(dy * x, axis=axes), np.sum(dy, axis=axes)
