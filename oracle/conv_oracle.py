"""Float64 oracle for the block-sparse conv: a restatement of the reference's spatial helpers and NumPy checkers
(blocksparse/conv.py), written as direct loops over output positions and filter taps rather than the reference's
slices. Nothing under blocksparse_b200/ imports it.

  get_padding / out_dim / in_dim       conv.py:1016-1035
  fprop_lut / bprop_lut                conv.py:1037-1061 (per dimension; bprop lists taps flipped, -2 marks a hole)
  Conv.f_shape / collapse_filter       conv.py:490-499, 523-529
  Conv.fprop / bprop / updat           conv.py:540-615 (the deconv: 746-753)
  Conv.l2_normalize(_grad)             conv.py:617-661 (KCTRS), 756-801 (CKTRS)
"""
import numpy as np


def dilation_size(S, dilate):
    return S * dilate - dilate + 1


def out_dim(S, W, padding, stride, dilate):
    return -(-(W - dilation_size(S, dilate) + 1 + 2 * padding) // stride)


def in_dim(S, W, padding, stride, dilate):
    return W * stride + S - 2 * padding - (S & 1)


def expand(dims, fill=1):
    return [fill] * (3 - len(dims)) + list(dims)


def get_padding(padding, TRS, dilates):
    if isinstance(padding, str):
        return [dilation_size(S, d) // 2 for S, d in zip(TRS, dilates)] if padding.upper() == "SAME" else [0, 0, 0]
    return expand(padding, 0)


def fprop_lut(q, X, S, padding, stride, dilate):
    """Input coordinate each tap of output coordinate q reads, -1 past the edge."""
    xs = [q * stride - padding + s * dilate for s in range(S)]
    return [x if 0 <= x < X else -1 for x in xs]


def bprop_lut(x, Q, S, padding, stride, dilate):
    """Output coordinate each (flipped) tap of input coordinate x receives from: -1 past the edge, -2 in a stride
    hole."""
    out = []
    for s in reversed(range(S)):
        q = x + padding - s * dilate
        out.append(-2 if q % stride else (q // stride if 0 <= q // stride < Q else -1))
    return out


class Conv(object):
    """BCK as the reference takes it; deconv=True gives the BlocksparseDeconv (C <=> K, DHW <=> MPQ swapped)."""

    def __init__(self, BCK, TRS, DHW, MPQ=None, strides=(1, 1, 1), dilates=(1, 1, 1), padding="SAME", deconv=False):
        self.userTRS = list(TRS)
        TRS, DHW, strides, dilates = expand(TRS), expand(DHW), expand(strides), expand(dilates)
        pad = get_padding(padding, TRS, dilates)
        if deconv:
            BCK = [[k, c] for c, k in BCK]
            if MPQ is None:
                MPQ = [in_dim(*d) for d in zip(TRS, DHW, pad, strides, dilates)]
            DHW, MPQ = expand(MPQ), DHW
        elif MPQ is None:
            MPQ = [out_dim(*d) for d in zip(TRS, DHW, pad, strides, dilates)]
        self.BCK, self.TRS, self.DHW, self.MPQ, self.padding = BCK, TRS, DHW, expand(MPQ), pad
        self.strides, self.dilates, self.deconv = strides, dilates, deconv
        self.C = len({c for lc, _ in BCK for c in lc})
        self.K = len({k for _, lk in BCK for k in lk})
        self.sizeF = sum(len(lc) * len(lk) for lc, lk in BCK) * int(np.prod(TRS))

    def f_shape(self, block=None):
        if block is None:
            sizes = {(len(lk), len(lc)) for lc, lk in self.BCK}
            if len(sizes) == 1:
                kb, cb = sizes.pop()
                return [len(self.BCK), kb, cb] + self.userTRS
            return [self.sizeF]
        lc, lk = self.BCK[block]
        return [len(lk), len(lc)] + self.userTRS

    def collapse_filter(self, F):
        return np.concatenate([np.asarray(f, dtype=np.float64).ravel() for f in F])

    def split_filter(self, flat):
        out, off = [], 0
        for lc, lk in self.BCK:
            n = len(lc) * len(lk) * int(np.prod(self.TRS))
            out.append(np.asarray(flat[off:off + n], dtype=np.float64).reshape([len(lk), len(lc)] + self.TRS))
            off += n
        return out

    def _taps(self):
        """(output position, tap, input position) triples of the conv, over the 3-D grids."""
        fd = list(zip(self.TRS, self.padding, self.strides, self.dilates))
        for m, p, q in np.ndindex(*self.MPQ):
            luts = [fprop_lut(o, X, *f) for o, X, f in zip((m, p, q), self.DHW, fd)]
            for t, r, s in np.ndindex(*self.TRS):
                d, h, w = luts[0][t], luts[1][r], luts[2][s]
                if min(d, h, w) >= 0:
                    yield (m, p, q), (t, r, s), (d, h, w)

    def _fprop(self, F, I):
        I = np.asarray(I, dtype=np.float64).reshape([I.shape[0], self.C] + self.DHW)
        O = np.zeros([I.shape[0], self.K] + self.MPQ)
        for (lc, lk), f in zip(self.BCK, F):
            f = f.reshape([len(lk), len(lc)] + self.TRS)
            for o, t, i in self._taps():
                O[(slice(None), lk) + o] += I[(slice(None), lc) + i] @ f[(slice(None), slice(None)) + t].T
        return O

    def _bprop(self, F, E):
        E = np.asarray(E, dtype=np.float64).reshape([E.shape[0], self.K] + self.MPQ)
        O = np.zeros([E.shape[0], self.C] + self.DHW)
        for (lc, lk), f in zip(self.BCK, F):
            f = f.reshape([len(lk), len(lc)] + self.TRS)
            for o, t, i in self._taps():
                O[(slice(None), lc) + i] += E[(slice(None), lk) + o] @ f[(slice(None), slice(None)) + t]
        return O

    def _updat(self, E, I):
        N = I.shape[0]
        I = np.asarray(I, dtype=np.float64).reshape([N, self.C] + self.DHW)
        E = np.asarray(E, dtype=np.float64).reshape([N, self.K] + self.MPQ)
        U = []
        for lc, lk in self.BCK:
            u = np.zeros([len(lk), len(lc)] + self.TRS)
            for o, t, i in self._taps():
                u[(slice(None), slice(None)) + t] += E[(slice(None), lk) + o].T @ I[(slice(None), lc) + i]
            U.append(u)
        return self.collapse_filter(U)

    def fprop(self, F, I):
        return self._bprop(F, I) if self.deconv else self._fprop(F, I)

    def bprop(self, F, E):
        return self._fprop(F, E) if self.deconv else self._bprop(F, E)

    def updat(self, E, I):
        return self._updat(I, E) if self.deconv else self._updat(E, I)

    def _rows(self, f):
        """f (K_b, C_b, TRS...) as rows of the normalisation: per output channel (KCTRS), per input channel (CKTRS)."""
        f = f.reshape(f.shape[0], f.shape[1], -1)
        return np.moveaxis(f, 1, 0) if self.deconv else f

    def l2_normalize(self, F, gain=None, epsilon=1e-12):
        out, off = [], 0
        for f in F:
            r = self._rows(f)
            nrm = np.sqrt(np.maximum((r * r).sum(axis=(1, 2)), epsilon))
            g = np.ones(len(r)) if gain is None else np.asarray(gain, dtype=np.float64)[off:off + len(r)]
            y = r * (g / nrm)[:, None, None]
            out.append((np.moveaxis(y, 0, 1) if self.deconv else y).ravel())
            off += len(r)
        return np.concatenate(out)

    def l2_normalize_grad(self, F, U, gain=None, epsilon=1e-12):
        D, dg, off = [], [], 0
        for f, u in zip(F, U):
            r, du = self._rows(f), self._rows(u)
            ss = (r * r).sum(axis=(1, 2))
            mx = np.maximum(ss, epsilon)
            s = (du * r).sum(axis=(1, 2))
            g = np.ones(len(r)) if gain is None else np.asarray(gain, dtype=np.float64)[off:off + len(r)]
            d = (du * g[:, None, None] - r * ((ss >= epsilon) * s * g / mx)[:, None, None]) / np.sqrt(mx)[:, None, None]
            D.append((np.moveaxis(d, 0, 1) if self.deconv else d).ravel())
            dg.append(s / np.sqrt(mx))
            off += len(r)
        return np.concatenate(D), (None if gain is None else np.concatenate(dg))
