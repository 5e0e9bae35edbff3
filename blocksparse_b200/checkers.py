"""NumPy checker methods of the op classes (`fprop_test`, `nt_test`, ... in the reference: blocksparse/matmul.py:353-453,
blocksparse/transformer.py:186-305).

The reference carries these on the op objects as CPU test helpers; they are part of its public surface, so they exist
here too.  They are NOT a compute path: no op calls them, and they are written independently of `oracle/` (vectorised
einsum / segment sums over the LUT arrays instead of per-block loops), which makes `tests/test_checkers.py` a cross-check
of two restatements of the same reference code.
"""
import numpy as np


class MatmulCheckers(object):
    """Mixin for BlocksparseMatMul: needs updat_lut, bsize, axis, CB, KB, C, K, w_shape, fprop_list."""

    def _dense(self, W):
        bs = self.bsize
        D = np.zeros((self.CB, bs, self.KB, bs), dtype=np.float64)
        D[self.updat_lut[:, 0], :, self.updat_lut[:, 1], :] = W
        return D.reshape(self.C, self.K)

    def fprop_test(self, I, W, gate=None):
        """O = I . W over the active blocks (matmul.py:353-375)."""
        Wg = W if gate is None else W * np.asarray(gate, dtype=W.dtype).reshape(-1, 1, 1)
        D = self._dense(Wg)
        return I.astype(np.float64) @ D if self.axis else D.T @ I.astype(np.float64)

    def bprop_test(self, E, W, gate=None):
        """B = E . W^T (matmul.py:377-399)."""
        Wg = W if gate is None else W * np.asarray(gate, dtype=W.dtype).reshape(-1, 1, 1)
        D = self._dense(Wg)
        return E.astype(np.float64) @ D.T if self.axis else D @ E.astype(np.float64)

    def updat_test(self, I, E, gate=None, dw_gated=False):
        """U[w] = I[c-blk] . E[k-blk]^T over the minibatch (matmul.py:401-419)."""
        bs = self.bsize
        cs, ks = self.updat_lut[:, 0], self.updat_lut[:, 1]
        if self.axis:
            Iv = I.astype(np.float64).reshape(-1, self.CB, bs)
            Ev = E.astype(np.float64).reshape(-1, self.KB, bs)
            U = np.einsum('nbi,nbj->bij', Iv[:, cs, :], Ev[:, ks, :])
        else:
            Iv = I.astype(np.float64).reshape(self.CB, bs, -1)
            Ev = E.astype(np.float64).reshape(self.KB, bs, -1)
            U = np.einsum('bin,bjn->bij', Iv[cs], Ev[ks])
        if dw_gated and gate is not None:
            U = U * np.asarray(gate, dtype=np.float64).reshape(-1, 1, 1)
        return U

    def _column_ids(self):
        """block id -> output block column, and blocks sorted by column."""
        return self.updat_lut[:, 1].astype(np.int64)

    def l2_normalize_test(self, W, epsilon=1e-12):
        """matmul.py:421-429: every output feature of a block column is normalised over all rows of all its blocks."""
        col = self._column_ids()
        ss = np.zeros((self.KB, self.bsize), dtype=np.float64)
        np.add.at(ss, col, np.square(W.astype(np.float64)).sum(axis=1))
        norm = np.sqrt(np.maximum(ss, epsilon))
        return (W / norm[col][:, None, :]).astype(W.dtype)

    def l2_normalize_grad_test(self, W, U, epsilon=1e-12):
        """matmul.py:431-443."""
        col = self._column_ids()
        W64, U64 = W.astype(np.float64), U.astype(np.float64)
        ss = np.zeros((self.KB, self.bsize), dtype=np.float64)
        np.add.at(ss, col, np.square(W64).sum(axis=1))
        mx = np.maximum(ss, epsilon)
        red = np.zeros_like(ss)
        np.add.at(red, col, (-U64 * W64).sum(axis=1))
        red = red / mx * (ss >= epsilon)
        return ((U64 + W64 * red[col][:, None, :]) / np.sqrt(mx)[col][:, None, :]).astype(U.dtype)


class TransformerCheckers(object):
    """Mixin for BlocksparseTransformer: needs nt_lut, heads, lut_heads, blk_size, blocks, ctx_blks_q/k, softmax_mask_np."""

    def _head_lut(self, h):
        return self.nt_lut[h if self.lut_heads > 1 else 0]

    def _split_heads(self, X, ctx_blks):
        B, _, S = X.shape
        return X.reshape(B, ctx_blks, self.blk_size, self.heads, S // self.heads)

    def nt_test(self, A, B):
        """C[n,h,b] = A[n,q-blk,:,h,:] . B[n,k-blk,:,h,:]^T (transformer.py:186-203)."""
        Av, Bv = self._split_heads(A, self.ctx_blks_q), self._split_heads(B, self.ctx_blks_k)
        C = np.empty((A.shape[0], self.heads, self.blocks, self.blk_size, self.blk_size), dtype=np.float32)
        for h in range(self.heads):
            lut = self._head_lut(h)
            C[:, h] = np.einsum('nbid,nbjd->nbij', Av[:, :, :, h, :][:, lut[:, 0]], Bv[:, :, :, h, :][:, lut[:, 1]])
        return C

    def _xn_check(self, A, B, out_col, in_col, n_out, transpose):
        Bv = self._split_heads(B, self.ctx_blks_q if transpose else self.ctx_blks_k)
        nb, S = B.shape[0], B.shape[2]
        C = np.zeros((nb, n_out, self.blk_size, self.heads, S // self.heads), dtype=np.float32)
        for h in range(self.heads):
            lut = self._head_lut(h)
            Ah = A[:, h].astype(np.float32)
            if transpose:
                Ah = Ah.transpose(0, 1, 3, 2)
            prod = np.einsum('nbij,nbjd->nbid', Ah, Bv[:, :, :, h, :][:, lut[:, in_col]])
            for n in range(nb):
                Ch = np.zeros((n_out,) + prod.shape[2:], dtype=np.float32)
                np.add.at(Ch, lut[:, out_col], prod[n])
                C[n, :, :, h, :] = Ch
        return C.reshape(nb, n_out * self.blk_size, S)

    def nn_test(self, A, B):
        """C[n,q-blk] += A[n,h,b] . B[n,k-blk] (transformer.py:205-223)."""
        return self._xn_check(A, B, 0, 1, self.ctx_blks_q, False)

    def tn_test(self, A, B):
        """C[n,k-blk] += A[n,h,b]^T . B[n,q-blk] (transformer.py:225-243)."""
        return self._xn_check(A, B, 1, 0, self.ctx_blks_k, True)

    def _visible(self, h, autoregress_at_key=None):
        """bool [blocks, bs, bs]: key j of block b visible to query r (bit j of mask word r; transformer.py:262-279)."""
        bs = self.blk_size
        if self.softmax_mask_np is None:
            return np.ones((self.blocks, bs, bs), dtype=bool)
        hl = h if self.lut_heads > 1 else 0
        words = self.softmax_mask_np[hl].astype(np.uint64)                    # [blocks, bs]
        if autoregress_at_key is not None:
            lut = self._head_lut(h).astype(np.int64)
            q0, k0 = lut[:, 0] * bs, lut[:, 1] * bs
            r = np.arange(bs, dtype=np.int64)
            sa = bs - np.clip(autoregress_at_key - k0, 0, bs)                 # [blocks]
            sb = np.clip(bs - 1 + k0[:, None] - (q0[:, None] + r[None, :]), 0, bs)
            shift = np.minimum(sa[:, None], sb).astype(np.uint64)
            ones = np.uint64((1 << bs) - 1) if bs < 64 else np.uint64(0xFFFFFFFFFFFFFFFF)
            shifted = np.where(shift >= 64, np.uint64(0), ones >> np.minimum(shift, np.uint64(63)))
            words = words & shifted
        j = np.arange(bs, dtype=np.uint64)
        return ((words[:, :, None] >> j[None, None, :]) & np.uint64(1)).astype(bool)

    def masked_softmax_test(self, x, scale=1.0, autoregress_at_key=None):
        """Row softmax over all the blocks of a query-block row; masked entries count as -FLT_MAX (transformer.py:246-286)."""
        y = np.empty_like(x)
        neg = -np.finfo(np.float32).max
        bs = self.blk_size
        for h in range(self.heads):
            q = self._head_lut(h)[:, 0]
            vis = self._visible(h, autoregress_at_key)
            xm = np.where(vis[None], x[:, h].astype(np.float32) * np.float32(scale), np.float32(neg))
            mx = np.full((x.shape[0], self.ctx_blks_q, bs), neg, dtype=np.float32)
            for n in range(x.shape[0]):
                np.maximum.at(mx[n], q, xm[n].max(axis=2))
            e = np.exp(xm - mx[:, q][..., None])
            sm = np.zeros((x.shape[0], self.ctx_blks_q, bs), dtype=np.float32)
            for n in range(x.shape[0]):
                np.add.at(sm[n], q, e[n].sum(axis=2))
            y[:, h] = e / sm[:, q][..., None]
        return y

    def masked_softmax_grad_test(self, dy, y, scale=1.0):
        """dx = (dy - sum_row(dy * y)) * y * scale (transformer.py:289-305)."""
        dx = np.empty_like(dy)
        bs = self.blk_size
        for h in range(self.heads):
            q = self._head_lut(h)[:, 0]
            prod = (dy[:, h] * y[:, h]).sum(axis=3)
            tot = np.zeros((dy.shape[0], self.ctx_blks_q, bs), dtype=prod.dtype)
            for n in range(dy.shape[0]):
                np.add.at(tot[n], q, prod[n])
            dx[:, h] = (dy[:, h] - tot[:, q][..., None]) * y[:, h] * scale
        return dx


# ---- module-level checkers of the dense ops (reference blocksparse/transformer.py:536-549, 609-656) ----------------------
# The reference's NumPy checkers restated with NumPy broadcasting of the mask, which also gives the right answer for a
# (D1, 1, D3) mask where the reference's flattening checker does not (transformer.py:613), and with a stable sort, so
# that ties rank by index ascending like the ops.
def _masked_values(x, mask, scale):
    x = np.asarray(x, dtype=np.float32)
    if mask is None:
        return x * np.float32(scale)
    m = np.broadcast_to(np.asarray(mask, dtype=np.float32), x.shape)
    return np.where(m != 0, x * m * np.float32(scale), -np.finfo(np.float32).max).astype(np.float32)


def _rank(v):
    """Column order of each row of v (..., D3): value descending, then index ascending."""
    return np.argsort(-v, axis=-1, kind="stable")


def masked_softmax_test(x, mask=None, scale=1.0):
    """transformer.py:609-625."""
    y = _masked_values(x, mask, scale)
    e = np.exp(y - y.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)


def masked_top_k_softmax_test(x, k, mask=None, scale=1.0):
    """transformer.py:627-649."""
    y = _masked_values(x, mask, scale)
    top = _rank(y)[..., :k]
    v = np.take_along_axis(y, top, axis=-1)
    e = np.exp(v - v[..., :1])
    z = np.zeros(y.shape, dtype=np.float32)
    np.put_along_axis(z, top, (e / e.sum(axis=-1, keepdims=True)).astype(np.float32), axis=-1)
    return z


def masked_softmax_grad_test(dy, y, mask=None, scale=1.0):
    """transformer.py:651-656."""
    m = 1.0 if mask is None else mask
    return (dy - np.sum(dy * y, axis=-1, keepdims=True)) * y * m * scale


def rectified_top_k_test(x, k, rebase=True):
    """transformer.py:536-549."""
    x = np.asarray(x, dtype=np.float32)
    top = _rank(x)[..., :k]
    v = np.take_along_axis(x, top, axis=-1)
    base = np.maximum(v[..., k - 1:k], 0.0) if rebase else np.zeros_like(v[..., :1])
    y = np.zeros(x.shape, dtype=np.float32)
    np.put_along_axis(y, top, np.maximum(v, base) - base, axis=-1)
    return y


# ---- module-level checkers of layer norm (reference blocksparse/norms.py, layer_norm_test / layer_norm_grad_test) ------
# Restated on a (rows, segments, L) view: the feature axis last, or first (x viewed as (K, N) and transposed).
def _segment_view(a, axis, segments):
    a = np.asarray(a)
    K = a.shape[axis]
    a2 = a.reshape(K, -1).T if axis == 0 else a.reshape(-1, K)
    return a2.reshape(a2.shape[0], segments, K // segments)


def _segment_unview(v, shape, axis):
    v = v.reshape(v.shape[0], -1)
    return (v.T if axis == 0 else v).reshape(shape)


def layer_norm_test(x, g, b, axis=1, segments=1, epsilon=1e-6, relu=False):
    """y = relu?(xhat * g + b), the mean and the (biased) variance per segment of each row along `axis`."""
    xs = _segment_view(x, axis, segments)
    gs, bs = (np.asarray(p).reshape(1, segments, -1) for p in (g, b))
    xhat = (xs - xs.mean(axis=2, keepdims=True)) / np.sqrt(xs.var(axis=2, keepdims=True) + epsilon)
    y = xhat * gs + bs
    if relu:
        y = np.maximum(y, 0.0)
    return _segment_unview(y, np.shape(x), axis).astype(np.result_type(x, np.float32))


def layer_norm_grad_test(dy, x, g, b, axis=1, segments=1, epsilon=1e-6, relu=False):
    """(dx, dg, db) of layer_norm_test; with relu, dy is masked where the pre-activation is not positive. dg and db
    have g's shape: (K, 1) for axis 0, (1, K) otherwise, as the reference returns them."""
    xs, dys = _segment_view(x, axis, segments), _segment_view(dy, axis, segments)
    gs, bs = (np.asarray(p).reshape(1, segments, -1) for p in (g, b))
    L = xs.shape[2]
    rstd = 1.0 / np.sqrt(xs.var(axis=2, keepdims=True) + epsilon)
    xhat = (xs - xs.mean(axis=2, keepdims=True)) * rstd
    if relu:
        dys = dys * (xhat * gs + bs > 0)
    dg = (dys * xhat).sum(axis=0).reshape(-1)
    db = dys.sum(axis=0).reshape(-1)
    dyg = dys * gs
    dx = (dyg - (xhat * (dyg * xhat).sum(axis=2, keepdims=True) + dyg.sum(axis=2, keepdims=True)) / L) * rstd
    shape = (-1, 1) if axis == 0 else (1, -1)
    dt = np.result_type(x, np.float32)
    return (_segment_unview(dx, np.shape(x), axis).astype(dt), dg.reshape(shape).astype(dt), db.reshape(shape).astype(dt))


def sparse_relu_test(x, alpha=1.0):
    """y = max(x - (mean + alpha * std), 0) along the last axis, std the population standard deviation (the reference's
    checker, lstm.py:111-117)."""
    x = np.asarray(x)
    cutoff = x.mean(axis=-1, keepdims=True) + alpha * x.std(axis=-1, keepdims=True)
    return np.maximum(x - cutoff, 0.0)


class ConvCheckers(object):
    """Mixin for BlocksparseConv / BlocksparseDeconv (conv.py:540-661, 746-801): needs BCK, blocks, C, K, DHW, MPQ, trs,
    sizeF, f_shape and the spatial tables _lut_f / _lut_b ([positions][trs], -1 where a tap reads nothing). F and U
    are lists of per-block arrays of f_shape(block), as in the reference; results are float64, updat's and l2's
    collapsed to [sizeF] as the reference's are (in float32 there)."""

    @staticmethod
    def _gather(a, lut):
        """a (N, C, P) -> (N, C, P_out, trs), zero where lut is -1."""
        a = np.asarray(a, dtype=np.float64)
        N, C = a.shape[:2]
        a = np.concatenate([a.reshape(N, C, -1), np.zeros((N, C, 1))], axis=2)
        return a[:, :, np.where(lut < 0, a.shape[2] - 1, lut)]

    def _f3(self, block, f):
        return np.asarray(f, dtype=np.float64).reshape(len(self.BCK[block][1]), len(self.BCK[block][0]), self.trs)

    def _conv_fprop(self, F, I):
        N = I.shape[0]
        cols = self._gather(I, self._lut_f)
        O = np.zeros((N, self.K, int(np.prod(self.MPQ))))
        for b, (lutC, lutK) in enumerate(self.BCK):
            O[:, lutK] += np.einsum("ncpt,kct->nkp", cols[:, lutC], self._f3(b, F[b]))
        return O.reshape([N, self.K] + list(self.MPQ))

    def _conv_bprop(self, F, E):
        N = E.shape[0]
        cols = self._gather(E, self._lut_b)
        O = np.zeros((N, self.C, int(np.prod(self.DHW))))
        for b, (lutC, lutK) in enumerate(self.BCK):
            O[:, lutC] += np.einsum("nkpt,kct->ncp", cols[:, lutK], self._f3(b, F[b]))
        return O.reshape([N, self.C] + list(self.DHW))

    def _conv_updat(self, E, I):
        N = I.shape[0]
        cols = self._gather(I, self._lut_f)
        E = np.asarray(E, dtype=np.float64).reshape(N, self.K, -1)
        return np.concatenate([np.einsum("nkp,ncpt->kct", E[:, lutK], cols[:, lutC]).ravel()
                               for lutC, lutK in self.BCK])

    def fprop_test(self, F, I, alpha=1.0):
        """O = conv(I, F) (conv.py:540-563); the deconv's is the conv's bprop (conv.py:746-747)."""
        return (self._conv_bprop(F, I) if self.deconv else self._conv_fprop(F, I)) * alpha

    def bprop_test(self, F, I, alpha=1.0):
        """dI from dO = I (conv.py:565-589); the deconv's is the conv's fprop."""
        return (self._conv_fprop(F, I) if self.deconv else self._conv_bprop(F, I)) * alpha

    def updat_test(self, E, I, alpha=1.0, transpose=False):
        """dF, collapsed to [sizeF] (conv.py:591-615); the deconv swaps E and I (conv.py:752-753)."""
        return (self._conv_updat(I, E) if self.deconv else self._conv_updat(E, I)) * alpha

    def _l2_axes(self):
        return (0, 2) if self.deconv else (1, 2)

    def l2_normalize_test(self, F, gain=None, epsilon=1e-12):
        """Each block's rows (KCTRS: per output channel; CKTRS for the deconv: per input channel) scaled to unit l2
        norm and by gain (conv.py:617-631, 756-772)."""
        out, off = [], 0
        for b, f in enumerate(F):
            f = self._f3(b, f)
            ax = self._l2_axes()
            nrm = np.sqrt(np.maximum(np.sum(f * f, axis=ax, keepdims=True), epsilon))
            y = f / nrm
            if gain is not None:
                n = f.shape[1 if self.deconv else 0]
                g = np.asarray(gain, dtype=np.float64)[off:off + n]
                y = y * (g.reshape(1, n, 1) if self.deconv else g.reshape(n, 1, 1))
                off += n
            out.append(y.ravel())
        return np.concatenate(out)

    def l2_normalize_grad_test(self, F, U, gain=None, epsilon=1e-12):
        """(dF collapsed to [sizeF], dgain or None) (conv.py:633-661, 774-801)."""
        D, dg, off = [], [], 0
        for b, (f, u) in enumerate(zip(F, U)):
            f, u = self._f3(b, f), self._f3(b, u)
            ax = self._l2_axes()
            n = f.shape[1 if self.deconv else 0]
            shape = (1, n, 1) if self.deconv else (n, 1, 1)
            g = np.ones(shape) if gain is None else np.asarray(gain, dtype=np.float64)[off:off + n].reshape(shape)
            ss = np.sum(f * f, axis=ax, keepdims=True)
            mx = np.maximum(ss, epsilon)
            rn = 1.0 / np.sqrt(mx)
            dg.append(np.sum(u * f * rn, axis=ax).ravel())
            D.append(((u * g + f * (ss >= epsilon) * np.sum(-u * f * g / mx, axis=ax, keepdims=True)) * rn).ravel())
            off += n
        return np.concatenate(D), (None if gain is None else np.concatenate(dg))


class EdgeBiasCheckers(object):
    """Mixin for ConvEdgeBias (conv.py:163-214): needs layout, shape, edgeBiasDim and the position table _pos_edge
    (the edge pattern of each output position, or -1). x, dy: NumPy arrays of the op's input shape; g, b: self.shape.
    Written on the position table rather than the reference's per-edge position lists."""

    def _flat(self, a):
        a = np.asarray(a)
        N, P = a.shape[0], len(self._pos_edge)
        return a.reshape(N, P, a.shape[-1]) if self.layout else a.reshape(N, a.shape[1], P)

    def _per_position(self, p):
        """p (edges, K) or (K, edges) -> per output position, broadcastable against _flat: 1 off the edges."""
        e = self._pos_edge
        p = np.asarray(p)
        if self.layout:
            return np.where((e >= 0)[:, None], p[np.maximum(e, 0)], 1)[None]
        return np.where((e >= 0)[None, :], p[:, np.maximum(e, 0)], 1)[None]

    def edge_bias_test(self, x, g, b):
        if not self.edgeBiasDim:
            return x
        mask = (self._pos_edge >= 0)[None, :, None] if self.layout else (self._pos_edge >= 0)[None, None, :]
        xf = self._flat(x)
        bias = np.where(mask, self._per_position(b), 0)
        y = np.where(mask, xf * self._per_position(g) + bias, xf)
        return y.astype(np.asarray(x).dtype).reshape(np.shape(x))

    def edge_bias_grad_test(self, dy, x, g):
        """(dx, dg, db): dx = g * dy at edge positions, dg = sum(dy * x), db = sum(dy) per (edge, k); (dy, None, None)
        without edges."""
        if not self.edgeBiasDim:
            return dy, None, None
        d, xf = self._flat(dy), self._flat(x)
        mask = (self._pos_edge >= 0)[None, :, None] if self.layout else (self._pos_edge >= 0)[None, None, :]
        dx = np.where(mask, d * self._per_position(g), d).astype(np.asarray(dy).dtype).reshape(np.shape(dy))
        E = self.edgeBiasDim
        onehot = (self._pos_edge[:, None] == np.arange(E)[None, :]).astype(np.float64)     # (P, E)
        if self.layout:
            dg = np.einsum("npk,pe->ek", d * xf, onehot)
            db = np.einsum("npk,pe->ek", d, onehot)
        else:
            dg = np.einsum("nkp,pe->ke", d * xf, onehot)
            db = np.einsum("nkp,pe->ke", d, onehot)
        return dx, dg.astype(np.float32), db.astype(np.float32)
