"""CPU oracle for the block-sparse transformer path (TEST INFRASTRUCTURE ONLY).

Plain NumPy restatement of the reference's host-side LUT construction and of its
NumPy checkers for the NT / NN / TN block-sparse attention GEMMs and the (masked)
softmax.  Imported only by tests/, __graft_entry__.smoke() and bench.py's CPU
baseline legs; the product package never imports it.

Parity status: PINNED against tests/golden/bst_*.npz, produced by importing the
reference's blocksparse/transformer.py (see tests/golden/make_golden.py).

Reference anchors (relative to the openai/blocksparse source tree):
  blocksparse/transformer.py:61-133    __init__ (nt/nn/tn lists and LUTs)
  blocksparse/transformer.py:135-159   init_softmax_mask (bit packing)
  blocksparse/transformer.py:161-181   xn_lut
  blocksparse/transformer.py:186-203   nt_test
  blocksparse/transformer.py:205-223   nn_test
  blocksparse/transformer.py:225-243   tn_test
  blocksparse/transformer.py:246-286   masked_softmax_test
  blocksparse/transformer.py:289-305   masked_softmax_grad_test
"""
import numpy as np

_MASK_DTYPE = {8: np.uint8, 16: np.uint16, 32: np.uint32, 64: np.uint64}


def _xn_lut(outs, ins, n_blocks, n_out):
    """transformer.py:161-181: header rows (offset, len) then (block, in) rows."""
    rows = [[] for _ in range(n_out)]
    for b in range(n_blocks):
        rows[outs[b]].append((b, ins[b]))
    lut = np.empty((n_out + n_blocks, 2), dtype=np.int32)
    off, longest = n_out, 0
    for o, row in enumerate(rows):
        lut[o] = (off, len(row))
        longest = max(longest, len(row))
        for e in row:
            lut[off] = e
            off += 1
    return lut, rows, longest


class TransformerOracle(object):

    def __init__(self, layout, block_size=64, heads=None, mask_callback=None):
        layout = np.asarray(layout)
        if layout.ndim == 2:
            assert heads is not None
            layout = layout[None]
        if heads is None:
            heads = layout.shape[0]
        assert block_size in (8, 16, 32, 64)
        assert layout.ndim == 3
        self.blk_size = block_size
        self.heads = heads
        self.lut_heads, self.ctx_blks_q, self.ctx_blks_k = layout.shape
        self.nn_max = self.tn_max = 0
        nt_luts, nn_luts, tn_luts = [], [], []
        self.nt_list, self.nn_list, self.tn_list = [], [], []
        self.blocks = None
        for h in range(self.lut_heads):
            qs, ks = np.nonzero(layout[h])                  # row-major == sorted (q,k), :107
            if self.blocks is None:
                self.blocks = len(qs)
            assert len(qs) == self.blocks, "number of layout blocks must be equal across heads"
            pairs = [(int(q), int(k)) for q, k in zip(qs, ks)]
            qs = [p[0] for p in pairs]
            ks = [p[1] for p in pairs]
            nn_lut, nn_rows, nn_max = _xn_lut(qs, ks, self.blocks, self.ctx_blks_q)   # :112
            tn_lut, tn_rows, tn_max = _xn_lut(ks, qs, self.blocks, self.ctx_blks_k)   # :113
            nt_luts.append(np.array(pairs, dtype=np.int32).reshape(-1, 2))
            nn_luts.append(nn_lut)
            tn_luts.append(tn_lut)
            self.nt_list.append(pairs)
            self.nn_list.append(nn_rows)
            self.tn_list.append(tn_rows)
            self.nn_max = max(self.nn_max, nn_max)
            self.tn_max = max(self.tn_max, tn_max)
        self.nt_lut = np.array(nt_luts, dtype=np.int32)
        self.nn_lut = np.array(nn_luts, dtype=np.int32)
        self.tn_lut = np.array(tn_luts, dtype=np.int32)
        self.softmax_mask = self.softmax_mask_np = None
        if mask_callback is not None:
            self._init_mask(mask_callback)

    def _init_mask(self, cb):
        """transformer.py:135-159: bit j of word r of block b == key j visible to query r."""
        bs = self.blk_size
        dt = _MASK_DTYPE[bs]
        per_head = []
        for h in range(self.lut_heads):
            words = []
            for b, (q, k) in enumerate(self.nt_list[h]):
                m = np.asarray(cb((bs, bs), h, q, k, b)).astype(bool)
                w = np.zeros(bs, dtype=np.uint64)
                for j in range(bs):
                    w |= m[:, j].astype(np.uint64) << np.uint64(j)
                words.append(w.astype(dt))
            per_head.append(words)
        self.softmax_mask_np = np.array(per_head, dtype=dt)                   # heads, blocks, bs
        self.softmax_mask = np.ascontiguousarray(self.softmax_mask_np.transpose(0, 2, 1))

    def _hl(self, h):
        return h if self.lut_heads > 1 else 0

    def _split(self, X, ctx_blks):
        B, _, S = X.shape
        return X.reshape(B, ctx_blks, self.blk_size, self.heads, S // self.heads)

    def nt(self, A, B):
        """transformer.py:186-203: C[n,h,b] = A[n,q-blk,:,h,:] @ B[n,k-blk,:,h,:].T"""
        Av, Bv = self._split(A, self.ctx_blks_q), self._split(B, self.ctx_blks_k)
        bs = self.blk_size
        C = np.empty((A.shape[0], self.heads, self.blocks, bs, bs), dtype=np.float32)
        for n in range(A.shape[0]):
            for h in range(self.heads):
                for b, (q, k) in enumerate(self.nt_list[self._hl(h)]):
                    C[n, h, b] = Av[n, q, :, h, :] @ Bv[n, k, :, h, :].T
        return C

    def nn(self, A, B):
        """transformer.py:205-223: C[n,q-blk,:,h,:] += A[n,h,b] @ B[n,k-blk,:,h,:]"""
        Bv = self._split(B, self.ctx_blks_k)
        nb, S = B.shape[0], B.shape[2]
        C = np.zeros((nb, self.ctx_blks_q, self.blk_size, self.heads, S // self.heads), dtype=np.float32)
        for n in range(nb):
            for h in range(self.heads):
                for q, row in enumerate(self.nn_list[self._hl(h)]):
                    for b, k in row:
                        C[n, q, :, h, :] += A[n, h, b] @ Bv[n, k, :, h, :]
        return C.reshape(nb, self.ctx_blks_q * self.blk_size, S)

    def tn(self, A, B):
        """transformer.py:225-243: C[n,k-blk,:,h,:] += A[n,h,b].T @ B[n,q-blk,:,h,:]"""
        Bv = self._split(B, self.ctx_blks_q)
        nb, S = B.shape[0], B.shape[2]
        C = np.zeros((nb, self.ctx_blks_k, self.blk_size, self.heads, S // self.heads), dtype=np.float32)
        for n in range(nb):
            for h in range(self.heads):
                for k, row in enumerate(self.tn_list[self._hl(h)]):
                    for b, q in row:
                        C[n, k, :, h, :] += A[n, h, b].T @ Bv[n, q, :, h, :]
        return C.reshape(nb, self.ctx_blks_k * self.blk_size, S)

    def _mask_bits(self, hl, b, k, autoregress_at_key):
        """Visible-key matrix bool[bs,bs] for block b (transformer.py:262-279)."""
        bs = self.blk_size
        words = self.softmax_mask_np[hl, b].astype(np.uint64)
        if autoregress_at_key is not None:                                     # :264-274
            ones = (1 << bs) - 1
            q0 = self.nt_list[hl][b][0] * bs
            k0 = k * bs
            out = np.empty(bs, dtype=np.uint64)
            for r in range(bs):
                sa = bs - min(max(autoregress_at_key - k0, 0), bs)
                sb = min(max(bs - 1 + k0 - (q0 + r), 0), bs)
                out[r] = int(words[r]) & (ones >> int(min(sa, sb)))
            words = out
        j = np.arange(bs, dtype=np.uint64)
        return ((words[:, None] >> j[None, :]) & np.uint64(1)).astype(bool)

    def masked_softmax(self, x, scale=1.0, autoregress_at_key=None):
        """transformer.py:246-286 (masked entries -> -FLT_MAX; max/sum over the row's blocks)."""
        y = np.empty_like(x)
        neg = -np.finfo(np.float32).max
        for n in range(x.shape[0]):
            for h in range(x.shape[1]):
                hl = self._hl(h)
                for row in self.nn_list[hl]:
                    if not row:
                        continue
                    bids = [b for b, _ in row]
                    xm = x[n, h, bids].astype(np.float32) * np.float32(scale)    # (L, bs, bs)
                    if self.softmax_mask_np is not None:
                        vis = np.stack([self._mask_bits(hl, b, k, autoregress_at_key) for b, k in row])
                        xm = np.where(vis, xm, np.float32(neg))
                    e = np.exp(xm - xm.max(axis=(0, 2), keepdims=True))
                    y[n, h, bids] = e / e.sum(axis=(0, 2), keepdims=True)
        return y

    def softmax(self, x, scale=1.0):
        saved = self.softmax_mask_np
        self.softmax_mask_np = None
        try:
            return self.masked_softmax(x, scale)
        finally:
            self.softmax_mask_np = saved

    def masked_softmax_grad(self, dy, y, scale=1.0):
        """transformer.py:289-305: dx = (dy - sum_row(dy*y)) * y * scale."""
        dx = np.empty_like(dy)
        for n in range(dy.shape[0]):
            for h in range(dy.shape[1]):
                for row in self.nn_list[self._hl(h)]:
                    if not row:
                        continue
                    bids = [b for b, _ in row]
                    d, p = dy[n, h, bids], y[n, h, bids]
                    dx[n, h, bids] = (d - (d * p).sum(axis=(0, 2), keepdims=True)) * p * scale
        return dx

    # ---- dense cross-check: ordinary attention with the layout as a block mask ----

    def dense_attention(self, Q, K, V, scale=1.0):
        bs = self.blk_size
        B, ctxq, S = Q.shape
        hs = S // self.heads
        Qh = Q.reshape(B, ctxq, self.heads, hs).transpose(0, 2, 1, 3).astype(np.float64)
        Kh = K.reshape(B, -1, self.heads, hs).transpose(0, 2, 1, 3).astype(np.float64)
        Vh = V.reshape(B, -1, self.heads, hs).transpose(0, 2, 1, 3).astype(np.float64)
        out = np.zeros_like(Qh)
        for h in range(self.heads):
            hl = self._hl(h)
            vis = np.zeros((self.ctx_blks_q * bs, self.ctx_blks_k * bs), dtype=bool)
            for b, (q, k) in enumerate(self.nt_list[hl]):
                blk = np.ones((bs, bs), bool) if self.softmax_mask_np is None else self._mask_bits(hl, b, k, None)
                vis[q * bs:(q + 1) * bs, k * bs:(k + 1) * bs] = blk
            s = np.einsum('bqd,bkd->bqk', Qh[:, h], Kh[:, h]) * scale
            s = np.where(vis[None], s, -np.inf)
            e = np.exp(s - s.max(axis=-1, keepdims=True))
            p = e / e.sum(axis=-1, keepdims=True)
            out[:, h] = np.einsum('bqk,bkd->bqd', p, Vh[:, h])
        return out.transpose(0, 2, 1, 3).reshape(B, ctxq, S)
