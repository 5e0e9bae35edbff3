"""CPU oracle for the block-sparse matmul path (TEST INFRASTRUCTURE ONLY).

This file is a plain NumPy restatement of the reference's host-side algorithm and
of its NumPy checkers.  It is imported only by tests/, __graft_entry__.smoke() and
the cpu_baseline / --impl reference legs of bench.py.  The product package
(blocksparse_b200/) never imports it.

Parity status: PINNED.  tests/test_oracle_golden.py checks every function here
against fixtures in tests/golden/ that were produced by importing the reference's
own blocksparse/matmul.py (TensorFlow mocked, see tests/golden/make_golden.py).

Reference anchors (relative to the openai/blocksparse source tree):
  blocksparse/utils.py:95-103     z_order_2d
  blocksparse/matmul.py:82-162    BlocksparseMatMul.__init__ (block order, lists)
  blocksparse/matmul.py:172-270   xprop_lut (segments, locks, wire format)
  blocksparse/matmul.py:353-375   fprop_test
  blocksparse/matmul.py:377-399   bprop_test
  blocksparse/matmul.py:401-419   updat_test
"""
import numpy as np

SEG_MAX = (1 << 63) - 1


def ceil_div(x, y):
    return -(-x // y)


def z_order_2d(x, y):
    """Morton code with x on the even bits, y on the odd bits (utils.py:95-103)."""
    x, y = int(x), int(y)
    code, bit = 0, 0
    while (x >> bit) or (y >> bit):
        code |= ((x >> bit) & 1) << (2 * bit)
        code |= ((y >> bit) & 1) << (2 * bit + 1)
        bit += 1
    return code


def _segment_lut(n_out, ins, outs, wids, order, max_seg, min_seg):
    """Restates xprop_lut (matmul.py:172-270).

    `order` enumerates blocks grouped by output index.  Returns
    (cols, lut, shared_bytes, n_segments, n_locks) where `cols` is the
    un-segmented per-output list [(out, [(in, w), ...]), ...] and `lut` is the
    int32 wire format: 4 ints of header per segment (offset in int2 units,
    length, out index, 1-based lock id or 0) followed by (in, w) pairs.
    """
    remaining = [0] * n_out
    for i in order:
        remaining[outs[i]] += 1                                 # :183-185

    segs, cols, lock_of, seen = [], [], {}, set()
    locks = 0
    cur_out = outs[order[0]]
    seg, col, n_seg_for_out = [], [], 0

    def close_output(o):
        nonlocal seg, col, n_seg_for_out, locks
        cols.append((o, col))                                   # :194-195
        col = []
        if seg:                                                 # :198-201
            segs.append((o, seg))
            seg = []
            n_seg_for_out += 1
        if n_seg_for_out > 1:                                   # :203-206
            locks += 1
            lock_of[o] = locks
        n_seg_for_out = 0

    for i in order:
        o = outs[i]
        seen.add(o)
        if o != cur_out:
            close_output(cur_out)
            cur_out = o
        col.append((ins[i], wids[i]))
        seg.append((ins[i], wids[i]))
        remaining[o] -= 1
        if len(seg) >= max_seg and remaining[o] >= min_seg:     # :218
            segs.append((o, seg))
            seg = []
            n_seg_for_out += 1
    close_output(cur_out)                                       # :224-230

    for o in range(n_out):                                      # :233-236
        if o not in seen:
            segs.append((o, []))
            cols.append((o, []))

    n_blocks = len(wids)
    lut = np.empty(4 * len(segs) + 2 * n_blocks, dtype=np.int32)
    off, longest = 4 * len(segs), 0
    for s, (o, entries) in enumerate(segs):                     # :243-252
        lut[4 * s:4 * s + 4] = (off // 2, len(entries), o, lock_of.get(o, 0))
        longest = max(longest, len(entries))
        for e in entries:
            lut[off:off + 2] = e
            off += 2
    return cols, lut, longest * 8, len(segs), locks


class MatmulOracle(object):
    """Restatement of BlocksparseMatMul's host state and NumPy checkers.

    Block enumeration follows the *intended* behaviour of matmul.py:113-117
    (blocks discovered in column-major order: sorted by k then c); modern SciPy's
    sparse.find no longer returns them in that order, hence the explicit sort.
    """

    def __init__(self, layout, block_size=32, feature_axis=0, z_order=True):
        layout = np.asarray(layout)
        assert layout.ndim == 2
        ok = (feature_axis == 0 and block_size in (8, 16, 32)) or \
             (feature_axis == 1 and block_size in (32, 64))
        if not ok:
            raise ValueError("Unsupported block size with this feature axis")   # :84-89
        self.axis, self.bsize = feature_axis, block_size
        lay = (layout != 0).astype(np.int32)
        CB, KB = lay.shape

        col_sizes = lay.sum(axis=0)                                # :94
        big = int(col_sizes.max())
        small = int(col_sizes[np.nonzero(col_sizes)].min())
        max_seg = max(ceil_div(big, 4), small * 2) if big / small > 2.0 else SEG_MAX   # :97-100
        min_seg = max(ceil_div(max_seg, 4), 4)                     # :105

        # column-major discovery order: k ascending, then c ascending
        ks, cs = np.nonzero(lay.T)
        cs, ks = [int(c) for c in cs], [int(k) for k in ks]
        n = len(cs)
        by_k = list(range(n))
        by_c = sorted(by_k, key=lambda i: cs[i])                   # :117 (stable)

        wid = list(range(n))
        if z_order:                                                # :121-126
            ranked = sorted((z_order_2d(cs[i], ks[i]), i) for i in range(n))
            self.updat_list = []
            for b, (_, i) in enumerate(ranked):
                wid[i] = b
                self.updat_list.append((cs[i], ks[i]))
        else:
            self.updat_list = list(zip(cs, ks))                    # :129
        self.updat_lut = np.array(self.updat_list, dtype=np.int32).reshape(-1, 2)

        f = _segment_lut(KB, cs, ks, wid, by_k, max_seg, min_seg)  # :137
        b = _segment_lut(CB, ks, cs, wid, by_c, max_seg, min_seg)  # :138
        (self.fprop_list, self.fprop_lut, self.fprop_shared,
         self.fprop_segments, self.fprop_locks) = f
        (self.bprop_list, self.bprop_lut, self.bprop_shared,
         self.bprop_segments, self.bprop_locks) = b

        self.blocks = n
        self.CB, self.KB = CB, KB
        self.C, self.K = CB * block_size, KB * block_size
        self.w_shape = (n, block_size, block_size)
        self.flops = n * block_size * block_size * 2
        self.sparsity = round(float(n) / float(CB * KB), 3)
        self.layout = lay > 0

    def i_shape(self, N):
        return (N, self.C) if self.axis else (self.C, N)

    def o_shape(self, N):
        return (N, self.K) if self.axis else (self.K, N)

    # ---- NumPy checkers (float64 accumulation, as np.zeros defaults to) ----

    def fprop(self, I, W, gate=None):
        """matmul.py:353-375."""
        bs = self.bsize
        if self.axis:
            N = I.shape[0]
            Iv = I.reshape(N, self.CB, bs)
            O = np.zeros((N, self.KB, bs))
            for k, col in self.fprop_list:
                for c, w in col:
                    O[:, k, :] += Iv[:, c, :] @ W[w]
            return O.reshape(N, -1)
        N = I.shape[1]
        Iv = I.reshape(self.CB, bs, N)
        O = np.zeros((self.KB, bs, N))
        for k, col in self.fprop_list:
            for c, w in col:
                if gate is None:
                    O[k] += W[w].T @ Iv[c]
                elif gate[w] != 0.0:
                    O[k] += (W[w].T @ Iv[c]) * gate[w]
        return O.reshape(-1, N)

    def bprop(self, E, W, gate=None):
        """matmul.py:377-399."""
        bs = self.bsize
        if self.axis:
            N = E.shape[0]
            Ev = E.reshape(N, self.KB, bs)
            B = np.zeros((N, self.CB, bs))
            for c, row in self.bprop_list:
                for k, w in row:
                    B[:, c, :] += Ev[:, k, :] @ W[w].T
            return B.reshape(N, -1)
        N = E.shape[1]
        Ev = E.reshape(self.KB, bs, N)
        B = np.zeros((self.CB, bs, N))
        for c, row in self.bprop_list:
            for k, w in row:
                if gate is None:
                    B[c] += W[w] @ Ev[k]
                elif gate[w] != 0.0:
                    B[c] += (W[w] @ Ev[k]) * gate[w]
        return B.reshape(-1, N)

    def updat(self, I, E, gate=None, dw_gated=False):
        """matmul.py:401-419."""
        bs = self.bsize
        U = np.zeros(self.w_shape)
        if self.axis:
            Iv = I.reshape(-1, self.CB, bs)
            Ev = E.reshape(-1, self.KB, bs)
            for w, (c, k) in enumerate(self.updat_list):
                U[w] = Iv[:, c, :].T @ Ev[:, k, :]
            return U
        Iv = I.reshape(self.CB, bs, -1)
        Ev = E.reshape(self.KB, bs, -1)
        for w, (c, k) in enumerate(self.updat_list):
            if dw_gated and gate is not None:
                if gate[w] != 0.0:
                    U[w] = (Iv[c] @ Ev[k].T) * gate[w]
            else:
                U[w] = Iv[c] @ Ev[k].T
        return U

    def updat_blocks(self, I, E, block_ids):
        """matmul.py:401-419 restricted to the listed block ids (full-size checks sample the blocks: the loop body
        is the reference's `U[w] = dot(I[c], E[k].T)` line unchanged)."""
        bs = self.bsize
        U = np.zeros((len(block_ids), bs, bs))
        if self.axis:
            Iv = I.reshape(-1, self.CB, bs)
            Ev = E.reshape(-1, self.KB, bs)
            for i, w in enumerate(block_ids):
                c, k = self.updat_list[w]
                U[i] = Iv[:, c, :].astype(np.float64).T @ Ev[:, k, :].astype(np.float64)
            return U
        Iv = I.reshape(self.CB, bs, -1)
        Ev = E.reshape(self.KB, bs, -1)
        for i, w in enumerate(block_ids):
            c, k = self.updat_list[w]
            U[i] = Iv[c].astype(np.float64) @ Ev[k].astype(np.float64).T
        return U

    # ---- dense cross-check ("NumPy einsum reference of the same layout") ----

    def dense_weight(self, W):
        """Scatter the (blocks, bs, bs) tensor into a dense (C, K) matrix."""
        bs = self.bsize
        D = np.zeros((self.C, self.K), dtype=np.float64)
        for w, (c, k) in enumerate(self.updat_list):
            D[c * bs:(c + 1) * bs, k * bs:(k + 1) * bs] = W[w]
        return D

    def fprop_dense(self, I, W):
        D = self.dense_weight(W)
        return np.einsum('nc,ck->nk', I, D) if self.axis else np.einsum('ck,cn->kn', D, I)

    def bprop_dense(self, E, W):
        D = self.dense_weight(W)
        return np.einsum('nk,ck->nc', E, D) if self.axis else np.einsum('ck,kn->cn', D, E)

    def updat_dense(self, I, E):
        full = np.einsum('nc,nk->ck', I, E) if self.axis else np.einsum('cn,kn->ck', I, E)
        bs = self.bsize
        U = np.zeros(self.w_shape)
        for w, (c, k) in enumerate(self.updat_list):
            U[w] = full[c * bs:(c + 1) * bs, k * bs:(k + 1) * bs]
        return U


# ---------------------------------------------------------------------------
# Fast variant used ONLY as the timed CPU baseline (bench.py): same math as the
# checkers above, restated so NumPy/BLAS does one batched matmul per output
# block-row instead of one np.dot per block (BASELINE.md section 3).
# ---------------------------------------------------------------------------

def fprop_fast(orc, I, W):
    bs = orc.bsize
    if orc.axis:
        N = I.shape[0]
        Iv = I.reshape(N, orc.CB, bs)
        O = np.zeros((N, orc.KB, bs), dtype=np.float32)
        for k, col in orc.fprop_list:
            if col:
                cidx = [c for c, _ in col]
                widx = [w for _, w in col]
                O[:, k, :] = Iv[:, cidx, :].reshape(N, -1) @ W[widx].reshape(-1, bs)
        return O.reshape(N, -1)
    N = I.shape[1]
    Iv = I.reshape(orc.CB, bs, N)
    O = np.zeros((orc.KB, bs, N), dtype=np.float32)
    for k, col in orc.fprop_list:
        if col:
            cidx = [c for c, _ in col]
            widx = [w for _, w in col]
            O[k] = W[widx].reshape(-1, bs).T @ Iv[cidx].reshape(-1, N)
    return O.reshape(-1, N)


def bprop_fast(orc, E, W):
    bs = orc.bsize
    if orc.axis:
        N = E.shape[0]
        Ev = E.reshape(N, orc.KB, bs)
        B = np.zeros((N, orc.CB, bs), dtype=np.float32)
        for c, row in orc.bprop_list:
            if row:
                kidx = [k for k, _ in row]
                widx = [w for _, w in row]
                Wt = W[widx].transpose(0, 2, 1).reshape(-1, bs)
                B[:, c, :] = Ev[:, kidx, :].reshape(N, -1) @ Wt
        return B.reshape(N, -1)
    N = E.shape[1]
    Ev = E.reshape(orc.KB, bs, N)
    B = np.zeros((orc.CB, bs, N), dtype=np.float32)
    for c, row in orc.bprop_list:
        if row:
            kidx = [k for k, _ in row]
            widx = [w for _, w in row]
            Wc = W[widx].transpose(1, 0, 2).reshape(bs, -1)
            B[c] = Wc @ Ev[kidx].reshape(-1, N)
    return B.reshape(-1, N)


def updat_fast(orc, I, E):
    bs = orc.bsize
    cs = orc.updat_lut[:, 0]
    ks = orc.updat_lut[:, 1]
    if orc.axis:
        Iv = I.reshape(-1, orc.CB, bs).transpose(1, 2, 0)   # CB, bs, N
        Ev = E.reshape(-1, orc.KB, bs).transpose(1, 0, 2)   # KB, N, bs
        return np.matmul(Iv[cs], Ev[ks]).astype(np.float32)
    Iv = I.reshape(orc.CB, bs, -1)
    Ev = E.reshape(orc.KB, bs, -1).transpose(0, 2, 1)
    return np.matmul(Iv[cs], Ev[ks]).astype(np.float32)
