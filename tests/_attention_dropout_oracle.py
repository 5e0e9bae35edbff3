"""Float64 statement of the fused attention op with dropout on its probabilities, and of its gradients, built on a
TransformerOracle's layout and mask and on the Philox4x32-10 bits of oracle/ewops_oracle.py (test infrastructure).

The keep bit of probability (batch b, head h, layout block blk, query row i of the block, key column j) is element
e = (((b * heads + h) * blocks + blk) * bs + i) * bs + j of the row-major (batch, heads, blocks, bs, bs) probability
tensor, drawn as ewops.dropout draws it: word e % 4 of Philox4x32-10(counter = (e / 4, call), key = seed) below
floor(keep_prob * 2^32). tests/test_attention_dropout_oracle.py pins these functions to the float64 chain
nt -> masked_softmax -> ewops_oracle.dropout_apply -> nn and its backward, and to central differences; with
keep_prob = 1 they equal tests/_attention_oracle.py and tests/_attention_grad_oracle.py exactly."""
import numpy as np

from oracle.ewops_oracle import keep_threshold, philox4x32_10
from tests._attention_grad_oracle import _heads, _merge, attention_probs


def keep_bits_at(seed, call, e, keep_prob):
    """bool of e's shape: element e (int64 array, any values, 2^32 and past included) of the mask drawn at
    (seed, call)."""
    e = np.asarray(e, np.int64).astype(np.uint64)
    seed, call = int(seed) % 2 ** 64, int(call) % 2 ** 64
    g = e >> np.uint64(2)
    lo = np.uint64(0xFFFFFFFF)
    ctr = np.stack([g & lo, g >> np.uint64(32), np.full_like(g, call & 0xFFFFFFFF), np.full_like(g, call >> 32)], -1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint32), g.shape + (2,))
    words = philox4x32_10(ctr.astype(np.uint32), key)
    w = np.take_along_axis(words, (e & np.uint64(3)).astype(np.int64)[..., None], axis=-1)[..., 0]
    return w.astype(np.uint64) < np.uint64(keep_threshold(keep_prob))


def attention_keep(orc, batch, seed, call, keep_prob, batches=None, rows=None):
    """Z bool (len(batches), heads, len(rows), ctx_k): the keep bit of every probability of the dense attention matrix,
    False outside the layout. batches / rows (default: all) select batch indices and dense query rows, so that a large
    problem can be checked on a sample."""
    bs, H = orc.blk_size, orc.heads
    batches = np.arange(batch) if batches is None else np.asarray(batches)
    rows = np.arange(orc.ctx_blks_q * bs) if rows is None else np.asarray(rows)
    Z = np.zeros((len(batches), H, len(rows), orc.ctx_blks_k * bs), bool)
    for h in range(H):
        for blk, (qb, kb) in enumerate(orc.nt_list[orc._hl(h)]):
            sel = np.nonzero(rows // bs == qb)[0]
            if not len(sel):
                continue
            i = (rows[sel] % bs).astype(np.int64)
            j = np.arange(bs, dtype=np.int64)
            base = ((batches.astype(np.int64) * H + h) * orc.blocks + blk) * bs
            e = ((base[:, None, None] + i[None, :, None]) * bs + j[None, None, :])
            Z[:, h, sel, kb * bs:(kb + 1) * bs] = keep_bits_at(seed, call, e, keep_prob)
    return Z


def oracle_attention_dropout(orc, Q, K, V, Z, keep_prob, scale=1.0, autoregress_at_key=None):
    """O (batch, ctx_q, heads*hs) in float64 of attention with dropout: per head, (P o Z / keep_prob) V with P the
    probabilities of oracle_attention (uniform on a fully masked row, zero on a row with no layout block), formed as
    oracle_attention forms them."""
    bs = orc.blk_size
    B, ctxq, S = Q.shape
    hs = S // orc.heads
    Qh = Q.reshape(B, ctxq, orc.heads, hs).transpose(0, 2, 1, 3).astype(np.float64)
    Kh = K.reshape(B, -1, orc.heads, hs).transpose(0, 2, 1, 3).astype(np.float64)
    Vh = V.reshape(B, -1, orc.heads, hs).transpose(0, 2, 1, 3).astype(np.float64)
    neg = -float(np.finfo(np.float32).max)
    out = np.zeros_like(Qh)
    for h in range(orc.heads):
        hl = orc._hl(h)
        inlay = np.zeros((orc.ctx_blks_q * bs, orc.ctx_blks_k * bs), dtype=bool)
        vis = np.zeros_like(inlay)
        for b, (q, k) in enumerate(orc.nt_list[hl]):
            blk = (np.ones((bs, bs), bool) if orc.softmax_mask_np is None
                   else orc._mask_bits(hl, b, k, autoregress_at_key))
            inlay[q * bs:(q + 1) * bs, k * bs:(k + 1) * bs] = True
            vis[q * bs:(q + 1) * bs, k * bs:(k + 1) * bs] = blk
        rows = inlay.any(axis=1)
        s = (Qh[:, h] @ Kh[:, h].transpose(0, 2, 1)) * scale
        s = np.where(vis, s, np.where(inlay, neg, -np.inf))[:, rows]
        e = np.exp(s - s.max(axis=-1, keepdims=True))
        out[:, h, rows] = (np.where(Z[:, h][:, rows], e / e.sum(axis=-1, keepdims=True), 0.0) / keep_prob) @ Vh[:, h]
    return out.transpose(0, 2, 1, 3).reshape(B, ctxq, S)


def oracle_attention_dropout_grad(orc, Q, K, V, dY, Z, keep_prob, scale=1.0, autoregress_at_key=None):
    """(dQ, dK, dV) in float64 of oracle_attention_dropout for the output gradient dY: dV = (P o Z / keep_prob)^T dY,
    dP = (dY V^T) o Z / keep_prob, dS = scale * P * (dP - rowsum(dP * P)), dQ = dS K, dK = dS^T Q, as the chain's
    backward through ewops.dropout defines them (rowsum(dP * P) = dY . O)."""
    Qh, Kh, Vh, dYh = (_heads(X, orc.heads) for X in (Q, K, V, dY))
    P = attention_probs(orc, Q, K, scale, autoregress_at_key)
    Pd = np.where(Z, P, 0.0) / keep_prob
    dP = np.where(Z, dYh @ Vh.transpose(0, 1, 3, 2), 0.0) / keep_prob
    dS = scale * P * (dP - (dP * P).sum(axis=-1, keepdims=True))
    dQ = dS @ Kh
    dK = dS.transpose(0, 1, 3, 2) @ Qh
    dV = Pd.transpose(0, 1, 3, 2) @ dYh
    return _merge(dQ), _merge(dK), _merge(dV)
