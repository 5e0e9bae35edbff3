"""Float64 statement of the gradients of the fused attention op, built on a TransformerOracle's layout and mask (test
infrastructure).

tests/test_attention_grad_oracle.py pins it to the oracle's chain backward (nt, masked_softmax_grad, nn and tn, the
methods the reference fixtures pin) and to central differences; the GPU tests of the fused backward compare against
it."""
import numpy as np


def _dense_probs(orc, h, Qh, Kh, scale, ak):
    """(P, inlay rows) of head h: P (batch, ctx_q, ctx_k) float64 softmax as oracle_attention forms it, zero outside the
    layout and on rows with no layout block."""
    bs = orc.blk_size
    hl = orc._hl(h)
    inlay = np.zeros((orc.ctx_blks_q * bs, orc.ctx_blks_k * bs), dtype=bool)
    vis = np.zeros_like(inlay)
    for b, (q, k) in enumerate(orc.nt_list[hl]):
        blk = np.ones((bs, bs), bool) if orc.softmax_mask_np is None else orc._mask_bits(hl, b, k, ak)
        inlay[q * bs:(q + 1) * bs, k * bs:(k + 1) * bs] = True
        vis[q * bs:(q + 1) * bs, k * bs:(k + 1) * bs] = blk
    rows = inlay.any(axis=1)
    neg = -float(np.finfo(np.float32).max)
    s = (Qh @ Kh.transpose(0, 2, 1)) * scale
    s = np.where(vis, s, np.where(inlay, neg, -np.inf))
    P = np.zeros_like(s)
    e = np.exp(s[:, rows] - s[:, rows].max(axis=-1, keepdims=True))
    P[:, rows] = e / e.sum(axis=-1, keepdims=True)
    return P


def _heads(X, heads):
    B, ctx, S = X.shape
    return X.reshape(B, ctx, heads, S // heads).transpose(0, 2, 1, 3).astype(np.float64)


def _merge(Xh):
    B, H, ctx, hs = Xh.shape
    return Xh.transpose(0, 2, 1, 3).reshape(B, ctx, H * hs)


def attention_probs(orc, Q, K, scale=1.0, autoregress_at_key=None):
    """P (batch, heads, ctx_q, ctx_k) in float64: the dense probabilities of the fused attention op."""
    Qh, Kh = _heads(Q, orc.heads), _heads(K, orc.heads)
    return np.stack([_dense_probs(orc, h, Qh[:, h], Kh[:, h], scale, autoregress_at_key) for h in range(orc.heads)], axis=1)


def oracle_attention_grad(orc, Q, K, V, dY, scale=1.0, autoregress_at_key=None):
    """(dQ, dK, dV) in float64 of O = oracle_attention(orc, Q, K, V, scale, autoregress_at_key) for the output gradient
    dY, as the chain's backward defines them: dV = P^T dY; dP = dY V^T; dS = scale * P * (dP - rowsum(dP * P));
    dQ = dS K; dK = dS^T Q. Entries outside the layout have P = 0 and contribute nothing. A row whose keys are all masked
    has uniform P over its layout keys, and its dS reaches dQ and dK as in the chain, although O does not depend on
    them there."""
    Qh, Kh, Vh, dYh = (_heads(X, orc.heads) for X in (Q, K, V, dY))
    P = attention_probs(orc, Q, K, scale, autoregress_at_key)
    dP = dYh @ Vh.transpose(0, 1, 3, 2)
    dS = scale * P * (dP - (dP * P).sum(axis=-1, keepdims=True))
    dQ = dS @ Kh
    dK = dS.transpose(0, 1, 3, 2) @ Qh
    dV = P.transpose(0, 1, 3, 2) @ dYh
    return _merge(dQ), _merge(dK), _merge(dV)
