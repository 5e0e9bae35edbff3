"""Float64 statement of the fused attention op, built on a TransformerOracle's layout and mask (test infrastructure).

tests/test_attention_oracle.py pins it to the oracle's three-op chain nn(masked_softmax(nt(Q, K), ...), V), whose
methods the reference fixtures pin in turn; the GPU tests of BlocksparseTransformer.attention compare against it."""
import numpy as np


def oracle_attention(orc, Q, K, V, scale=1.0, autoregress_at_key=None):
    """nn(masked_softmax(nt(Q, K), scale, autoregress_at_key), V) of the oracle `orc` as one dense computation in
    float64. Per head, keys outside the layout score -inf and masked keys inside it -FLT_MAX, so a query row whose keys
    are all masked gets uniform weights over its layout keys (the reference's behaviour), and a query row with no
    layout block gives 0."""
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
        out[:, h, rows] = (e / e.sum(axis=-1, keepdims=True)) @ Vh[:, h]
    return out.transpose(0, 2, 1, 3).reshape(B, ctxq, S)
