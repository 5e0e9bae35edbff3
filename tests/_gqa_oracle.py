"""Float64 statement of grouped-query attention (test infrastructure): k and v of kv_heads heads expanded to heads
heads (query head h reads kv head h // (heads // kv_heads)), then the multi-head references; dk and dv are the
expanded gradients summed over each group. tests/test_attention_gqa_abi.py pins it to
torch.nn.functional.scaled_dot_product_attention(enable_gqa=True)."""
import numpy as np

from tests._attention_grad_oracle import oracle_attention_grad
from tests._attention_oracle import oracle_attention


def expand_kv(X, heads, kv_heads):
    """(batch, ctx, kv_heads*hs) -> (batch, ctx, heads*hs), each kv head repeated for the heads // kv_heads query heads
    of its group."""
    B, C, S = X.shape
    hs = S // kv_heads
    return np.repeat(X.reshape(B, C, kv_heads, 1, hs), heads // kv_heads, axis=3).reshape(B, C, heads * hs)


def sum_groups(X, heads, kv_heads):
    """(batch, ctx, heads*hs) -> (batch, ctx, kv_heads*hs): the sum over each group's query heads."""
    B, C, S = X.shape
    hs = S // heads
    return X.reshape(B, C, kv_heads, heads // kv_heads, hs).sum(axis=3).reshape(B, C, kv_heads * hs)


def oracle_attention_gqa(orc, kv_heads, Q, K, V, scale=1.0, autoregress_at_key=None):
    return oracle_attention(orc, Q, expand_kv(K, orc.heads, kv_heads), expand_kv(V, orc.heads, kv_heads), scale,
                            autoregress_at_key)


def oracle_attention_gqa_grad(orc, kv_heads, Q, K, V, dY, scale=1.0, autoregress_at_key=None):
    dQ, dK, dV = oracle_attention_grad(orc, Q, expand_kv(K, orc.heads, kv_heads), expand_kv(V, orc.heads, kv_heads),
                                       dY, scale, autoregress_at_key)
    return dQ, sum_groups(dK, orc.heads, kv_heads), sum_groups(dV, orc.heads, kv_heads)
