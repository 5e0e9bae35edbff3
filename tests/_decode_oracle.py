"""Float64 statement of BlocksparseTransformer.attention_decode (test infrastructure).

Row r = positions[b] + i of entry b is row r of attention over the cache, restricted to the valid keys (cache rows
< L_b = min(positions[b] + n, ctx_k)): per head, the keys of the row's LUT entries score scale * q.k, masked ones
-FLT_MAX, invalid ones -inf; softmax over them, times V. No valid key (or an empty LUT row) gives 0, a bad position NaN.
tests/test_attention_decode_abi.py pins it to tests._attention_oracle.oracle_attention where the two coincide."""
import numpy as np

NEG = -float(np.finfo(np.float32).max)


def oracle_rows(orc):
    """(rows_of, visible) of a TransformerOracle: rows_of(h, qb) lists the (block id, key block) entries of query block
    qb in head h; visible(h, bid, kb, ak) is the bool[bs, bs] mask of block bid (None: every key visible)."""
    def rows_of(h, qb):
        return orc.nn_list[orc._hl(h)][qb]

    def visible(h, bid, kb, ak):
        if orc.softmax_mask_np is None:
            return None
        return orc._mask_bits(orc._hl(h), bid, kb, ak)
    return rows_of, visible


def oracle_decode(rows_of, visible, bs, heads, ctx_q, Q, K, V, positions, scale=1.0, autoregress_at_key=None,
                  rows=None):
    """Returns (out, A, qk, nent) as float64 arrays of Q's shape (batch, n, heads*hs): the decode result, the same
    with |V| (the weight of the probability errors), the largest |q|.|k| over each row's valid keys, and the LUT entries
    of each row. rows: optional iterable of (b, i) to compute (the others stay 0)."""
    B, n, S = Q.shape
    hs = S // heads
    ctx_k = K.shape[1]
    out, A, qk, nent = (np.zeros((B, n, S)) for _ in range(4))
    todo = rows if rows is not None else [(b, i) for b in range(B) for i in range(n)]
    for b, i in todo:
        pos = int(positions[b])
        if pos < 0 or pos + n > ctx_q:
            out[b, i] = np.nan
            continue
        r = pos + i
        qb, rr = r // bs, r % bs
        L = min(pos + n, ctx_k)
        for h in range(heads):
            cols = slice(h * hs, (h + 1) * hs)
            ents = rows_of(h, qb)
            nent[b, i, cols] = len(ents)
            if not ents:
                continue
            keys = np.concatenate([np.arange(kb * bs, (kb + 1) * bs) for _, kb in ents])
            vis = np.concatenate([np.ones(bs, bool) if visible(h, bid, kb, autoregress_at_key) is None
                                  else visible(h, bid, kb, autoregress_at_key)[rr] for bid, kb in ents])
            valid = keys < L
            if not valid.any():
                continue
            keys, vis = keys[valid], vis[valid]
            q = np.asarray(Q[b, i, cols], np.float64)
            k = np.asarray(K[b, keys, cols], np.float64)
            v = np.asarray(V[b, keys, cols], np.float64)
            s = np.where(vis, (k @ q) * scale, NEG)
            e = np.exp(s - s.max())
            p = e / e.sum()
            out[b, i, cols] = p @ v
            A[b, i, cols] = p @ np.abs(v)
            qk[b, i, cols] = float((np.abs(k) @ np.abs(q)).max())
    return out, A, qk, nent
