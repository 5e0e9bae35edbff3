"""Float64 NumPy restatement of bias_relu, dropout and embedding_lookup with their gradients (reference
blocksparse/ewops.py:207-242, 307-350; blocksparse/embed.py; src/ew_op_gpu.cu:687-811, 918-1230;
src/embedding_op_gpu.cu), with Philox4x32-10 and the dropout mask format.

The RNG is not the reference's (its Tausworthe state is sized for 80 V100 SMs, so its stream depends on the grid):
element e is kept iff word e % 4 of Philox4x32-10(counter = (e / 4 as 64 bits, call as 64 bits), key = seed) is below
floor(keep_prob * 2^32).
"""
import numpy as np

GELU_A = 1.702            # fast_gelu = z * sigmoid(1.702 z), the reference's ew_swish(z, 1.702) (ew_op_gpu.cu:933)

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: uint32 (..., 4), key: uint32 (..., 2) -> uint32 (..., 4) (Random123's philox4x32 with 10 rounds)."""
    c = [np.asarray(ctr, np.uint32)[..., i].astype(np.uint64) for i in range(4)]
    k0 = np.asarray(key, np.uint32)[..., 0].copy()
    k1 = np.asarray(key, np.uint32)[..., 1].copy()
    with np.errstate(over="ignore"):
        for r in range(10):
            if r:
                k0 = k0 + _W0
                k1 = k1 + _W1
            p0, p1 = _M0 * c[0], _M1 * c[2]
            hi0, lo0 = p0 >> np.uint64(32), p0 & _LO
            hi1, lo1 = p1 >> np.uint64(32), p1 & _LO
            c = [hi1 ^ c[1] ^ k0.astype(np.uint64), lo1, hi0 ^ c[3] ^ k1.astype(np.uint64), lo0]
    return np.stack([x.astype(np.uint32) for x in c], axis=-1)


def _u64(v):
    return int(v) % 2 ** 64


def keep_threshold(keep_prob):
    return int(np.floor(float(keep_prob) * 2.0 ** 32))


def dropout_bits(seed, call, M, keep_prob):
    """bool [M]: element e kept."""
    seed, call = _u64(seed), _u64(call)
    g = np.arange((M + 3) // 4, dtype=np.uint64)
    ctr = np.stack([g & _LO, g >> np.uint64(32), np.full_like(g, call & 0xFFFFFFFF), np.full_like(g, call >> 32)], -1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint32), (len(g), 2))
    u = philox4x32_10(ctr.astype(np.uint32), key).reshape(-1)[:M]
    return u.astype(np.uint64) < np.uint64(keep_threshold(keep_prob))


def pack_mask(bits):
    """bool [M] -> int32 [ceil(M / 32)]: bit e % 32 of word e / 32 (reference ew_op_gpu.cu:687-721)."""
    M = len(bits)
    padded = np.zeros(((M + 31) // 32) * 32, np.uint64)
    padded[:M] = bits
    words = (padded.reshape(-1, 32) << np.arange(32, dtype=np.uint64)).sum(axis=1)
    return words.astype(np.uint32).view(np.int32)


def unpack_mask(words, M):
    w = np.asarray(words).view(np.uint32).astype(np.uint64)
    return ((w[:, None] >> np.arange(32, dtype=np.uint64)) & np.uint64(1)).reshape(-1)[:M].astype(bool)


def dropout_mask(seed, call, M, keep_prob):
    return pack_mask(dropout_bits(seed, call, M, keep_prob))


def broadcast_keep(words, x_shape, mask_shape=None):
    """bool x_shape: the mask bit of every element of x, the mask (mask_shape, default x_shape) broadcast over x
    (reference ew_op_gpu.cu:735-811)."""
    ms = tuple(x_shape) if mask_shape is None or len(mask_shape) == 0 else tuple(mask_shape)
    bits = unpack_mask(words, int(np.prod(ms, dtype=np.int64))).reshape(ms)
    return np.broadcast_to(bits, tuple(x_shape))


def dropout_apply(x, words, keep_prob, mask_shape=None):
    """float64: x / keep_prob where kept, 0 elsewhere (the device rounds fp32(x) * fp32(1 / keep_prob) once)."""
    keep = broadcast_keep(words, np.shape(x), mask_shape)
    return np.where(keep, np.asarray(x, np.float64) / keep_prob, 0.0)


def _move(x, axis):
    """x with the feature axis last (axis 0 of a (K, N) view moves to the end)."""
    x = np.asarray(x, np.float64)
    return np.moveaxis(x, 0, -1) if axis == 0 else x


def bias_relu(x, b, axis=-1, relu=False, fast_gelu=False):
    """act(x + b) along axis 0 or the last one (reference ewops.py:307-331)."""
    ax = 0 if axis == 0 and np.ndim(x) > 1 else -1
    z = _move(x, ax) + np.asarray(b, np.float64).reshape(-1)
    if relu:
        z = np.maximum(z, 0.0)
    elif fast_gelu:
        z = z / (1.0 + np.exp(-GELU_A * z))
    return np.moveaxis(z, -1, 0) if ax == 0 else z


def bias_relu_grad(dy, x, b, axis=-1, relu=False, fast_gelu=False):
    """(dx, db) (reference ewops.py:335-350, ew_op_gpu.cu:1039-1230): dx = dy * act'(x + b), db = sum of dx over every
    axis but the feature axis."""
    ax = 0 if axis == 0 and np.ndim(x) > 1 else -1
    z = _move(x, ax) + np.asarray(b, np.float64).reshape(-1)
    d = _move(dy, ax)
    if relu:
        dx = d * (z > 0)
    elif fast_gelu:
        s = 1.0 / (1.0 + np.exp(-GELU_A * z))
        dx = d * (s + GELU_A * z * s * (1.0 - s))
    else:
        dx = d
    db = dx.reshape(-1, dx.shape[-1]).sum(axis=0)
    return (np.moveaxis(dx, -1, 0) if ax == 0 else dx), db


def embedding_lookup(emb, idx):
    """emb[idx] with zero rows for indices outside [0, C) (reference embedding_op_gpu.cu:20, 40)."""
    emb = np.asarray(emb, np.float64)
    idx = np.asarray(idx).astype(np.int64)
    ok = (idx >= 0) & (idx < emb.shape[0])
    y = emb[np.where(ok, idx, 0)]
    y[~ok] = 0.0
    return y


def embedding_grad(dy, idx, C):
    """dw (C, K): sum of dy rows per index; out-of-range indices add nothing."""
    dy = np.asarray(dy, np.float64)
    K = dy.shape[-1]
    idx = np.asarray(idx).astype(np.int64).reshape(-1)
    d = dy.reshape(-1, K)
    ok = (idx >= 0) & (idx < C)
    dw = np.zeros((C, K))
    np.add.at(dw, idx[ok], d[ok])
    return dw
