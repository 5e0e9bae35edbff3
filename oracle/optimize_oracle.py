"""Float64 NumPy restatement of the reference's optimizer ops (blocksparse/optimize.py, src/optimize_op_gpu.cu), written
from their description: one Adam step (dense and gated), the global norm and its clip scale, the parameter EMA, and the
two 16-bit moment codes of ew_op_gpu.h:332-431.

Inputs are taken as given (already rounded to their storage dtype) and every result is float64, except the codes, which
are uint16.
"""
import numpy as np

MEAN_MAX = 15.984375          # 2^3 (1 + 511/512)
VAR_MAX = 15.9921875          # 2^3 (1 + 1023/1024)
MEAN_MIN = 2.0 ** -60 * (1 + 2.0 ** -9)
VAR_MIN = 2.0 ** -60 * (1 + 2.0 ** -10)


def _encode(v, mbits, signed):
    """Round |v| to `mbits` mantissa bits, half away from zero, into a (sign,) 6-bit exponent (bias 60), mantissa code."""
    v = np.asarray(v, dtype=np.float64)
    a = np.abs(v)
    live = a > 0
    e = np.zeros(v.shape, np.int64)
    e[live] = np.floor(np.log2(a[live])).astype(np.int64)
    # log2 can land one off at exact powers of two; pin e so that 1 <= a / 2^e < 2
    lo = live & (a < np.ldexp(1.0, e))
    e[lo] -= 1
    hi = live & (a >= np.ldexp(1.0, e + 1))
    e[hi] += 1
    f = np.floor((np.where(live, a / np.ldexp(1.0, e), 1.0) - 1.0) * (1 << mbits) + 0.5).astype(np.int64)
    carry = f == (1 << mbits)
    e[carry] += 1
    f[carry] = 0
    code = ((e + 60) << mbits) | f
    if signed:
        code |= (v < 0).astype(np.int64) << 15
    return code


def mean_encode(v):
    """Signed mean code: clamp to +-MEAN_MAX (NaN -> +MEAN_MAX), |v| < MEAN_MIN -> 0, else 9 mantissa bits."""
    v = np.fmax(np.fmin(np.asarray(v, dtype=np.float64), MEAN_MAX), -MEAN_MAX)
    code = _encode(v, 9, True)
    return np.where(np.abs(v) < MEAN_MIN, 0, code).astype(np.uint16)


def var_encode(v):
    """Unsigned variance code: clamp to VAR_MAX (NaN -> VAR_MAX), v < VAR_MIN -> 0, else 10 mantissa bits, half up."""
    v = np.fmin(np.asarray(v, dtype=np.float64), VAR_MAX)
    code = _encode(np.where(v < VAR_MIN, VAR_MIN, v), 10, False)
    return np.where(v < VAR_MIN, 0, code).astype(np.uint16)


def mean_decode(c):
    c = np.asarray(c).astype(np.int64) & 0xFFFF
    sign = np.where(c & 0x8000, -1.0, 1.0)
    val = sign * np.ldexp(1.0 + (c & 511) / 512.0, ((c >> 9) & 63) - 60)
    return np.where(c == 0, 0.0, val)


def var_decode(c):
    c = np.asarray(c).astype(np.int64) & 0xFFFF
    val = np.ldexp(1.0 + (c & 1023) / 1024.0, (c >> 10) - 60)
    return np.where(c == 0, 0.0, val)


def condition(g, saturate=0.0, zero_infs=False, zero_nans=False):
    """zero_infs, then zero_nans, then the clamp to +-saturate (NaN clamps to +saturate, as fminf / fmaxf order it)."""
    g = np.array(g, dtype=np.float64)
    if zero_infs:
        g[np.isinf(g)] = 0.0
    if zero_nans:
        g[np.isnan(g)] = 0.0
    if saturate != 0.0:
        g = np.fmax(np.fmin(g, saturate), -saturate)
    return g


def lr_t(lr, beta1_power, beta2_power):
    """Bias-corrected rate of optimize.py:57."""
    return lr * np.sqrt(1.0 - beta2_power) / (1.0 - beta1_power)


def _live(shape, gate, bs):
    """Boolean mask of the elements a gated step touches (all of them without a gate)."""
    if gate is None:
        return np.ones(shape, bool)
    per = bs * bs
    return np.repeat(np.asarray(gate) != 0, per).reshape(shape)


def adam(g, p, m, v, lr, beta1, beta2, epsilon, grad_scale=1.0, clip_sigma=0.0, norm_scale=1.0, saturate=0.0,
         zero_infs=False, zero_nans=False, gate=None, bs=0):
    """One Adam step (optimize_op_gpu.cu:454-502); returns (p, m, v). With a gate, blocks of bs*bs elements whose gate is 0
    keep p, m and v, and live blocks take one step. norm_scale == 0 returns the inputs unchanged."""
    p, m, v = (np.array(a, dtype=np.float64) for a in (p, m, v))
    if norm_scale == 0:
        return p, m, v
    g = condition(g, saturate, zero_infs, zero_nans) * (grad_scale * norm_scale)
    v1 = beta2 * v + (1 - beta2) * g * g
    sigma = np.sqrt(v1)
    if clip_sigma != 0.0:
        g = np.clip(g, -clip_sigma * sigma, clip_sigma * sigma)
    m1 = beta1 * m + (1 - beta1) * g
    p1 = p - lr * m1 / (sigma + epsilon)
    live = _live(p.shape, gate, bs)
    return np.where(live, p1, p), np.where(live, m1, m), np.where(live, v1, v)


def global_norm(grads, clip_norm=1.0, grad_scale=1.0, saturate=0.0, zero_infs=False, zero_nans=False):
    """(norm, scale): norm = sqrt(sum (grad_scale * sat(filter(x)))^2); scale = clip_norm / max(norm, clip_norm), or 0 when
    the norm is not finite. No grads at all: (0, 1)."""
    total = 0.0
    with np.errstate(over="ignore", invalid="ignore"):
        for x in grads:
            y = condition(x, saturate, zero_infs, zero_nans) * grad_scale
            total += np.sum(y * y)
        norm = np.sqrt(total)
        scale = clip_norm / max(norm, clip_norm) if np.isfinite(norm) else 0.0
    return float(norm), float(scale)


def ema(e, p, decay, gate=None, bs=0):
    """ema -= (1 - decay) * (ema - p), skipping gated-off blocks."""
    e = np.array(e, dtype=np.float64)
    e1 = e - (1 - decay) * (e - np.asarray(p, dtype=np.float64))
    return np.where(_live(e.shape, gate, bs), e1, e)
