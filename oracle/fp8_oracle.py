"""NumPy restatement of the fp8 quantisation of include/bsmm_b200.h (bsmm_fp8_quantize / bsmm_fp8_weights) and of the
products bsmm_xprop_fp8 forms from it (TEST INFRASTRUCTURE ONLY; the product package never imports it).

  amax(x)                    max |x| in fp32: NaN if any element is NaN, else +inf if any is infinite, 0 when empty
  scales(amax, fmt)          (s, scale_inv) as fp32: FP8_MAX / amax and amax / FP8_MAX, 1 for amax = 0, scale_inv NaN
                             for a non-finite amax
  round_fp8(v, fmt)          fp32 values -> fp8 codes (uint8): round to nearest even, subnormals kept, magnitudes past
                             FP8_MAX (infinities included) saturated, the sign of zero kept, NaN -> 0x7f (the
                             hardware's canonical NaN; torch's cast keeps a NaN's sign bit instead)
  decode(codes, fmt)         fp8 codes -> float64
  quantize(x, fmt)           (codes, amax, scale_inv) of a whole tensor
  quantize_weights(w, fmt)   (wq, wq_t, amax, scale_inv) of (blocks, bs, bs) weights, wq_t each block transposed

fmt is "e4m3" (torch.float8_e4m3fn: 4 exponent bits, bias 7, 3 mantissa bits, largest finite 448, no infinities) or
"e5m2" (torch.float8_e5m2: 5 exponent bits, bias 15, 2 mantissa bits, largest finite 57344).
"""
import numpy as np

FORMATS = {"e4m3": (4, 3, 7, 448.0), "e5m2": (5, 2, 15, 57344.0)}     # exponent bits, mantissa bits, bias, max
FP8_MAX = {k: v[3] for k, v in FORMATS.items()}


def amax(x):
    a = np.abs(np.asarray(x, dtype=np.float32)).ravel()
    if a.size == 0:
        return np.float32(0)
    if np.isnan(a).any():
        return np.float32(np.nan)
    return np.float32(a.max())


def scales(am, fmt):
    """(s, scale_inv) in fp32, each one IEEE fp32 division (numpy float32 division rounds to nearest even)."""
    am, mx = np.float32(am), np.float32(FP8_MAX[fmt])
    if am == 0:
        return np.float32(1), np.float32(1)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        s = mx / am
    return s, (am / mx if np.isfinite(am) else np.float32(np.nan))


def round_fp8(v, fmt):
    """fp32 values -> uint8 fp8 codes, cvt.rn.satfinite semantics."""
    ebits, mbits, bias, mx = FORMATS[fmt]
    v = np.asarray(v, dtype=np.float32)
    sign = np.signbit(v).astype(np.uint8) << 7
    a = np.abs(v.astype(np.float64))
    nan = np.isnan(a)
    a = np.where(nan, 0.0, np.minimum(a, mx))                   # satfinite: anything past max (inf too) is max
    emin = 1 - bias                                             # exponent of the smallest normal
    _, e2 = np.frexp(a)                                         # a = m 2^e2, m in [0.5, 1)
    e = np.maximum(e2 - 1, emin)                                # floor(log2 a), subnormals share emin
    q = np.ldexp(1.0, e - mbits)                                # spacing of representable values around a
    r = np.rint(a / q) * q                                      # round half to even (a / q is exact)
    r = np.minimum(r, mx)
    _, re2 = np.frexp(r)
    re = re2 - 1
    normal = (r > 0) & (re >= emin)
    expf = np.where(normal, re + bias, 0)
    mant = np.where(normal, (np.ldexp(r, -re) - 1.0) * (1 << mbits), np.ldexp(r, mbits - emin))   # subnormal: r / 2^(emin - mbits)
    code = sign | (expf.astype(np.uint8) << mbits) | np.rint(mant).astype(np.uint8)
    return np.where(nan, np.uint8(0x7F), code).astype(np.uint8)


def decode(codes, fmt):
    ebits, mbits, bias, _ = FORMATS[fmt]
    c = np.asarray(codes, dtype=np.uint8).astype(np.int64)
    sign = np.where(c & 0x80, -1.0, 1.0)
    expf = (c >> mbits) & ((1 << ebits) - 1)
    mant = c & ((1 << mbits) - 1)
    val = np.where(expf == 0, np.ldexp(mant.astype(np.float64), 1 - bias - mbits),
                   np.ldexp(1.0 + mant / float(1 << mbits), expf - bias))
    if fmt == "e4m3":
        special = (c & 0x7F) == 0x7F                            # e4m3fn: only S.1111.111 is NaN
        val = np.where(special, np.nan, val)
    else:
        val = np.where(expf == 31, np.where(mant == 0, np.inf, np.nan), val)
    return sign * val


def quantize(x, fmt):
    x = np.asarray(x, dtype=np.float32)
    am = amax(x)
    s, scale_inv = scales(am, fmt)
    with np.errstate(invalid="ignore", over="ignore"):
        v = x * s                                               # fp32 product, rounded to nearest even
    return round_fp8(v, fmt), am, scale_inv


def quantize_weights(w, fmt):
    wq, am, scale_inv = quantize(w, fmt)
    return wq, np.ascontiguousarray(wq.transpose(0, 2, 1)), am, scale_inv
