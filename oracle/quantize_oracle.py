"""NumPy restatement of the quantize module: the reference kernel's rounding on uint32 bit patterns, its exponent update,
its statistics schedule and its statistics in float64, and the log row formats.

Rounding of one fp32 value x (bit pattern b, exponent field E, significand M = 2^23 + mantissa):
  1. fp32 subnormals and zeros flush to a zero of their sign (the ftz of the add);
  2. add w * 2^(E - 150 - 32 - fbits) to |x|, rounding toward zero to fp32 (w = 2^31 for round-half-away, a Philox word
     converted to fp32 for stochastic rounding), and clear the mantissa bits below fbits; this is exact integer
     arithmetic on M * 2^(9 + fbits) + w;
  3. clamp to +-max_float; below min_float give +0;
  4. subtract exp_norm from the bits, multiply by 2^-23 rounding to nearest in fp32's subnormals, multiply by 2^23
     (toward zero), add exp_norm back (all mod 2^32, NaN intermediates canonical as on the GPU).
NaN inputs give NaN (0x7fffffff)."""
import numpy as np

from oracle.ewops_oracle import philox4x32_10

NAN_BITS = 0x7FFFFFFF
FREQ2 = 4


def top_exponent(ebits):
    return 254 if ebits == 8 else (1 << ebits) - 1


def biased(e, ebits):
    """The record value e as the kernels read it: biased, at least the format's top exponent, at most 254."""
    return int(min(max(int(e) + 127, top_exponent(ebits)), 254))


def fmt(e, ebits, fbits, denorm):
    """dict of the format at record value e: max_float, min_float, ftz_float bit patterns and exp_norm (uint32)."""
    em = biased(e, ebits)
    exp_min = max(em - top_exponent(ebits) + 1 - (fbits if denorm else 0), 2)
    mask = (0xFFFFFFFF << (23 - fbits)) & 0xFFFFFFFF
    return dict(em=em, exp_min=exp_min, mask=mask, max_float=((em << 23) | 0x7FFFFF) & mask, min_float=exp_min << 23,
                ftz_float=((exp_min - 1) << 23) | 0x400000,
                exp_norm=((exp_min - 1 - (0 if denorm else fbits)) << 23) & 0xFFFFFFFF)


def _f(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def _b(vals):
    return np.asarray(vals, np.float32).view(np.uint32)


def _canon(vals):
    v = np.asarray(vals, np.float32).copy()
    b = v.view(np.uint32)
    b[np.isnan(v)] = NAN_BITS
    return v


def quantize_bits(xbits, e, ebits, fbits, denorm, words=None):
    """uint32 array of quantized fp32 bit patterns. words: uint32 random words per element (stochastic) or None."""
    xb = np.asarray(xbits, np.uint32).reshape(-1).astype(np.uint64)
    f = fmt(e, ebits, fbits, denorm)
    sign = xb & np.uint64(0x80000000)
    E = (xb >> np.uint64(23)) & np.uint64(0xFF)
    mant = xb & np.uint64(0x7FFFFF)
    nan = (E == 255) & (mant != 0)
    inf = (E == 255) & (mant == 0)
    zero = E == 0                                          # zeros and fp32 subnormals, flushed
    if words is None:
        w = np.full(xb.shape, 2 ** 31, np.uint64)
    else:
        w = np.asarray(words, np.uint32).reshape(-1).astype(np.float32).astype(np.uint64)   # RN to fp32, then exact
    sh = np.uint64(9 + fbits)
    S = ((mant | np.uint64(1 << 23)) << sh) + w
    carry = S >= (np.uint64(1) << (np.uint64(24) + sh))
    Mn = np.where(carry, S >> (sh + np.uint64(1)), S >> sh)
    En = E + carry.astype(np.uint64)
    r = (En << np.uint64(23)) | (Mn & np.uint64(0x7FFFFF))
    r = np.where(En >= 255, np.uint64(0x7F7FFFFF), r)      # rounding toward zero never overflows to inf
    r = r & np.uint64(f["mask"])
    r = np.where(zero, np.uint64(0), r)
    r = np.where(inf, np.uint64(0x7F800000), r)
    r = (r | sign).astype(np.uint32)
    # inf times a zero word is NaN (canonical, unsigned) before the mask
    r = np.where(inf & (w == 0), np.uint32(NAN_BITS & f["mask"]), r).astype(np.uint32)
    # clamp as fmaxf / fminf do (a NaN operand gives the other one), flush, subnormal range
    v = _f(r)
    mx = _f(np.uint32(f["max_float"]))
    v = np.fmin(np.fmax(v, -mx), mx)
    small = np.abs(v) < _f(np.uint32(f["min_float"]))
    en = np.uint32(f["exp_norm"])
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        s = _f((_b(v) - en).astype(np.uint32))
        s = _canon(s * np.float32(2.0 ** -23))
        s2 = _canon(s * np.float32(2.0 ** 23))
    # the second product is exact except where s is inf / NaN; both are kept as the GPU gives them
    out = (_b(s2) + en).astype(np.uint32)
    out = np.where(small, np.uint32(0), out)
    out = np.where(nan, np.uint32(NAN_BITS), out)
    return out.astype(np.uint32)


def quantize(x, e, ebits, fbits, denorm, words=None):
    """fp32 array of x (fp32) quantized."""
    x = np.ascontiguousarray(x, np.float32)
    return quantize_bits(x.view(np.uint32), e, ebits, fbits, denorm, words).view(np.float32).reshape(x.shape)


def quantize_bf16_bits(xbits16, e, ebits, fbits, denorm, words=None):
    """uint16 bit patterns of bf16 x quantized (the fp32 result's top half)."""
    xb = np.asarray(xbits16, np.uint16).astype(np.uint32) << 16
    return (quantize_bits(xb, e, ebits, fbits, denorm, words) >> 16).astype(np.uint16)


def philox_words(seed, call, n):
    """uint32 [n]: element e's word e % 4 of Philox4x32-10 at key seed, counter (e / 4, call)."""
    seed, call = int(seed) % 2 ** 64, int(call) % 2 ** 64
    g = np.arange((n + 3) // 4, dtype=np.uint64)
    lo = np.uint64(0xFFFFFFFF)
    ctr = np.stack([g & lo, g >> np.uint64(32), np.full_like(g, call & 0xFFFFFFFF), np.full_like(g, call >> 32)], -1)
    key = np.broadcast_to(np.array([seed & 0xFFFFFFFF, seed >> 32], np.uint32), (len(g), 2))
    return philox4x32_10(ctr.astype(np.uint32), key).reshape(-1)[:n]


def stats(x, sat_val, ftz_val, half=False):
    """(mean |x|, stdv, sat %, ftz %, max |x|) as fp32, from float64 sums: NaN counts as inf, fp16 clamps to 65504."""
    v = np.asarray(x, np.float32).reshape(-1)
    v = np.where(np.isnan(v), np.float32(np.inf), v)
    if half:
        v = np.clip(v, np.float32(-65504), np.float32(65504))
    a = np.abs(v).astype(np.float64)
    n = float(v.size)
    with np.errstate(invalid="ignore", over="ignore"):
        mean = a.sum() / n
        var = (a * a).sum() / n - mean * mean
        var = 0.0 if not var > 0.0 else var
    sat = np.count_nonzero(np.abs(v) >= np.float32(sat_val))
    ftz = np.count_nonzero((v != 0) & (np.abs(v) < np.float32(ftz_val)))
    return (np.float32(mean), np.float32(np.sqrt(var)), np.float32(100.0 * sat / n), np.float32(100.0 * ftz / n),
            np.float32(np.abs(v).max() if v.size else 0.0))


def quant_stats(x, e, ebits, fbits, denorm, half=False):
    """Statistics in quantize mode: thresholds max_float and the flush threshold of the format at record e."""
    f = fmt(e, ebits, fbits, denorm)
    return stats(x, _f(np.uint32(f["max_float"])), _f(np.uint32(f["ftz_float"])), half)


def fexp(v):
    return int(np.array([v], np.float32).view(np.int32)[0] >> 23) - 127


def next_exponent(st, ebits, mode, bias_pad, stdv_mul):
    """The record value after a statistics call: the exponent of max |x| (mode 0) or of mean + stdv * stdv_mul in fp32
    (mode 1), plus bias_pad, clamped to the format."""
    mean, stdv, _, _, mx = st
    m = np.float32(mean + np.float32(stdv * np.float32(stdv_mul))) if mode else np.float32(mx)
    return biased(fexp(m) + int(bias_pad), ebits) - 127


class Schedule(object):
    """The reference QuantizeOp's statistics schedule: count from 1, pow2 from 1, pow2_count from 0, freq2 = 4."""

    def __init__(self, freq):
        self.freq, self.count, self.pow2, self.pow2_count = freq, 1, 1, 0

    def step(self):
        """True when this call computes statistics."""
        hit = bool(self.freq) and self.count % self.pow2 == 0
        if hit and 2 * self.pow2 <= self.freq:
            if self.pow2_count == FREQ2:
                self.pow2 *= 2
                self.pow2_count = 0
            self.pow2_count += 1
        self.count += 1
        return hit


def log_steps(freq):
    """The steps log_stats logs below freq: the powers of two below it."""
    p = int(np.log2(freq)) if freq else 0
    return [1 << i for i in range(p)]


def quant_log_row(st, e_new, ebits, fbits, denorm, lo, hi, count, name):
    """A quantize log row: %.3f percentages, then exponents of max_float / min_float of the updated format, of max, mean,
    stdv, mean + 5 stdv, max_stat_lo / hi, then the count and the name."""
    mean, stdv, sat, ftz, mx = (np.float32(v) for v in st)
    f = fmt(e_new, ebits, fbits, denorm)
    cols = ["%.3f" % sat, "%.3f" % ftz] + ["%3d" % c for c in (
        f["em"] - 127, f["exp_min"] - 127, fexp(mx), fexp(mean), fexp(stdv), fexp(mean + stdv * np.float32(5)),
        fexp(lo), fexp(hi))] + ["%d" % count, name]
    return "\t".join(cols) + "\n"


def stat_log_row(st, lo, hi, step, name):
    mean, stdv, sat, ftz, mx = (np.float32(v) for v in st)
    cols = ["%.6f" % sat, "%.6f" % ftz] + ["%3d" % c for c in (
        fexp(mx), fexp(mean), fexp(stdv), fexp(mean + stdv * np.float32(5)), fexp(lo), fexp(hi))] + ["%d" % step, name]
    return "\t".join(cols) + "\n"


def run(xs, spec, e0=None, seed=None, call0=0, half=False):
    """Replays quantize() over the calls xs (fp32 arrays) with one state: returns [(output fp32, record after the call,
    statistics or None)]. spec: dict with ebits, fbits, denorm, stoch, freq, mode, bias_pad, stdv_mul, emax."""
    e = spec["emax"] if e0 is None else e0
    sch = Schedule(spec["freq"])
    out, call = [], call0
    for x in xs:
        st = None
        if sch.step():
            st = quant_stats(x, e, spec["ebits"], spec["fbits"], spec["denorm"], half)
            e = next_exponent(st, spec["ebits"], spec["mode"], spec["bias_pad"], spec["stdv_mul"])
        words = None
        if spec["stoch"]:
            words = philox_words(seed, call, np.asarray(x).size)
            call += 1
        out.append((quantize(x, e, spec["ebits"], spec["fbits"], spec["denorm"], words), e, st))
    return out
