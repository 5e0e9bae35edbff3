"""The reference's blocksparse/quantize.py on torch tensors: emulation of narrow float formats in training.

  QuantizeSpec(ebits, fbits, emax, stochastic, denorm, frequency, mode, bias_pad, stdv_mul, logfile, copy)
  quantize(x, qspec, b_qspec=None, name=None)      y = x rounded to qspec; the gradient is dy rounded to b_qspec
  log_stats(x, step, sat_val, ftz_val, freq, bfreq, logfile, name)
                                                   identity that logs statistics of x (and of dy in the backward)
  quantize_state(name, device) / reset_quantize_states()
                                                   the per-name exponents and counters quantize keeps

Rounding and statistics run as the multi-tensor sm_90a kernels of csrc/quantize.cuh (bsmm_quantize,
bsmm_quantize_stats); AdamOptimizer(param_qspec=, mean_qspec=, var_qspec=) and Ema.apply(qspec=) use the same path.

A format's exponent exp_max lives in device memory as an int64 record, and the statistics kernel rewrites it there on
the calls the schedule picks, so quantize never synchronises the host unless a logfile asks for the statistics. The
schedule (which calls compute statistics) is host state: under CUDA graph capture it is taken once at capture time, and
a replay repeats the captured launches, statistics included, while the exponent and the Philox call counter advance on
the device. See DESIGN.md 7i.
"""
import math
import time

import numpy as np
import torch

from . import _lib

__all__ = ["QuantizeSpec", "quantize", "log_stats", "quantize_state", "reset_quantize_states"]

FREQ2 = 4                        # statistics calls at each power-of-two spacing before the spacing doubles


class QuantizeSpec(object):
    """A float format and how its exponent follows the data (reference quantize.py:20-46).

    ebits / fbits: exponent and fraction bits (1..8, 0..23). emax: the initial exp_max, by default the symmetric
    (1 << (ebits - 1)) - 1. stochastic: 0 rounds half away from zero; 1 or 2 rounds stochastically with words from the
    device's Philox state (ewops.set_entropy), so results depend on (seed, call, x) only; 1 is no longer clock-seeded.
    denorm: keep the format's subnormals. frequency: statistics (and a new exp_max) on the scheduled calls, 0 never.
    mode 0 sets exp_max from max |x|, mode 1 from mean |x| + stdv_mul * stdv; both add bias_pad. logfile: a file that
    gets one tab-separated row per statistics call. copy: take every field of another spec, keeping this spec's logfile
    when the copied one has none."""

    def __init__(self, ebits=4, fbits=3, emax=None, stochastic=0, denorm=True, frequency=1024, mode=0, bias_pad=2,
                 stdv_mul=4.0, logfile="", copy=None):
        if copy is None:
            self.ebits, self.fbits = ebits, fbits
            self.emax = (1 << (ebits - 1)) - 1 if emax is None else emax
            self.stoch, self.denorm, self.freq, self.mode = stochastic, denorm, frequency, mode
            self.bias_pad, self.stdv_mul, self.logfile = bias_pad, stdv_mul, logfile
        else:
            for k in ("ebits", "fbits", "emax", "stoch", "denorm", "freq", "mode", "bias_pad", "stdv_mul"):
                setattr(self, k, getattr(copy, k))
            self.logfile = copy.logfile or logfile

    def __repr__(self):
        return ("QuantizeSpec(ebits=%r, fbits=%r, emax=%r, stochastic=%r, denorm=%r, frequency=%r, mode=%r, bias_pad=%r, "
                "stdv_mul=%r, logfile=%r)" % (self.ebits, self.fbits, self.emax, self.stoch, self.denorm, self.freq,
                                              self.mode, self.bias_pad, self.stdv_mul, self.logfile))


def _check_spec(spec, what="qspec"):
    if not isinstance(spec, QuantizeSpec):
        raise ValueError("%s must be a QuantizeSpec, got %r" % (what, spec))
    for k, lo, hi in (("ebits", 1, 8), ("fbits", 0, 23)):
        v = getattr(spec, k)
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not lo <= v <= hi:
            raise ValueError("%s.%s must be an integer in %d..%d, got %r" % (what, k, lo, hi, v))
    if spec.stoch not in (0, 1, 2):
        raise ValueError("%s: stochastic must be 0, 1 or 2, got %r" % (what, spec.stoch))
    if spec.mode not in (0, 1):
        raise ValueError("%s: mode must be 0 or 1, got %r" % (what, spec.mode))
    if isinstance(spec.freq, bool) or not isinstance(spec.freq, (int, np.integer)) or spec.freq < 0:
        raise ValueError("%s: frequency must be an integer >= 0, got %r" % (what, spec.freq))
    for k in ("emax", "bias_pad"):
        if isinstance(getattr(spec, k), bool) or not isinstance(getattr(spec, k), (int, np.integer)):
            raise ValueError("%s.%s must be an integer, got %r" % (what, k, getattr(spec, k)))


def _check_dtype(dtype, specs, what):
    if dtype not in (torch.float32, torch.bfloat16):
        raise ValueError("%s: float32 and bfloat16 only (as the reference registers it), got %s" % (what, dtype))
    if dtype == torch.bfloat16:
        for s in specs:
            if s.fbits > 7:
                raise ValueError("%s: bfloat16 holds at most 7 fraction bits, the spec has %d" % (what, s.fbits))


# ---- schedule and state ------------------------------------------------------------------------------------------------
def new_schedule():
    """[count, pow2, pow2_count, max_stat_lo, max_stat_hi]: the reference QuantizeOp's counters (quantize_op.cc:60)."""
    return [1, 1, 0, float(np.finfo(np.float32).max), 0.0]


def _tick(sched, freq):
    """Advances a schedule by one call; returns (statistics on this call, the call's count)."""
    count, pow2, pow2_count = sched[0], sched[1], sched[2]
    now = bool(freq) and (count & (pow2 - 1)) == 0
    if now and (pow2 << 1) <= freq:
        if pow2_count == FREQ2:
            pow2, pow2_count = pow2 << 1, 0
        pow2_count += 1
    sched[0], sched[1], sched[2] = count + 1, pow2, pow2_count
    return now, count


def new_exponent(emax, device):
    """An exponent record: a 0-dim int64 tensor on `device`. Refused under CUDA graph capture, where its initial value
    would be a captured fill that every replay repeats."""
    if torch.cuda.is_current_stream_capturing():
        raise ValueError("quantize: a new exponent state cannot be created during CUDA graph capture; run the op once "
                         "before capturing it")
    return torch.full((), int(emax), dtype=torch.int64, device=device)


class QuantizeState(object):
    """The state quantize keeps per (name, device): exp_f / exp_b, the forward and backward exponents (0-dim int64 CUDA
    tensors, read or overwritten like the reference's variables: exp_f.fill_(3)), and the forward and backward
    schedules sched_f / sched_b ([count, pow2, pow2_count, max_stat_lo, max_stat_hi]; count - 1 calls so far).
    stats_f / stats_b hold the last statistics (fp32 [5]: mean |x|, stdv, sat %, ftz %, max |x|)."""

    def __init__(self, name, device, emax_f, emax_b):
        self.name, self.device = name, device
        self.exp_f, self.exp_b = new_exponent(emax_f, device), new_exponent(emax_b, device)
        self.sched_f, self.sched_b = new_schedule(), new_schedule()
        self.stats_f = torch.zeros(5, dtype=torch.float32, device=device)
        self.stats_b = torch.zeros(5, dtype=torch.float32, device=device)

    @property
    def calls_f(self):
        return self.sched_f[0] - 1

    @property
    def calls_b(self):
        return self.sched_b[0] - 1


_STATES = {}                     # (name, device index) -> QuantizeState
_LOG_STATES = {}                 # (name, device index) -> _LogStatsState


def _device_of(device):
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise ValueError("quantize state lives on a CUDA device, got %s" % dev)
    return dev if dev.index is not None else torch.device("cuda", torch.cuda.current_device())


def quantize_state(name="quantize", device=None):
    """The QuantizeState of `name` on `device` (default: the current one), or None before its first quantize call."""
    return _STATES.get((name, _device_of(device).index))


def reset_quantize_states():
    """Forgets every quantize and log_stats state: the next call of each name starts again from its spec's emax."""
    _STATES.clear()
    _LOG_STATES.clear()


# ---- log files ---------------------------------------------------------------------------------------------------------
QUANT_HEADERS = ["sat_pct", "ftz_pct", "exp_max", "exp_min", "max", "mean", "stdv", "mean+stdv5", "max_stat_lo",
                 "max_stat_hi", "count", "name"]
STAT_HEADERS = ["sat_pct", "ftz_pct", "max", "mean", "stdv", "mean+stdv5", "max_stat_lo", "max_stat_hi", "count", "name"]
_LOG_INIT = set()
_TIMESTAMP = None


def get_timestamp():
    global _TIMESTAMP
    if _TIMESTAMP is None:
        _TIMESTAMP = time.strftime("%Y_%m_%d_%H_%M_%S")
    return _TIMESTAMP


def _init_log(logfile, headers):
    if logfile and logfile not in _LOG_INIT:
        with open(logfile, "w") as f:
            f.write("\t".join(headers) + "\n")
        _LOG_INIT.add(logfile)


def fexp(v):
    """The unbiased exponent field of v's fp32 bit pattern, as the reference's log columns print it."""
    return int(np.array([v], np.float32).view(np.int32)[0] >> 23) - 127


def format_exponents(exp, spec):
    """(exponent of max_float, exponent of min_float) of the format at exponent record value `exp`."""
    top = 254 if spec.ebits == 8 else (1 << spec.ebits) - 1
    em = min(max(int(exp) + 127, top), 254)
    exp_min = max(em - top + 1 - (spec.fbits if spec.denorm else 0), 2)
    return em - 127, exp_min - 127


def quant_row(stats, exp, spec, sched, count, name):
    """One row of a quantize log: stats (mean, stdv, sat %, ftz %, max) as fp32, exp the updated record."""
    mean, stdv, sat, ftz, mx = (np.float32(v) for v in stats)
    e_max, e_min = format_exponents(exp, spec)
    return "%.3f\t%.3f\t%3d\t%3d\t%3d\t%3d\t%3d\t%3d\t%3d\t%3d\t%d\t%s\n" % (
        sat, ftz, e_max, e_min, fexp(mx), fexp(mean), fexp(stdv), fexp(mean + stdv * np.float32(5.0)),
        fexp(sched[3]), fexp(sched[4]), count, name)


def stat_row(stats, lo, hi, step, name):
    mean, stdv, sat, ftz, mx = (np.float32(v) for v in stats)
    return "%.6f\t%.6f\t%3d\t%3d\t%3d\t%3d\t%3d\t%3d\t%d\t%s\n" % (
        sat, ftz, fexp(mx), fexp(mean), fexp(stdv), fexp(mean + stdv * np.float32(5.0)), fexp(lo), fexp(hi), step, name)


def _track(sched, mx):
    mx = float(np.float32(mx))
    sched[3] = min(sched[3], mx)
    sched[4] = max(sched[4], mx)


# ---- launches ----------------------------------------------------------------------------------------------------------
def _arr(vals, dtype):
    return np.array(vals, dtype=dtype)


def _stats_launch(xs, exps, out, spec=None, sat_val=0.0, ftz_val=0.0):
    """bsmm_quantize_stats over xs (one device, current) into out (fp32 [len(xs), 5]); quantize mode when exps."""
    lib = _lib.load()
    sizes = _arr([x.numel() for x in xs], np.int64)
    ws = torch.empty(max(lib.bsmm_quantize_stats_workspace_bytes(len(xs), sizes.ctypes.data) // 4, 1),
                     dtype=torch.float32, device=xs[0].device)
    xp = _arr([x.data_ptr() for x in xs], np.uint64)
    ep = _arr([e.data_ptr() for e in exps], np.uint64) if exps is not None else None
    s = spec or QuantizeSpec()
    rc = lib.bsmm_quantize_stats(len(xs), _lib.dtype_code(xs[0].dtype), xp.ctypes.data, sizes.ctypes.data,
                                 None if ep is None else ep.ctypes.data, out.data_ptr(), int(s.ebits), int(s.fbits),
                                 int(bool(s.denorm)), int(s.mode), int(s.bias_pad), float(s.stdv_mul), float(sat_val),
                                 float(ftz_val), ws.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "bsmm_quantize_stats")


def quantize_tensors(xs, ys, exps, scheds, spec, names, stats_out=None):
    """Rounds xs[i] into ys[i] (ys[i] may be xs[i]) with spec and the exponent record exps[i], all contiguous, non-empty,
    of one dtype and on the current device; scheds[i] is tensor i's schedule. One statistics launch covers the tensors
    whose schedule picks this call (quantize mode: it rewrites their records), then one quantize launch covers all of
    them (one more of each per 256 tensors). With spec.logfile the statistics are copied back and one row per tensor is
    appended, named names[i]. stats_out, when given, receives each scheduled tensor's statistics row (a list of fp32 [5]
    tensors aligned with xs, or None entries to skip)."""
    if spec.logfile and torch.cuda.is_current_stream_capturing():
        raise ValueError("quantize: a logfile reads the statistics back, which CUDA graph capture does not allow")
    lib = _lib.load()
    picked = []
    for i, sched in enumerate(scheds):
        now, count = _tick(sched, spec.freq)
        if now:
            picked.append((i, count))
    if picked:
        out = torch.empty((len(picked), 5), dtype=torch.float32, device=xs[0].device)
        _stats_launch([xs[i] for i, _ in picked], [exps[i] for i, _ in picked], out, spec)
        if stats_out is not None:
            for r, (i, _) in enumerate(picked):
                if stats_out[i] is not None:
                    stats_out[i].copy_(out[r])
        if spec.logfile:
            host = out.cpu().numpy()
            ex = [int(exps[i].item()) for i, _ in picked]
            _init_log(spec.logfile, QUANT_HEADERS)
            with open(spec.logfile, "a") as f:
                for r, (i, count) in enumerate(picked):
                    _track(scheds[i], host[r][4])
                    f.write(quant_row(host[r], ex[r], spec, scheds[i], count, names[i]))
    entropy = None
    if spec.stoch:
        from .ewops import get_entropy
        entropy = get_entropy(xs[0].device)
    sizes = _arr([x.numel() for x in xs], np.int64)
    xp, yp, ep = (_arr([t.data_ptr() for t in ts], np.uint64) for ts in (xs, ys, exps))
    rc = lib.bsmm_quantize(len(xs), _lib.dtype_code(xs[0].dtype), xp.ctypes.data, yp.ctypes.data, ep.ctypes.data,
                           sizes.ctypes.data, int(spec.ebits), int(spec.fbits), int(bool(spec.denorm)), int(spec.stoch),
                           _lib.ptr(entropy), _lib.stream_ptr())
    _lib.check(rc, "bsmm_quantize")


# ---- quantize ----------------------------------------------------------------------------------------------------------
def _state(name, device, qspec, b_qspec):
    key = (name, device.index)
    st = _STATES.get(key)
    if st is None:
        st = _STATES[key] = QuantizeState(name, device, qspec.emax, b_qspec.emax)
    return st


def _quantize_one(x, spec, exp, sched, stats, name):
    x = x.contiguous()
    y = torch.empty_like(x)
    if x.numel():
        with torch.cuda.device(x.device):
            quantize_tensors([x], [y], [exp], [sched], spec, [name], stats_out=[stats])
    return y


class _QuantizeFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, qspec, b_qspec, st):
        ctx.args = (b_qspec, st)
        return _quantize_one(x, qspec, st.exp_f, st.sched_f, st.stats_f, st.name)

    @staticmethod
    def backward(ctx, dy):
        b_qspec, st = ctx.args
        _check_dtype(dy.dtype, [b_qspec], "quantize backward")
        return _quantize_one(dy, b_qspec, st.exp_b, st.sched_b, st.stats_b, st.name + "_grad"), None, None, None


def quantize(x, qspec, b_qspec=None, name=None):
    """x rounded to qspec's format (reference quantize.py:74-121); differentiable: the gradient is dy rounded to b_qspec
    (default qspec) with a separate backward state.

    x: a float32 or bfloat16 CUDA tensor (fp16 raises ValueError, as the reference registers fp32 and bf16 only; so does
    bf16 with fbits > 7); a non-contiguous x is copied and an empty one returns without a launch. Rounding is the
    reference kernel's, bit for bit, except that NaN stays NaN. State is kept per (name, device), name=None meaning
    "quantize": the forward and backward exponents start at qspec.emax and b_qspec.emax, and each direction has its own
    call count and statistics schedule (see quantize_state). Creating a state during CUDA graph capture raises
    ValueError; capture after one eager call. No call synchronises the host unless a spec has a logfile."""
    name = "quantize" if name is None else str(name)
    b_qspec = qspec if b_qspec is None else b_qspec
    _check_spec(qspec, "qspec")
    _check_spec(b_qspec, "b_qspec")
    if not torch.is_tensor(x):
        raise ValueError("quantize: x must be a tensor, got %r" % type(x))
    _check_dtype(x.dtype, (qspec, b_qspec), "quantize")
    if not x.is_cuda:
        raise ValueError("quantize needs a CUDA tensor (there is no CPU path)")
    if (qspec.logfile or b_qspec.logfile) and torch.cuda.is_current_stream_capturing():
        raise ValueError("quantize: a logfile reads the statistics back, which CUDA graph capture does not allow")
    for spec in (qspec, b_qspec):
        _init_log(spec.logfile, QUANT_HEADERS)
    with torch.cuda.device(x.device):
        st = _state(name, x.device, qspec, b_qspec)
        if (qspec.stoch or b_qspec.stoch):
            from .ewops import get_entropy
            get_entropy(x.device)          # created now, not inside a later capture of the backward
    return _QuantizeFunction.apply(x, qspec, b_qspec, st)


# ---- log_stats ---------------------------------------------------------------------------------------------------------
def _is_pow2_or_0(v):
    return isinstance(v, (int, np.integer)) and not isinstance(v, bool) and (v == 0 or (v > 0 and v & (v - 1) == 0))


def _logs_at(step, freq, first_steps, prev):
    """The reference LogStatsOp's rule (quantize_op.cc:236-253): once per step value, at first_steps below freq and at
    multiples of freq from there on. prev is a one-element list holding the last step seen."""
    if not freq or step == prev[0]:
        return False
    prev[0] = step
    if step < freq:
        return step in first_steps
    return (step & (freq - 1)) == 0


def log_statistics(x, sat_val, ftz_val):
    """fp32 [5] CUDA tensor: mean |x|, stdv, sat % (|x| >= sat_val), ftz % (non-zero |x| < ftz_val) and max |x| over x
    (fp32, fp16 or bf16), from the deterministic statistics kernel. No host synchronisation."""
    x = x.contiguous()
    out = torch.zeros((1, 5), dtype=torch.float32, device=x.device)
    if x.numel():
        with torch.cuda.device(x.device):
            _stats_launch([x], None, out, sat_val=sat_val, ftz_val=ftz_val)
    return out[0]


class _LogStatsState(object):
    def __init__(self):
        self.prev = [[-1], [-1]]                       # forward, backward
        self.sched = [new_schedule(), new_schedule()]  # only the max_stat_lo / hi slots are used
        self.stats = [None, None]                      # the last statistics, fp32 [5] CUDA tensors


def _log_one(x, step, which, st, sat_val, ftz_val, freq, first_steps, logfile, name):
    if not _logs_at(step, freq, first_steps, st.prev[which]) or x.numel() == 0:
        return
    s = st.stats[which] = log_statistics(x, sat_val, ftz_val)
    if logfile:
        host = s.cpu().numpy()
        _track(st.sched[which], host[4])
        _init_log(logfile, STAT_HEADERS)
        with open(logfile, "a") as f:
            f.write(stat_row(host, st.sched[which][3], st.sched[which][4], step, name))


class _LogStatsFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, step, st, args):
        sat_val, ftz_val, freq, bfreq, first_steps, logfile, name = args
        ctx.args = (step, st, args)
        _log_one(x, step, 0, st, sat_val, ftz_val, freq, first_steps, logfile, name)
        return x.view_as(x)

    @staticmethod
    def backward(ctx, dy):
        step, st, (sat_val, ftz_val, freq, bfreq, first_steps, logfile, name) = ctx.args
        _log_one(dy, step, 1, st, sat_val, ftz_val, bfreq, first_steps, logfile, name + "_grad")
        return dy, None, None, None


def log_stats(x, step, sat_val=65504.0, ftz_val=2.0 ** -24, freq=512, bfreq=512, logfile="", name=None):
    """Identity on x that logs statistics of x, and of dy in the backward (reference quantize.py:155-191).

    A step logs when its value differs from the previous call's and it is one of 1, 2, 4, ... below freq, or a multiple
    of freq from freq on; the backward does the same with bfreq. freq and bfreq must be 0 (never) or a power of two
    (ValueError otherwise). On a logging step the statistics kernel runs (mean |x|, stdv, the shares of |x| >= sat_val
    and of non-zero |x| < ftz_val, max |x|) and, with a logfile, its five values are copied back and appended as one
    row in the reference's columns; other steps launch nothing. logfile may contain "%(timestamp)s", replaced by the
    process's first-call time. x: fp32, fp16 or bf16 on a CUDA device. step: an int or a one-element tensor; reading a
    CUDA one synchronises the host. State (the previous step, max_stat_lo / hi) is kept per (name, device)."""
    if not _is_pow2_or_0(freq) or not _is_pow2_or_0(bfreq):
        raise ValueError("log_stats: freq and bfreq must be 0 or a power of two, got %r and %r" % (freq, bfreq))
    if not torch.is_tensor(x) or x.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise ValueError("log_stats: x must be a float32, float16 or bfloat16 tensor")
    if not x.is_cuda:
        raise ValueError("log_stats needs a CUDA tensor (there is no CPU path)")
    if torch.is_tensor(step):
        if step.numel() != 1 or step.dtype not in (torch.int32, torch.int64):
            raise ValueError("log_stats: step must be an int or a one-element int32 / int64 tensor")
        step = int(step.item())
    elif isinstance(step, (int, np.integer)) and not isinstance(step, bool):
        step = int(step)
    else:
        raise ValueError("log_stats: step must be an int or a one-element tensor, got %r" % (step,))
    logfile = logfile % {"timestamp": get_timestamp()}
    if logfile and torch.cuda.is_current_stream_capturing():
        raise ValueError("log_stats: a logfile reads the statistics back, which CUDA graph capture does not allow")
    _init_log(logfile, STAT_HEADERS)
    pow2 = int(math.log2(freq or bfreq)) if (freq or bfreq) else 0
    first_steps = [1 << p for p in range(pow2)]
    name = name or "log_stats"
    key = (name, x.device.index)
    st = _LOG_STATES.get(key)
    if st is None:
        st = _LOG_STATES[key] = _LogStatsState()
    args = (float(sat_val), float(ftz_val), int(freq), int(bfreq), first_steps, logfile, name)
    return _LogStatsFunction.apply(x, step, st, args)
