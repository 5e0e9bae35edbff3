"""The quantize oracle (oracle/quantize_oracle.py) on the CPU: rounding properties over every format, the statistics
schedule against an independent loop, the log rows' columns, and no reference line kept under oracle/."""
import importlib
import os
import subprocess

import numpy as np
import pytest

from oracle import quantize_oracle as qo

qm = importlib.import_module("blocksparse_b200.quantize")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("BLOCKSPARSE_REFERENCE") or "/root/reference"
FORMATS = [(e, f, d) for e in range(1, 9) for f in range(0, 24) for d in (True, False)]


def _inputs(rng, e, ebits, fbits, denorm, n=3000):
    """Finite values around the format's range: its normal and subnormal range, ties, max_float and just past it,
    min_float and just below it, fp32 subnormals and zeros."""
    f = qo.fmt(e, ebits, fbits, denorm)
    lo, hi = f["exp_min"] - 127, f["em"] - 127
    ex = rng.uniform(lo - 3, hi + 2, n)
    x = (np.sign(rng.normal(size=n)) * np.exp2(ex) * rng.uniform(1, 2, n)).astype(np.float32)
    grid = qo.quantize(x, e, ebits, fbits, denorm)
    ulp = np.exp2(np.floor(np.log2(np.abs(grid.astype(np.float64)) + 1e-300)) - fbits).astype(np.float32)
    mx, mn = qo._f(np.uint32(f["max_float"])), qo._f(np.uint32(f["min_float"]))
    extra = np.array([0, -0.0, 1e-45, -1e-40, mx, -mx, np.nextafter(mx, np.float32(np.inf)), mn, -mn,
                      np.nextafter(mn, np.float32(0)), 3.4e38, -3.4e38], np.float32)
    ties = (grid + np.float32(0.5) * ulp).astype(np.float32)
    return np.concatenate([x, extra, ties[np.isfinite(ties)]]).astype(np.float32)


def _wraps(x, f):
    """Elements whose subnormal shift wraps past bit 31: without denorm, exp_norm is negative once exp_min is clamped
    at 2, and a clamped value whose exponent field plus that shift reaches 255 leaves the fp32 range. The reference
    kernel wraps the same way and the port keeps its arithmetic; such values have no meaning in the format."""
    if f["exp_norm"] < 2 ** 31:
        return np.zeros(np.shape(x), bool)
    k = (2 ** 32 - f["exp_norm"]) >> 23
    v = np.minimum(np.abs(x), qo._f(np.uint32(f["max_float"])))
    return ((v.view(np.uint32) >> 23) + k) >= 255


@pytest.mark.parametrize("ebits", range(1, 9))
def test_rounding_properties_over_every_format(ebits):
    rng = np.random.default_rng(ebits)
    for fbits in range(0, 24):
        for denorm in (True, False):
            top = qo.top_exponent(ebits) - 127
            for e in sorted({top, top + 3, (1 << (ebits - 1)) - 1, 0, -20, 127}):
                x = _inputs(rng, e, ebits, fbits, denorm)
                q = qo.quantize(x, e, ebits, fbits, denorm)
                f = qo.fmt(e, ebits, fbits, denorm)
                mx = qo._f(np.uint32(f["max_float"]))
                ok = ~_wraps(x, f)
                if f["exp_min"] == f["em"] - qo.top_exponent(ebits) + 1 - (fbits if denorm else 0):
                    # never past max_float, unless the format reaches below fp32's normal range: exp_min is then
                    # clamped at 2 and the round to nearest in fp32's subnormals may carry max_float up a binade
                    assert np.all(np.abs(q[ok]) <= mx), (ebits, fbits, denorm, e)
                np.testing.assert_array_equal(qo.quantize(q[ok], e, ebits, fbits, denorm), q[ok])   # idempotent
                np.testing.assert_array_equal(qo.quantize(-x[ok], e, ebits, fbits, denorm), -q[ok])  # odd
                srt = np.sort(x[ok])
                qs = qo.quantize(srt, e, ebits, fbits, denorm)
                assert np.all(np.diff(qs.astype(np.float64)) >= 0), (ebits, fbits, denorm, e)         # monotonic
                # within half an ulp in the format's normal range
                norm = ok & (np.abs(x) >= np.float32(2.0 ** (f["exp_min"] - 127 + (fbits if denorm else 0)))) & \
                    (np.abs(x) <= mx)
                xv = x[norm].astype(np.float64)
                ulp = np.exp2(np.floor(np.log2(np.abs(xv))) - fbits)
                assert np.all(np.abs(q[norm] - xv) <= 0.5 * ulp), (ebits, fbits, denorm, e)
                if fbits <= 7:
                    # every quantized value fits bf16 exactly: nothing below bit 16 of the fp32 pattern
                    assert not np.any(q[ok].view(np.uint32) & 0xFFFF), (ebits, fbits, denorm, e)


def test_wrapping_subnormal_shift_is_only_a_no_denorm_corner():
    """With denorm=False the subnormal shift subtracts (exp_min - 1 - fbits) << 23, which is negative once exp_min is
    clamped at 2, so large exponents wrap past bit 31 as in the reference kernel. That happens only without denorm."""
    for ebits, fbits, denorm in FORMATS:
        for e in (-200, 0, 127):
            f = qo.fmt(e, ebits, fbits, denorm)
            if f["exp_norm"] >= 2 ** 31:
                assert not denorm


def test_special_values():
    x = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-40, -1e-40], np.float32)
    q = qo.quantize(x, 7, 4, 3, True)
    assert np.all(q.view(np.uint32)[:2] == qo.NAN_BITS)
    assert q[2] == 240 and q[3] == -240 and np.all(q.view(np.uint32)[4:] == 0)
    # round half away from zero at fbits, ties of the format
    assert list(qo.quantize(np.array([1.0625, -1.0625, 1.1875], np.float32), 7, 4, 3, True)) == [1.125, -1.125, 1.25]
    # stochastic: a zero word truncates, an all-ones word rounds up
    x = np.array([1.01, 1.01], np.float32)
    assert list(qo.quantize(x, 7, 4, 3, True, words=np.array([0, 0xFFFFFFFF], np.uint32))) == [1.0, 1.125]


def _schedule_by_rule(freq, n):
    """Statistics calls from the counters' meaning: at spacing s = 1, 2, 4, ... < freq a call runs them when its count
    is a multiple of s, and the spacing doubles after four calls at it (counted with the call that doubles it)."""
    if not freq:
        return []
    out, s, k = [], 1, 0
    for c in range(1, n + 1):
        if c % s:
            continue
        out.append(c)
        if 2 * s <= freq:
            if k == 4:
                s, k = 2 * s, 0
            k += 1
    return out


@pytest.mark.parametrize("freq", [0, 1, 2, 8, 1024])
def test_schedule_matches_the_reference_loop(freq):
    orc = qo.Schedule(freq)
    got = [c for c in range(1, 5001) if orc.step()]
    assert got == _schedule_by_rule(freq, 5000)
    sched = qm.new_schedule()
    assert [c for c in range(1, 5001) if qm._tick(sched, freq)[0]] == got
    if freq == 8:
        assert got[:14] == [1, 2, 3, 4, 5, 6, 8, 10, 12, 16, 20, 24, 28, 32]
        assert all(c % 8 == 0 for c in got[13:])
    if freq == 1024:
        assert got[-4:] == [2560, 3072, 3584, 4096] and max(np.diff(got)) <= 1024


def test_log_row_formats():
    st = (np.float32(0.03), np.float32(0.2), np.float32(1.5), np.float32(12.25), np.float32(7.5))
    spec = qm.QuantizeSpec(ebits=4, fbits=3)
    sched = qm.new_schedule()
    qm._track(sched, 7.5)
    qm._track(sched, 0.25)
    row = qm.quant_row(st, 5, spec, sched, 17, "fc1")
    assert row == qo.quant_log_row(st, 5, 4, 3, True, np.float32(0.25), np.float32(7.5), 17, "fc1")
    cols = row.rstrip("\n").split("\t")
    assert len(cols) == len(qm.QUANT_HEADERS) == 12
    assert cols[:2] == ["1.500", "12.250"] and cols[2:4] == ["  5", "-12"] and cols[4:8] == ["  2", " -6", " -3", "  0"]
    assert cols[8:] == [" -2", "  2", "17", "fc1"]
    row = qm.stat_row(st, np.float32(0.25), np.float32(7.5), 512, "x")
    assert row == qo.stat_log_row(st, np.float32(0.25), np.float32(7.5), 512, "x")
    cols = row.rstrip("\n").split("\t")
    assert len(cols) == len(qm.STAT_HEADERS) == 10 and cols[:2] == ["1.500000", "12.250000"] and cols[-2:] == ["512", "x"]


def test_headers_match_the_reference():
    path = os.path.join(REF, "blocksparse", "quantize.py")
    if not os.path.isfile(path):
        pytest.skip("no reference checkout")
    import ast
    tree = ast.parse(open(path).read())
    lists = {t.targets[0].id: ast.literal_eval(t.value) for t in tree.body
             if isinstance(t, ast.Assign) and isinstance(t.targets[0], ast.Name) and t.targets[0].id.endswith("headers")}
    assert lists["quant_headers"] == qm.QUANT_HEADERS and lists["stat_headers"] == qm.STAT_HEADERS


def test_statistics_and_exponent_update():
    rng = np.random.default_rng(3)
    x = rng.normal(0, 3, 10001).astype(np.float32)
    x[:3] = [np.nan, 1e-30, 0.0]
    st = qo.stats(x, 4.0, 2.0 ** -24)
    a = np.abs(np.where(np.isnan(x), np.inf, x)).astype(np.float64)
    assert st[0] == np.float32(a.mean()) and st[4] == np.inf and st[2] == np.float32(100.0 * (a >= 4).sum() / a.size)
    assert st[3] == np.float32(100.0 / a.size)
    # an inf statistic clamps the exponent so that max_float stays finite
    assert qo.next_exponent(st, 5, 0, 2, 4.0) == 127
    assert qo.next_exponent((0, 0, 0, 0, np.float32(0.0)), 5, 0, 2, 4.0) == 31 - 127
    assert qo.next_exponent((np.float32(1.0), np.float32(0.5), 0, 0, np.float32(100.0)), 4, 1, 2, 4.0) == 1 + 2
    assert qo.next_exponent((np.float32(1.0), np.float32(0.5), 0, 0, np.float32(100.0)), 4, 0, 1, 4.0) == 6 + 1


def test_no_reference_line_in_oracle():
    srcs = [os.path.join(REF, "src", f) for f in ("quantize_op_gpu.cu", "quantize_op.cc")]
    if not all(os.path.isfile(p) for p in srcs):
        pytest.skip("no reference checkout")
    lines = set()
    for p in srcs:
        with open(p, errors="replace") as fh:
            for line in fh:
                s = "".join(line.split())
                if len(s) >= 10:
                    lines.add(s)
    tracked = subprocess.run(["git", "ls-files", "oracle"], cwd=ROOT, capture_output=True, text=True)
    if tracked.returncode != 0:
        pytest.skip("not a git checkout")
    paths = tracked.stdout.split() + ["oracle/quantize_oracle.py", "oracle/ref/quantize.cu", "oracle/ref_quantize.py"]
    for path in sorted(set(paths)):
        if not os.path.isfile(os.path.join(ROOT, path)):
            continue
        with open(os.path.join(ROOT, path), errors="replace") as fh:
            for n, line in enumerate(fh, 1):
                s = "".join(line.split())
                assert s not in lines, "%s:%d repeats a line of the reference's quantize sources" % (path, n)
