"""The float64 optimizer oracle (oracle/optimize_oracle.py) against the CPU formula of the reference's test/adam_test.py
and the documented 16-bit moment codes. No GPU needed."""
import numpy as np
import pytest

from oracle import optimize_oracle as oo

# test/adam_test.py: beta1 0.8, beta2 0.5, lr 0.5, clip_norm 1, grad_scale 1, clip_sigma 0, epsilon 1e-8, and its shapes
SHAPES = [(1,), (3,), (127,), (1, 1024), (1023, 1024), (1024, 1024)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_adam_matches_reference_test_formula(shape):
    rng = np.random.default_rng(len(shape) * 7 + shape[-1])
    G, P, M = (rng.uniform(-1, 1, shape).astype(np.float16).astype(np.float64) for _ in range(3))
    M = np.abs(M)
    V = rng.uniform(0, 1, shape).astype(np.float16).astype(np.float64)
    b1, b2, lr, eps, clip_norm, grad_scale = 0.8, 0.5, 0.5, 1e-8, 1.0, 1.0
    norm, scale = oo.global_norm([G], clip_norm=clip_norm, grad_scale=grad_scale)
    p, m, v = oo.adam(G, P, M, V, lr, b1, b2, eps, grad_scale=grad_scale, norm_scale=scale)
    # the reference's CPU restatement, line for line
    GN = np.sqrt(np.sum(np.square(G * grad_scale)))
    NS = clip_norm / np.maximum(GN, clip_norm)
    Gs = G * NS * grad_scale
    Mr = b1 * M + (1.0 - b1) * Gs
    Vr = b2 * V + (1.0 - b2) * Gs * Gs
    Pr = P - lr * Mr / (np.sqrt(Vr) + eps)
    assert norm == pytest.approx(GN, rel=1e-12) and scale == pytest.approx(NS, rel=1e-12)
    np.testing.assert_allclose(m, Mr, rtol=1e-12, atol=0)
    np.testing.assert_allclose(v, Vr, rtol=1e-12, atol=0)
    np.testing.assert_allclose(p, Pr, rtol=1e-12, atol=1e-15)


def test_adam_clip_sigma_and_gate():
    rng = np.random.default_rng(1)
    bs, blocks = 8, 5
    g, p, m = (rng.normal(0, 1, (blocks, bs, bs)) for _ in range(3))
    v = rng.uniform(0, 1, (blocks, bs, bs))
    gate = np.array([1, 0, 1, 0, 0.5], np.float32)
    p1, m1, v1 = oo.adam(g, p, m, v, 0.1, 0.9, 0.99, 1e-8, clip_sigma=0.5, gate=gate, bs=bs)
    for b in (1, 3):
        assert np.array_equal(p1[b], p[b]) and np.array_equal(m1[b], m[b]) and np.array_equal(v1[b], v[b])
    vv = 0.99 * v[0] + 0.01 * g[0] ** 2
    gc = np.clip(g[0], -0.5 * np.sqrt(vv), 0.5 * np.sqrt(vv))
    np.testing.assert_allclose(m1[0], 0.9 * m[0] + 0.1 * gc)
    assert np.all(np.abs(gc) <= 0.5 * np.sqrt(vv))


def test_adam_conditioning_order():
    g = np.array([np.inf, -np.inf, np.nan, 3.0, -3.0, 0.5])
    assert np.array_equal(oo.condition(g, zero_infs=True, zero_nans=True), [0, 0, 0, 3, -3, 0.5])
    assert np.array_equal(oo.condition(g, saturate=1.0, zero_nans=True), [1, -1, 0, 1, -1, 0.5])
    p, m, v = oo.adam(g, np.ones(6), np.zeros(6), np.zeros(6), 0.1, 0.9, 0.999, 1e-8, norm_scale=0.0)
    assert np.array_equal(p, np.ones(6)) and not m.any() and not v.any()


def test_codec_examples():
    assert oo.mean_encode(np.array([1.0, -1.0, oo.MEAN_MAX, 0.0])).tolist() == [0x7800, 0xF800, 0x7FFF, 0]
    assert oo.var_encode(np.array([1.0, oo.VAR_MAX, 0.0])).tolist() == [0xF000, 0xFFFF, 0]
    assert oo.mean_decode(0x7800) == 1.0 and oo.mean_decode(0xF800) == -1.0 and oo.mean_decode(0x7FFF) == oo.MEAN_MAX
    assert oo.var_decode(0xF000) == 1.0 and oo.var_decode(0xFFFF) == oo.VAR_MAX
    assert oo.mean_decode(0) == 0.0 and oo.var_decode(0) == 0.0


def test_codec_clamps_and_flushes():
    assert oo.mean_encode(np.array([100.0, -1e30, np.inf, -np.inf, np.nan])).tolist() == [0x7FFF, 0xFFFF, 0x7FFF, 0xFFFF, 0x7FFF]
    assert oo.var_encode(np.array([100.0, np.inf, np.nan])).tolist() == [0xFFFF] * 3
    tiny = np.array([oo.MEAN_MIN * 0.999, -oo.MEAN_MIN * 0.999, 2.0 ** -61, 1e-30])
    assert not oo.mean_encode(tiny).any()
    assert oo.mean_encode(np.array([oo.MEAN_MIN])).tolist() == [1]
    assert not oo.var_encode(np.array([oo.VAR_MIN * 0.999, 2.0 ** -61, -1.0])).any()
    assert oo.var_encode(np.array([oo.VAR_MIN])).tolist() == [1]


@pytest.mark.parametrize("which", ["mean", "var"])
def test_codec_round_trip_monotone_and_within_half_ulp(which):
    rng = np.random.default_rng(3)
    enc, dec, mbits = (oo.mean_encode, oo.mean_decode, 9) if which == "mean" else (oo.var_encode, oo.var_decode, 10)
    top = oo.MEAN_MAX if which == "mean" else oo.VAR_MAX
    lo = oo.MEAN_MIN if which == "mean" else oo.VAR_MIN
    mag = np.exp(rng.uniform(np.log(lo), np.log(top), 200000)).astype(np.float32).astype(np.float64)
    vals = np.sort(mag)
    codes = enc(vals)
    back = dec(codes)
    assert np.all(np.diff(codes.astype(np.int64)) >= 0)                     # monotone
    assert np.all(np.diff(back) >= 0)
    ulp = np.ldexp(1.0, np.floor(np.log2(vals)).astype(int) - mbits)
    assert np.all(np.abs(back - vals) <= 0.5 * ulp * (1 + 1e-12))
    # every code decodes and re-encodes to itself
    allc = np.arange(1, 0x8000 if which == "mean" else 0x10000)
    assert np.array_equal(enc(dec(allc)), allc.astype(np.uint16))
    if which == "mean":
        assert np.array_equal(enc(-vals), codes | 0x8000)                  # sign-symmetric
    # half-ulp ties round away from zero (mean) / up (var)
    x = 1.0 + 0.5 / (1 << mbits)
    assert dec(enc(np.array([x])))[0] == 1.0 + 1.0 / (1 << mbits)


def test_global_norm_and_scale():
    rng = np.random.default_rng(5)
    gs = [rng.normal(0, 1, n) for n in (0, 3, 1000)]
    n, s = oo.global_norm(gs, clip_norm=1.0, grad_scale=0.5)
    assert n == pytest.approx(0.5 * np.sqrt(sum((g ** 2).sum() for g in gs)))
    assert s == pytest.approx(1.0 / n)
    assert oo.global_norm(gs, clip_norm=1e9)[1] == 1.0
    assert oo.global_norm([]) == (0.0, 1.0)


@pytest.mark.parametrize("bad", [np.inf, -np.inf, np.nan])
def test_non_finite_global_norm_gives_zero_scale(bad):
    g = np.array([1.0, bad, 2.0])
    n, s = oo.global_norm([g])
    assert not np.isfinite(n) and s == 0.0
    n, s = oo.global_norm([g], zero_infs=True, zero_nans=True)
    assert n == pytest.approx(np.sqrt(5.0)) and s == pytest.approx(1 / np.sqrt(5.0))


def test_global_norm_overflow_gives_zero_scale():
    assert oo.global_norm([np.array([1e200, 1e200])])[1] == 0.0


def test_ema_dense_and_gated():
    rng = np.random.default_rng(7)
    e, p = rng.normal(0, 1, (3, 8, 8)), rng.normal(0, 1, (3, 8, 8))
    np.testing.assert_allclose(oo.ema(e, p, 0.9), 0.9 * e + 0.1 * p, rtol=1e-14)
    got = oo.ema(e, p, 0.9, gate=np.array([0, 1, 0], np.float32), bs=8)
    assert np.array_equal(got[0], e[0]) and np.array_equal(got[2], e[2])
    np.testing.assert_allclose(got[1], 0.9 * e[1] + 0.1 * p[1], rtol=1e-14)
