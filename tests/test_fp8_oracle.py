"""oracle/fp8_oracle.py against torch's own fp8 casts (no GPU): the rounding agrees bit for bit with
torch.float8_e4m3fn / float8_e5m2 casts of clamp(x * s) for every bf16 code at several scales, NaN aside (the
hardware and the oracle drop a NaN's sign, torch keeps it), and the scale rules follow the header."""
import numpy as np
import pytest
import torch

from oracle import fp8_oracle as fo

TORCH = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
ALL_BF16 = (np.arange(65536, dtype=np.uint32) << 16).view(np.float32)
SCALES = [1.0, 0.3, 3.7, 2.0 ** -120, 2.0 ** 100, 1e-30, 448 / 3.0e38, 57344 / 1.5, 448 / 0.75]


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
@pytest.mark.parametrize("scale", SCALES)
def test_rounding_matches_torch_for_every_bf16_code(fmt, scale):
    s = np.float32(scale)
    with np.errstate(all="ignore"):
        v = ALL_BF16 * s
    got = fo.round_fp8(v, fmt)
    mx = fo.FP8_MAX[fmt]
    ref = torch.from_numpy(v).clamp(-mx, mx).to(TORCH[fmt]).view(torch.uint8).numpy()
    nan = np.isnan(v)
    bad = (got != ref) & ~nan
    assert not bad.any(), (v[bad][:4], got[bad][:4], ref[bad][:4])
    assert (got[nan] == 0x7F).all()
    assert np.array_equal(fo.decode(got[~nan], fmt), torch.from_numpy(ref[~nan]).view(TORCH[fmt]).double().numpy())


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_decode_matches_torch_for_every_code(fmt):
    codes = np.arange(256, dtype=np.uint8)
    ref = torch.from_numpy(codes).view(TORCH[fmt]).double().numpy()
    got = fo.decode(codes, fmt)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert np.array_equal(got[ok], ref[ok])
    ok = np.isfinite(ref)                                   # satfinite maps e5m2's infinities to +-max
    assert np.array_equal(fo.round_fp8(got[ok].astype(np.float32), fmt), codes[ok])     # every finite code round-trips


@pytest.mark.parametrize("fmt", ["e4m3", "e5m2"])
def test_scales_and_special_cases(fmt):
    mx = np.float32(fo.FP8_MAX[fmt])
    assert fo.scales(0.0, fmt) == (1.0, 1.0)
    s, si = fo.scales(np.float32(3.0), fmt)
    assert s == mx / np.float32(3.0) and si == np.float32(3.0) / mx
    for bad in (np.inf, np.nan):
        assert np.isnan(fo.scales(bad, fmt)[1])
    x = np.array([1.0, -2.0, np.inf], np.float32)
    q, am, si = fo.quantize(x, fmt)
    assert am == np.inf and np.isnan(si)
    q, am, si = fo.quantize(np.array([1.0, np.nan, -np.inf], np.float32), fmt)
    assert np.isnan(am) and np.isnan(si) and (q == 0x7F).all()
    q, am, si = fo.quantize(np.zeros(5, np.float32), fmt)
    assert am == 0 and si == 1 and (q == 0).all()
    q, am, si = fo.quantize(np.array([-0.0, 0.0, 1e-30, -1.0], np.float32), fmt)
    assert list(q[:2]) == [0x80, 0x00] and q[3] == fo.round_fp8(-mx, fmt)
    q, am, si = fo.quantize(np.array([3.0, -3.0, 1.0], np.float32), fmt)     # the amax element lands on +-max
    assert fo.decode(q[:2], fmt).tolist() == [float(mx), -float(mx)]


def test_weights_transpose_each_block():
    w = np.random.default_rng(0).normal(0, 1, (3, 32, 32)).astype(np.float32)
    wq, wq_t, am, si = fo.quantize_weights(w, "e4m3")
    assert np.array_equal(wq_t, wq.transpose(0, 2, 1)) and am == np.abs(w).max()
    assert np.array_equal(wq, fo.quantize(w, "e4m3")[0])
