"""The fp8 weight gradient without a GPU: bsmm_fp8_quantize_t and bsmm_updat_fp8 are bound and refuse every argument
error before any launch with the documented code, and quantize_fp8_t, updat_fp8 and matmul_fp8(fp8_dw=True) raise on
what they do not take."""
import ctypes

import numpy as np
import pytest
import torch

import blocksparse_b200
from blocksparse_b200 import BlocksparseMatMul, _lib, fp8
from blocksparse_b200.fp8 import quantize_fp8_t, updat_fp8

E_DTYPE, E_BSIZE, E_ARG, E_LIMIT, E_ALIGN = -1, -2, -3, -4, -6
E4, E5, F32, F16, BF16 = _lib.E4M3, _lib.E5M2, _lib.F32, _lib.F16, _lib.BF16
FAKE = 0x100000                      # never dereferenced: every call below fails on the host
X, Y, YT, S, DW, SCHED = FAKE, FAKE + 0x10000, FAKE + 0x20000, FAKE + 0x30000, FAKE + 0x40000, FAKE + 0x50000


def test_entries_are_bound():
    for name in ("bsmm_fp8_quantize_t", "bsmm_updat_fp8"):
        assert name in _lib.SIGNATURES
        assert hasattr(_lib.load(), name)


def quantize_t(**kw):
    a = dict(src=BF16, fmt=E4, x=X, rows=100, cols=33, amax=S, si=S + 4, y=Y, yt=YT, pitch=112)
    a.update(kw)
    return _lib.load().bsmm_fp8_quantize_t(a["src"], a["fmt"], a["x"], a["rows"], a["cols"], a["amax"], a["si"], a["y"],
                                           a["yt"], a["pitch"], None)


@pytest.mark.parametrize("kw, code", [
    (dict(src=E4), E_DTYPE), (dict(src=7), E_DTYPE), (dict(fmt=F16), E_DTYPE), (dict(fmt=0), E_DTYPE),
    (dict(rows=-1), E_ARG), (dict(cols=-1), E_ARG), (dict(amax=None), E_ARG), (dict(si=None), E_ARG),
    (dict(y=None, yt=None), E_ARG), (dict(x=None), E_ARG), (dict(pitch=96), E_ARG), (dict(pitch=-16), E_ARG),
    (dict(pitch=120), E_ALIGN), (dict(pitch=101), E_ALIGN), (dict(yt=YT + 2), E_ALIGN),
])
def test_quantize_t_refuses_before_any_launch(kw, code):
    before = _lib.last_kernel()
    assert quantize_t(**kw) == code, _lib.device_error_text()
    assert _lib.last_kernel() == before


PA = ctypes.c_void_p * 8


def updat(**kw):
    a = dict(x=E4, dy=E5, dw=BF16, bs=32, blocks=12, cb=4, kb=4, xts=[X], dyts=[Y], xs=[S], ds=[S + 4], pcount=None,
             dwp=DW, N=1000, pitch=1008, beta=0.0, sched=SCHED, tiles=3, kt=8)
    a.update(kw)
    n = len(a["xts"] or [X])
    arr = lambda v: None if v is None else PA(*(list(v) + [None] * (8 - len(v))))
    return _lib.load().bsmm_updat_fp8(a["x"], a["dy"], a["dw"], a["bs"], a["blocks"], a["cb"], a["kb"], arr(a["xts"]),
                                      arr(a["dyts"]), arr(a["xs"]), arr(a["ds"]), n if a["pcount"] is None else a["pcount"],
                                      a["dwp"], a["N"], a["pitch"], a["beta"], a["sched"], a["tiles"], a["kt"], None)


@pytest.mark.parametrize("kw, code", [
    (dict(bs=16), E_BSIZE), (dict(bs=8), E_BSIZE), (dict(bs=128), E_BSIZE),
    (dict(x=BF16), E_DTYPE), (dict(dy=F16), E_DTYPE), (dict(x=7), E_DTYPE), (dict(dw=E4), E_DTYPE), (dict(dw=9), E_DTYPE),
    (dict(pcount=0), E_ARG), (dict(pcount=9), E_ARG), (dict(pcount=-1), E_ARG),
    (dict(xts=None), E_ARG), (dict(dyts=None), E_ARG), (dict(xs=None), E_ARG), (dict(ds=None), E_ARG),
    (dict(xts=[None]), E_ARG), (dict(dyts=[None]), E_ARG), (dict(xs=[None]), E_ARG), (dict(ds=[None]), E_ARG),
    (dict(xts=[X, X], dyts=[Y, None], xs=[S, S], ds=[S, S]), E_ARG),
    (dict(dwp=None), E_ARG), (dict(sched=None), E_ARG),
    (dict(N=-1), E_ARG), (dict(pitch=992), E_ARG), (dict(pitch=1012), E_ALIGN), (dict(N=0, pitch=8), E_ALIGN),
    (dict(beta=0.5), E_ARG), (dict(beta=2.0), E_ARG), (dict(beta=-1.0), E_ARG),
    (dict(blocks=0), E_ARG), (dict(tiles=0), E_ARG), (dict(kt=4), E_ARG), (dict(bs=64, kt=8), E_ARG),
    (dict(N=1 << 31, pitch=1 << 31), E_LIMIT),
    (dict(dwp=DW + 8), E_ALIGN), (dict(xts=[X + 4]), E_ALIGN), (dict(dyts=[Y + 1]), E_ALIGN),
])
def test_updat_fp8_refuses_before_any_launch(kw, code):
    before = _lib.last_kernel()
    assert updat(**kw) == code, _lib.device_error_text()
    assert _lib.last_kernel() == before


def test_updat_fp8_block_size_comes_before_dtype():
    assert updat(bs=16, x=BF16) == E_BSIZE


def test_existing_updat_still_refuses_the_fp8_codes():
    lib = _lib.load()
    xp, ep = (ctypes.c_void_p * 1)(X), (ctypes.c_void_p * 1)(Y)
    for dt in (E4, E5):
        rc = lib.bsmm_updat(dt, dt, 1, 32, SCHED, 12, 4, 4, xp, ep, 1, DW, 256, 1.0, 0.0, None, 0, None, 0, 0, 0, 0, None)
        assert rc in (E_DTYPE, E_ARG)
        rc = lib.bsmm_updat(BF16, dt, 1, 32, SCHED, 12, 4, 4, xp, ep, 1, DW, 256, 1.0, 0.0, None, 0, None, 0, 0, 0, 0, None)
        assert rc in (E_DTYPE, E_ARG)


def test_exports():
    for name in ("quantize_fp8_t", "updat_fp8"):
        assert name in fp8.__all__
        assert name not in blocksparse_b200.__all__


def layout(n=4):
    return np.ones((n, n), np.int32)


def test_quantize_fp8_t_refuses_bad_arguments_on_the_host():
    with pytest.raises(ValueError):
        quantize_fp8_t(torch.zeros((4, 4), dtype=torch.float16), torch.float16)
    with pytest.raises(ValueError):
        quantize_fp8_t(torch.zeros((4, 4), dtype=torch.int32))
    with pytest.raises(ValueError):
        quantize_fp8_t(torch.zeros(16, dtype=torch.float16))
    with pytest.raises(ValueError):
        quantize_fp8_t(torch.zeros((2, 4, 4), dtype=torch.float16))
    with pytest.raises(_lib.BsmmError):
        quantize_fp8_t(torch.zeros((4, 4), dtype=torch.bfloat16))


def fp8_operands(bsmm, pitch=16, xdt=torch.float8_e4m3fn, dydt=torch.float8_e5m2):
    return (torch.zeros((bsmm.C, pitch), dtype=xdt), torch.zeros((bsmm.K, pitch), dtype=dydt), torch.ones(1),
            torch.ones(1))


def test_updat_fp8_refuses_bad_arguments_on_the_host():
    bsmm = BlocksparseMatMul(layout(), block_size=32, feature_axis=1)
    xt, dyt, s, t = fp8_operands(bsmm)
    bad = [
        lambda: updat_fp8(BlocksparseMatMul(layout(), block_size=16, feature_axis=1), xt, dyt, s, t, 10),   # block size
        lambda: updat_fp8(BlocksparseMatMul(layout(), block_size=8, feature_axis=0), xt, dyt, s, t, 10),
        lambda: updat_fp8(bsmm, xt.to(torch.float16), dyt, s, t, 10),                                     # dtypes
        lambda: updat_fp8(bsmm, xt, dyt.view(torch.uint8), s, t, 10),
        lambda: updat_fp8(bsmm, [xt, xt.view(torch.float8_e5m2)], [dyt, dyt], [s, s], [t, t], 10),
        lambda: updat_fp8(bsmm, xt, dyt, s.double(), t, 10),
        lambda: updat_fp8(bsmm, xt, dyt, s, torch.ones(0), 10),
        lambda: updat_fp8(bsmm, xt, dyt, s, t, 10, dw_dtype=torch.float8_e4m3fn),
        lambda: updat_fp8(bsmm, xt, dyt, s, t, 10, dw=torch.zeros(bsmm.w_shape, dtype=torch.int32)),
        lambda: updat_fp8(bsmm, xt, dyt, s, t, 10, dw=torch.zeros((1, 32, 32))),                         # shapes
        lambda: updat_fp8(bsmm, xt[:-32], dyt, s, t, 10),
        lambda: updat_fp8(bsmm, xt, dyt[:, :8], s, t, 8),
        lambda: updat_fp8(bsmm, xt, torch.zeros((bsmm.K, 32), dtype=torch.float8_e5m2), s, t, 10),
        lambda: updat_fp8(bsmm, xt.t(), dyt, s, t, 10),
        lambda: updat_fp8(bsmm, xt[0], dyt, s, t, 10),
        lambda: updat_fp8(bsmm, xt, dyt, s, t, 17),                                                      # pitches
        lambda: updat_fp8(bsmm, xt, dyt, s, t, -1),
        lambda: updat_fp8(bsmm, *fp8_operands(bsmm, pitch=24), 10),
        lambda: updat_fp8(bsmm, [], [], [], [], 10),                                                     # pair counts
        lambda: updat_fp8(bsmm, [xt] * 9, [dyt] * 9, [s] * 9, [t] * 9, 10),
        lambda: updat_fp8(bsmm, [xt, xt], [dyt], [s, s], [t, t], 10),
        lambda: updat_fp8(bsmm, [xt, xt], [dyt, dyt], [s], [t, t], 10),
    ]
    for call in bad:
        with pytest.raises(ValueError):
            call()
    with pytest.raises(_lib.BsmmError):
        updat_fp8(bsmm, xt, dyt, s, t, 10)


@pytest.mark.parametrize("axis, bs, dtype", [(0, 32, torch.float16), (0, 64, torch.bfloat16), (1, 8, torch.float16),
                                             (1, 16, torch.bfloat16), (1, 32, torch.float32), (1, 64, torch.float32)])
def test_matmul_fp8_dw_refuses_unsupported_configurations(axis, bs, dtype):
    bsmm = BlocksparseMatMul(layout(), block_size=bs, feature_axis=axis)
    I = torch.zeros(bsmm.i_shape(8), dtype=dtype)
    W = torch.zeros(bsmm.w_shape, dtype=dtype)
    with pytest.raises(ValueError):
        bsmm.matmul_fp8(I, W, fp8_dw=True)


def test_matmul_fp8_dw_refuses_mixed_dtypes_and_cpu_tensors():
    bsmm = BlocksparseMatMul(layout(), block_size=32, feature_axis=1)
    I = torch.zeros(bsmm.i_shape(8), dtype=torch.float16)
    with pytest.raises(ValueError):
        bsmm.matmul_fp8(I, torch.zeros(bsmm.w_shape, dtype=torch.bfloat16), fp8_dw=True)
    with pytest.raises(_lib.BsmmError):
        bsmm.matmul_fp8(I, torch.zeros(bsmm.w_shape, dtype=torch.float16), fp8_dw=True)
