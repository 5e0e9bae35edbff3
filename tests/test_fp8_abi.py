"""The fp8 path without a GPU: the C entries are bound, every argument error is refused before any launch with the
documented code, the existing entries keep refusing the fp8 dtype codes, and matmul_fp8 / quantize_fp8 raise on the
configurations they do not take."""
import os
import re

import numpy as np
import pytest
import torch

from tests._util import ROOT
import blocksparse_b200
from blocksparse_b200 import BlocksparseMatMul, _lib, quantize_fp8
from blocksparse_b200.fp8 import quantize_fp8_weights, xprop_fp8

E_DTYPE, E_BSIZE, E_ARG, E_LIMIT, E_ALIGN = -1, -2, -3, -4, -6
E4, E5, F32, F16, BF16 = _lib.E4M3, _lib.E5M2, _lib.F32, _lib.F16, _lib.BF16
FAKE = 0x100000                      # never dereferenced: every call below fails on the host
LUT, X, W, Y, S = FAKE, FAKE + 0x10000, FAKE + 0x20000, FAKE + 0x30000, FAKE + 0x40000


def test_header_dtype_codes():
    src = open(os.path.join(ROOT, "include", "bsmm_b200.h")).read()
    m = re.search(r"enum\s*\{\s*BSMM_E4M3\s*=\s*(\d+),\s*BSMM_E5M2\s*=\s*(\d+)\s*\}", src)
    assert m and (int(m.group(1)), int(m.group(2))) == (3, 4) == (E4, E5)
    for name in ("bsmm_fp8_quantize", "bsmm_fp8_weights", "bsmm_xprop_fp8"):
        assert name in _lib.SIGNATURES


def xprop(**kw):
    a = dict(x=E4, w=E4, y=BF16, axis=1, bs=32, bprop=0, lut=LUT, n_out=4, n_in=4, blocks=4, xp=X, wp=W, yp=Y, N=256,
             xs=S, ws=S + 4)
    a.update(kw)
    lib = _lib.load()
    return lib.bsmm_xprop_fp8(a["x"], a["w"], a["y"], a["axis"], a["bs"], a["bprop"], a["lut"], a["n_out"], a["n_in"],
                              a["blocks"], a["xp"], a["wp"], a["yp"], a["N"], a["xs"], a["ws"], None)


@pytest.mark.parametrize("kw, code", [
    (dict(axis=0), E_BSIZE), (dict(axis=2), E_BSIZE), (dict(bs=8), E_BSIZE), (dict(bs=16), E_BSIZE),
    (dict(bs=128), E_BSIZE),
    (dict(x=BF16), E_DTYPE), (dict(w=F16), E_DTYPE), (dict(x=F32, w=F32, y=F32), E_DTYPE), (dict(y=F32), E_DTYPE),
    (dict(y=E4), E_DTYPE), (dict(x=5), E_DTYPE), (dict(y=E5), E_DTYPE),
    (dict(lut=None), E_ARG), (dict(xp=None), E_ARG), (dict(wp=None), E_ARG), (dict(yp=None), E_ARG),
    (dict(xs=None), E_ARG), (dict(ws=None), E_ARG), (dict(bprop=2), E_ARG),
    (dict(n_out=0), E_ARG), (dict(n_in=-1), E_ARG), (dict(blocks=-1), E_ARG), (dict(N=-1), E_ARG),
    (dict(n_out=65536), E_LIMIT), (dict(n_in=70000), E_LIMIT),
    (dict(xp=X + 8), E_ALIGN), (dict(wp=W + 1), E_ALIGN), (dict(yp=Y + 2), E_ALIGN),
])
def test_xprop_fp8_refuses_before_any_launch(kw, code):
    before = _lib.last_kernel()
    assert xprop(**kw) == code, _lib.device_error_text()
    assert _lib.last_kernel() == before


def test_xprop_fp8_axis_and_block_size_come_before_dtype():
    """The documented order: a bad axis / block size is reported as such even with a bad dtype too."""
    assert xprop(axis=0, x=BF16) == E_BSIZE
    assert xprop(bs=16, y=F32) == E_BSIZE


def test_xprop_fp8_with_no_rows_launches_nothing():
    before = _lib.last_kernel()
    assert xprop(N=0) == 0
    assert _lib.last_kernel() == before


@pytest.mark.parametrize("args, code", [
    ((E4, E4, X, 16, S, S + 4, Y), E_DTYPE), ((F16, F16, X, 16, S, S + 4, Y), E_DTYPE), ((7, E4, X, 16, S, S + 4, Y), E_DTYPE),
    ((F16, 0, X, 16, S, S + 4, Y), E_DTYPE), ((BF16, E5, X, -1, S, S + 4, Y), E_ARG),
    ((BF16, E5, None, 16, S, S + 4, Y), E_ARG), ((BF16, E5, X, 16, None, S + 4, Y), E_ARG),
    ((BF16, E5, X, 16, S, None, Y), E_ARG), ((F32, E4, X, 16, S, S + 4, None), E_ARG),
])
def test_quantize_refuses_before_any_launch(args, code):
    before = _lib.last_kernel()
    assert _lib.load().bsmm_fp8_quantize(*args, None) == code, _lib.device_error_text()
    assert _lib.last_kernel() == before


@pytest.mark.parametrize("args, code", [
    ((F16, E4, 8, 4, W, S, S + 4, X, Y), E_BSIZE), ((F16, E4, 16, 4, W, S, S + 4, X, Y), E_BSIZE),
    ((E4, E4, 32, 4, W, S, S + 4, X, Y), E_DTYPE), ((F16, BF16, 32, 4, W, S, S + 4, X, Y), E_DTYPE),
    ((F16, E4, 32, 0, W, S, S + 4, X, Y), E_ARG), ((F16, E4, 64, 4, None, S, S + 4, X, Y), E_ARG),
    ((F16, E4, 64, 4, W, None, S + 4, X, Y), E_ARG), ((F16, E4, 64, 4, W, S, None, X, Y), E_ARG),
    ((F16, E4, 64, 4, W, S, S + 4, None, Y), E_ARG), ((F16, E4, 64, 4, W, S, S + 4, X, None), E_ARG),
    ((F16, E4, 64, 4, W, S, S + 4, X + 4, Y), E_ALIGN), ((F16, E4, 64, 4, W, S, S + 4, X, Y + 8), E_ALIGN),
])
def test_weights_refuse_before_any_launch(args, code):
    before = _lib.last_kernel()
    assert _lib.load().bsmm_fp8_weights(*args, None) == code, _lib.device_error_text()
    assert _lib.last_kernel() == before


def test_existing_entries_still_refuse_the_fp8_codes():
    """The fp8 codes are new to the three fp8 entries only: the 16-bit entries refuse them as any unknown dtype."""
    lib = _lib.load()
    os.environ["BSMM_QUIET"] = "1"
    for dt in (E4, E5):
        rc = lib.bsmm_xprop(dt, 1, 32, 0, LUT, 4, 4, 4, X, W, Y, 256, None, None, 0, 0, 0, 0, 0, 0, 0, None)
        assert rc == E_DTYPE
        rc = lib.bsmm_dw_matmul_large_n(dt, X, W, Y, 64, 8, 8, S, 0, None)
        assert rc == E_ARG
        rc = lib.bsmm_float_cast(dt, F16, X, Y, 16, None)
        assert rc == E_ARG


def test_dtype_code_is_unchanged_and_fp8_has_its_own():
    with pytest.raises(ValueError, match=r"unsupported dtype torch.float8_e4m3fn \(float32, float16, bfloat16 only\)"):
        _lib.dtype_code(torch.float8_e4m3fn)
    assert _lib.fp8_code(torch.float8_e4m3fn) == E4 and _lib.fp8_code(torch.float8_e5m2) == E5
    with pytest.raises(ValueError):
        _lib.fp8_code(torch.float16)


def test_quantize_fp8_is_exported_outside_all():
    assert blocksparse_b200.quantize_fp8 is quantize_fp8
    assert "quantize_fp8" not in blocksparse_b200.__all__


def layout(n=4):
    return np.ones((n, n), np.int32)


@pytest.mark.parametrize("axis, bs, dtype", [(0, 32, torch.float16), (0, 64, torch.bfloat16), (1, 8, torch.float16),
                                             (1, 16, torch.bfloat16), (1, 32, torch.float32), (1, 64, torch.float32)])
def test_matmul_fp8_refuses_unsupported_configurations(axis, bs, dtype):
    bsmm = BlocksparseMatMul(layout(), block_size=bs, feature_axis=axis)
    I = torch.zeros(bsmm.i_shape(8), dtype=dtype)
    W = torch.zeros(bsmm.w_shape, dtype=dtype)
    with pytest.raises(ValueError):
        bsmm.matmul_fp8(I, W)


def test_matmul_fp8_refuses_mixed_dtypes_and_cpu_tensors():
    bsmm = BlocksparseMatMul(layout(), block_size=32, feature_axis=1)
    I = torch.zeros(bsmm.i_shape(8), dtype=torch.float16)
    with pytest.raises(ValueError):
        bsmm.matmul_fp8(I, torch.zeros(bsmm.w_shape, dtype=torch.bfloat16))
    with pytest.raises(_lib.BsmmError):
        bsmm.matmul_fp8(I, torch.zeros(bsmm.w_shape, dtype=torch.float16))


def test_raw_fp8_calls_refuse_bad_arguments_on_the_host():
    bsmm = BlocksparseMatMul(layout(), block_size=32, feature_axis=1)
    with pytest.raises(ValueError):
        quantize_fp8(torch.zeros(4, dtype=torch.float16), torch.float16)
    with pytest.raises(ValueError):
        quantize_fp8(torch.zeros(4, dtype=torch.int32))
    with pytest.raises(_lib.BsmmError):
        quantize_fp8(torch.zeros(4, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        quantize_fp8_weights(BlocksparseMatMul(layout(), block_size=16, feature_axis=1),
                             torch.zeros((16, 16, 16), dtype=torch.float16))
    xq = torch.zeros((8, bsmm.C), dtype=torch.float8_e4m3fn)
    wq = torch.zeros(bsmm.w_shape, dtype=torch.float8_e4m3fn)
    s = torch.ones(1)
    with pytest.raises(ValueError):
        xprop_fp8(bsmm, xq.to(torch.float16), wq, s, s)
    with pytest.raises(ValueError):
        xprop_fp8(bsmm, xq, wq, s, s, out_dtype=torch.float32)
    with pytest.raises(_lib.BsmmError):
        xprop_fp8(bsmm, xq, wq, s, s)
