"""dw_matmul_large_n without a GPU: the C entries are bound, every argument error is refused before a launch, and the
workspace query follows the documented split rule, stays under its bound and does not depend on BSMM_SM_MARGIN."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from tests._util import ROOT
from blocksparse_b200 import _lib, dw_matmul_large_n

E_ARG = -3
FAKE = 0x10000                       # never dereferenced: every call below fails on the host
WS_BOUND = 264 * 128 * 256 * 4       # DESIGN.md: TARGET items x one 128 x 256 fp32 tile
F32, F16, BF16 = _lib.F32, _lib.F16, _lib.BF16


def split(N, C, K, tc):
    """The split rule as DESIGN.md states it: S = max(1, min(264 // tiles, N // 1024)), evened out over 64-row stages.
    Returns (S, rows per segment)."""
    tm, tn = (128, 256) if tc else (64, 64)
    tiles = -(-C // tm) * -(-K // tn)
    stages = -(-N // 64)
    s0 = max(1, min(264 // tiles, N // 1024))
    seg = -(-stages // s0)
    return (-(-stages // seg), 64 * seg) if seg else (1, 0)


def expected_ws(dt, N, C, K):
    ws = lambda tc: (lambda S: S * C * K * 4 if S > 1 else 0)(split(N, C, K, tc)[0])
    fma = ws(False)
    if dt != F32 and C % 8 == 0 and K % 8 == 0 and N < 2 ** 31:
        return max(fma, ws(True))
    return fma


def test_symbols_are_bound():
    lib = _lib.load()
    for name in ("bsmm_dw_matmul_large_n", "bsmm_dw_matmul_large_n_workspace_bytes"):
        assert name in _lib.SIGNATURES
        assert hasattr(ctypes.CDLL(_lib.LIB_PATH), name)
        assert getattr(lib, name).argtypes is not None


@pytest.mark.parametrize("args,what", [
    ((F16, FAKE, FAKE, FAKE, -1, 8, 8, None, 0), b"negative size"),
    ((F16, FAKE, FAKE, FAKE, 64, -8, 8, None, 0), b"negative size"),
    ((F32, FAKE, FAKE, FAKE, 64, 8, -1, None, 0), b"negative size"),
    ((7, FAKE, FAKE, FAKE, 64, 8, 8, None, 0), b"bad dtype"),
    ((F32, FAKE, FAKE, FAKE, 64, 8, 8, None, _lib.FLAG_FORCE_TC), b"fp32"),
    ((F16, FAKE, FAKE, FAKE, 64, 12, 8, None, _lib.FLAG_FORCE_TC), b"C % 8 == 0"),
    ((BF16, FAKE, FAKE, FAKE, 64, 8, 33, None, _lib.FLAG_FORCE_TC), b"C % 8 == 0"),
    ((F16, FAKE, FAKE, FAKE, 64, 8, 8, None, _lib.FLAG_FORCE_TC | _lib.FLAG_FORCE_GENERIC), b"contradictory"),
    ((F32, FAKE, FAKE, None, 64, 8, 8, None, 0), b"null u"),
    ((F32, None, FAKE, FAKE, 64, 8, 8, None, 0), b"null x"),
    ((F16, FAKE, None, FAKE, 64, 8, 8, None, _lib.FLAG_FORCE_GENERIC), b"null x"),
    ((F32, FAKE, FAKE, FAKE, 1 << 20, 32, 32, None, 0), b"null workspace"),
])
def test_c_argument_errors_before_any_launch(args, what):
    lib = _lib.load()
    before = _lib.last_kernel()
    rc = lib.bsmm_dw_matmul_large_n(*args, None)
    assert rc == E_ARG, (rc, lib.bsmm_last_error())
    assert what in lib.bsmm_last_error(), lib.bsmm_last_error()
    assert _lib.last_kernel() == before
    with pytest.raises(ValueError):
        _lib.check(rc, "bsmm_dw_matmul_large_n")


def test_empty_outputs_launch_nothing():
    lib = _lib.load()
    before = _lib.last_kernel()
    for C, K in ((0, 8), (8, 0), (0, 0)):
        assert lib.bsmm_dw_matmul_large_n(F16, None, None, None, 1 << 20, C, K, None, 0, None) == 0
    assert _lib.last_kernel() == before


@pytest.mark.parametrize("x,e,what", [
    (torch.zeros(4, 8), torch.zeros(4, 8, dtype=torch.float16), "x is"),
    (torch.zeros(4, 8, dtype=torch.int32), torch.zeros(4, 8, dtype=torch.int32), "float32, float16 or bfloat16"),
    (torch.zeros(4, 8, dtype=torch.int64), torch.zeros(4, 8, dtype=torch.int64), "float32, float16 or bfloat16"),
    (torch.zeros(4, 8), torch.zeros(5, 8), "same leading dims"),
    (torch.zeros(2, 4, 8), torch.zeros(8, 8), "one rank"),
    (torch.zeros(2, 4, 8), torch.zeros(4, 2, 8), "same leading dims"),
    (torch.zeros(()), torch.zeros(()), "one rank"),
    (torch.zeros(4, 8), torch.zeros(4, 3), "CUDA tensors"),
    (torch.zeros(4, 8).numpy(), torch.zeros(4, 8), "two tensors"),
])
def test_python_argument_errors(x, e, what):
    with pytest.raises(ValueError, match=what):
        dw_matmul_large_n(x, e)


SWEEP = [(n, c, k) for n in (0, 1, 63, 1000, 1024, 2047, 4096, 65536, 1 << 20, 2 ** 31 - 64)
         for c, k in ((1, 1), (7, 33), (32, 32), (128, 128), (129, 300), (512, 512), (1024, 1024), (4096, 4096),
                      (8192, 64), (64, 16384))]


def test_workspace_follows_the_split_rule_and_bound():
    lib = _lib.load()
    for dt in (F32, F16, BF16):
        for N, C, K in SWEEP:
            got = lib.bsmm_dw_matmul_large_n_workspace_bytes(dt, N, C, K)
            assert got == expected_ws(dt, N, C, K), (dt, N, C, K, got)
            assert got <= WS_BOUND, (dt, N, C, K, got)
    assert lib.bsmm_dw_matmul_large_n_workspace_bytes(F16, 4096, 4096, 4096) == 0      # 512 tiles: S == 1
    assert lib.bsmm_dw_matmul_large_n_workspace_bytes(F32, 2047, 32, 32) == 0          # shorter than two segments
    assert lib.bsmm_dw_matmul_large_n_workspace_bytes(F16, 1 << 20, 32, 32) > 0
    for bad in ((F16, -1, 8, 8), (F16, 64, 0, 8), (F16, 64, 8, -3), (9, 64, 8, 8)):
        assert lib.bsmm_dw_matmul_large_n_workspace_bytes(*bad) == 0


def test_split_bounds_items_and_segment_length():
    for N, C, K in SWEEP:
        for tc in (False, True):
            S, rows = split(N, C, K, tc)
            tm, tn = (128, 256) if tc else (64, 64)
            tiles = -(-C // tm) * -(-K // tn)
            assert S == 1 or (tiles * S <= 264 and rows >= 1024 and (S - 1) * rows < N <= S * rows), (N, C, K, tc, S)


def _child_ws(margin):
    code = ("import sys; sys.path.insert(0, %r)\n"
            "from blocksparse_b200 import _lib\n"
            "from tests.test_dw_matmul_abi import SWEEP\n"
            "lib = _lib.load()\n"
            "print([lib.bsmm_dw_matmul_large_n_workspace_bytes(dt, *s) for dt in (0, 1, 2) for s in SWEEP])\n" % ROOT)
    env = dict(os.environ, BSMM_SM_MARGIN=str(margin))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stdout.strip()


def test_workspace_does_not_depend_on_the_sm_margin():
    assert _child_ws(0) == _child_ws(12) == _child_ws(100)
