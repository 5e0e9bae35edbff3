"""The C-ABI shared library loads and exports every symbol include/bsmm_b200.h declares (no GPU needed)."""
import ctypes
import os
import re

import pytest

from tests._util import ROOT
from blocksparse_b200 import _lib

HEADER = os.path.join(ROOT, "include", "bsmm_b200.h")


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b((?:bsmm|bst)_[a-z_0-9]+)\s*\(", src)))


def test_header_declares_expected_entry_points():
    syms = declared_symbols()
    for must in ["bsmm_xprop", "bsmm_updat", "bst_nt", "bst_xn", "bst_softmax", "bst_softmax_grad",
                 "bst_autoregressive_mask", "bsmm_gate_grad", "bsmm_last_error"]:
        assert must in syms


def test_library_exports_every_declared_symbol():
    assert os.path.exists(_lib.LIB_PATH), "build first: python -c 'import __graft_entry__ as g; g.build()'"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for s in declared_symbols():
        assert hasattr(lib, s), "missing export %s" % s


def test_binding_covers_every_declared_symbol():
    assert sorted(_lib.SIGNATURES) == declared_symbols()
    lib = _lib.load()
    assert lib.bsmm_version() >= 1
    assert lib.bsmm_last_error() is not None


def test_argument_errors_are_reported_without_a_gpu():
    lib = _lib.load()
    # block size 12 is rejected before anything touches the device
    rc = lib.bsmm_xprop(_lib.F32, 0, 12, 0, None, 1, 1, 1, None, None, None, 4, None, None, 0, 0, 0, 0, 0, 0, 0, None)
    assert rc == -2 and b"block size" in lib.bsmm_last_error()
    rc = lib.bsmm_xprop(_lib.F32, 0, 32, 0, None, 1, 1, 1, None, None, None, 4, None, None, 0, 0, 0, 0, 0, 0, 0, None)
    assert rc == -3
    with pytest.raises(ValueError):
        _lib.check(rc, "bsmm_xprop")


def test_softmax_refuses_misaligned_pointers_before_any_launch():
    """Both softmax kernels load 16-byte vectors, so any operand that does not start on a 16-byte boundary is refused
    on the host. The pointers below are never dereferenced: the call must fail before touching the device."""
    lib = _lib.load()
    before = _lib.last_kernel()
    lut, a, b, c = 0x1000, 0x10000, 0x20000, 0x30000
    for dt, x, y in [(_lib.BF16, a + 2, b), (_lib.F16, a, b + 2), (_lib.F32, a + 8, b), (_lib.BF16, a + 14, b + 6)]:
        rc = lib.bst_softmax(dt, dt, 64, lut, None, 1, 4, 2, None, 1, -1, x, y, 1.0, 1, 1, 2, None)
        assert rc == -3 and b"16-byte aligned" in lib.bsmm_last_error(), (rc, lib.bsmm_last_error())
    for dt, dy, y, dx in [(_lib.BF16, a + 2, b, c), (_lib.F16, a, b + 4, c), (_lib.F32, a, b, c + 8), (_lib.F16, a + 1, b, c)]:
        rc = lib.bst_softmax_grad(dt, dt, 32, lut, 1, 4, 2, dy, y, dx, 1.0, 1, 1, 2, None)
        assert rc == -3 and b"16-byte aligned" in lib.bsmm_last_error(), (rc, lib.bsmm_last_error())
    assert _lib.last_kernel() == before          # nothing was launched
