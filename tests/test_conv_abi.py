"""Block-sparse conv host side without a GPU: signatures and defaults (pinned, the reference's conv.py:242, 730), every
ValueError of the constructors and calls, the C entries' argument errors, and the spatial tables against a brute-force
loop over positions and taps."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

from blocksparse_b200 import _lib, conv
from blocksparse_b200.conv import BlocksparseConv, BlocksparseDeconv

DIAG = [[list(range(b * 4, b * 4 + 4)), list(range(b * 6, b * 6 + 6))] for b in range(3)]


def test_signatures():
    assert str(inspect.signature(BlocksparseConv.__init__)) == (
        "(self, BCK, TRS, DHW, MPQ=None, strides=(1, 1, 1), dilates=(1, 1, 1), padding='SAME', debug=False, "
        "deconv=False)")
    assert str(inspect.signature(BlocksparseDeconv.__init__)) == (
        "(self, BCK, TRS, DHW, MPQ=None, strides=(1, 1, 1), dilates=(1, 1, 1), padding='SAME', debug=False)")
    assert str(inspect.signature(BlocksparseConv.l2_normalize)) == "(self, F, gain=None, epsilon=1e-12, dtype=None)"
    assert str(inspect.signature(BlocksparseConv.collapse_filter)) == "(self, F, dtype=None)"
    assert conv.__all__ == ["BlocksparseConv", "BlocksparseDeconv"]
    import blocksparse_b200
    assert blocksparse_b200.BlocksparseConv is BlocksparseConv and "BlocksparseConv" not in blocksparse_b200.__all__


@pytest.mark.parametrize("kw", [
    dict(BCK=DIAG, TRS=(3, 3), DHW=(8,)),                                   # rank mismatch
    dict(BCK=DIAG, TRS=(3, 3, 3, 3), DHW=(8, 8, 8, 8)),                     # 4 dims
    dict(BCK=DIAG, TRS=(0,), DHW=(8,)),                                     # empty filter
    dict(BCK=DIAG, TRS=(3,), DHW=(8,), padding="FULL"),
    dict(BCK=DIAG, TRS=(9,), DHW=(4,), padding="VALID"),                    # empty output
    dict(BCK=[], TRS=(3,), DHW=(8,)),
    dict(BCK=[[[0, 1], [0]], [[3], [1]]], TRS=(3,), DHW=(8,)),             # C list misses channel 2
    dict(BCK=[[[0, 1], [0, 2]]], TRS=(3,), DHW=(8,)),                      # K list misses channel 1
    dict(BCK=[[[0, 0], [0]]], TRS=(3,), DHW=(8,)),                         # repeated channel in a block
    dict(BCK=[[[-1], [0]]], TRS=(3,), DHW=(8,)),
    dict(BCK=[[[], [0]]], TRS=(3,), DHW=(8,)),
    dict(BCK=[[[0], [0]]], TRS=(3,), DHW=(8,), strides=(0,)),
])
def test_constructor_errors(kw):
    with pytest.raises(ValueError):
        BlocksparseConv(**kw)


def test_call_errors_before_any_launch():
    op = BlocksparseConv(DIAG, (3,), (8,))
    F, I = torch.zeros(op.f_shape()), torch.zeros(op.i_shape(2))
    with pytest.raises(ValueError):
        op(F, I)                                            # CPU tensors
    with pytest.raises(ValueError):
        op.l2_normalize(F)
    over = BlocksparseConv([[[0, 1], [0, 1]], [[1, 2], [1, 2]]], (3,), (8,))
    assert over.overlapK and over.overlapC


def test_c_abi_argument_errors():
    lib = _lib.load()
    null = None
    one = (ctypes.c_int * 2)(0, 1)
    fake = 16
    E_ARG, E_LIMIT = -3, -4
    args = [0, 0, fake, one, 1, 4, fake, fake, 3, fake, fake, fake, null, 2, 12, 8, 18, 8, 0, null]
    bad = list(args); bad[2] = null
    assert lib.bsmm_conv_xprop(*bad) == E_ARG
    bad = list(args); bad[0], bad[1] = 1, 2                  # fp16 with bf16
    assert lib.bsmm_conv_xprop(*bad) == E_ARG
    bad = list(args); bad[4] = 0
    assert lib.bsmm_conv_xprop(*bad) == E_ARG
    two = (ctypes.c_int * 3)(0, 1, 2)
    bad = list(args); bad[3], bad[4], bad[0], bad[1] = two, 2, 2, 2   # 16-bit y, two passes, no accumulator
    assert lib.bsmm_conv_xprop(*bad) == E_ARG
    bad = list(args); bad[13], bad[17] = 2 ** 30, 2 ** 7      # N * P_out = 2^37 rows: 64-row tiles past grid.x
    assert lib.bsmm_conv_xprop(*bad) == E_LIMIT
    bad = list(args); bad[17] = 2 ** 31                      # P_out * trs past int32
    assert lib.bsmm_conv_xprop(*bad) == E_LIMIT
    uargs = [0, 0, 0, fake, 1, 4, 4, fake, fake, 3, fake, fake, fake, fake, 2, 12, 8, 18, 8, 96, 0, null]
    bad = list(uargs); bad[13] = null
    assert lib.bsmm_conv_updat(*bad) == E_ARG
    bad = list(uargs); bad[14], bad[18] = 2 ** 20, 2 ** 19   # more than 65535 chunks
    assert lib.bsmm_conv_updat(*bad) == E_LIMIT
    bad = list(uargs); bad[19] = 2 ** 31
    assert lib.bsmm_conv_updat(*bad) == E_LIMIT
    assert lib.bsmm_conv_updat_workspace_bytes(8193, 10) == 2 * 10 * 4
    assert lib.bsmm_conv_l2_normalize(0, 1, fake, 1, 3, fake, null, fake, fake, 1e-12, null) == E_ARG
    assert lib.bsmm_conv_l2_normalize(0, 0, null, 1, 3, fake, null, fake, fake, 1e-12, null) == E_ARG
    assert lib.bsmm_conv_l2_normalize_grad(1, 2, fake, 1, 3, fake, fake, null, fake, fake, null, 1e-12, null) == E_ARG
    assert lib.bsmm_conv_l2_normalize_grad(0, 0, fake, 0, 3, fake, fake, null, fake, fake, null, 1e-12, null) == E_ARG


def brute_fprop(TRS, DHW, MPQ, pad, st, dl):
    out = np.full((int(np.prod(MPQ)), int(np.prod(TRS))), -1)
    for o, (m, p, q) in enumerate(np.ndindex(*MPQ)):
        for t, (a, b, c) in enumerate(np.ndindex(*TRS)):
            x = [o_ * s_ - p_ + f_ * d_ for o_, s_, p_, f_, d_ in zip((m, p, q), st, pad, (a, b, c), dl)]
            if all(0 <= xi < X for xi, X in zip(x, DHW)):
                out[o, t] = (x[0] * DHW[1] + x[1]) * DHW[2] + x[2]
    return out


@pytest.mark.parametrize("TRS,DHW,strides,dilates,padding", [
    ((3,), (17,), (2,), (1,), "SAME"), ((5,), (16,), (1,), (2,), "SAME"), ((3, 3), (7, 6), (1, 2), (1, 1), "VALID"),
    ((2, 3), (6, 5), (2, 1), (1, 2), (1, 2)), ((3, 3, 3), (4, 5, 3), (1, 1, 2), (1, 1, 1), "SAME")])
def test_spatial_tables_brute_force(TRS, DHW, strides, dilates, padding):
    op = BlocksparseConv(DIAG, TRS, DHW, strides=strides, dilates=dilates, padding=padding)
    f = brute_fprop(op.TRS, op.DHW, op.MPQ, op.padding, op.strides, op.dilates)
    np.testing.assert_array_equal(op._lut_f, f)
    # bprop: input position i receives tap t from output o exactly when the fprop table says o reads i through t
    b = np.full((int(np.prod(op.DHW)), op.trs), -1)
    for o, t in zip(*np.nonzero(f >= 0)):
        b[f[o, t], t] = o
    np.testing.assert_array_equal(op._lut_b, b)
    from oracle import conv_oracle
    for i in range(3):      # against the reference's per-dim bprop_lut, whose taps are flipped and holes -2
        fd = (op.TRS[i], op.padding[i], op.strides[i], op.dilates[i])
        for x in range(op.DHW[i]):
            ref = conv_oracle.bprop_lut(x, op.MPQ[i], *fd)[::-1]
            q = np.arange(op.TRS[i])
            mine = (x + op.padding[i] - q * op.dilates[i])
            ok = (mine % op.strides[i] == 0) & (mine >= 0) & (mine // op.strides[i] < op.MPQ[i])
            assert [r if r >= 0 else -1 for r in ref] == np.where(ok, mine // op.strides[i], -1).tolist()


def test_passes_keep_block_order_per_channel():
    order, offs = conv._passes([[0, 1], [2], [1, 2], [3], [0]])
    assert offs == [0, 3, 5] and order == [0, 1, 3, 2, 4]
