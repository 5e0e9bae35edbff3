"""Block-sparse conv fprop, bprop and updat on activations past 2^31 elements, on the wgmma and the FMA route.

1 x 1 taps and thin, overlapping blocks keep the work small, while N * C * W passes 2^31, so element offsets of the
input, the output, the fp32 pass accumulator and the updat's rows part ways with 32-bit arithmetic. The overlap runs
fprop and bprop as two passes, and updat reduces N * W / 8192, about 33 thousand, chunks. Each output starts as NaN
and is scanned whole for NaN. fprop / bprop are checked against float64 on sampled images: the first, the last, both
sides of offset 2^31, and seeded random ones. dF is checked whole against a float64 sum formed on the device."""
import numpy as np
import pytest
import torch

from blocksparse_b200 import _lib
from blocksparse_b200.conv import BlocksparseConv
from tests._util import _on_poisoned_output
from tests.test_conv_gpu import assert_close
from tests.test_large_offsets_gpu import _need, _no_nan, sample_ids

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
C = K = 8
W = 16384
N = 2 ** 31 // (C * W) + 8                  # N * C * W = 2^31 + 2^20
BCK = [[[0, 1, 2, 3, 4], [0, 1, 2, 3]], [[3, 4, 5, 6, 7], [2, 3, 4, 5, 6, 7]]]


def _dense(op, F):
    """The 1 x 1 conv as a dense (K, C) float64 matrix: blocks that share a (k, c) add."""
    D = np.zeros((op.K, op.C))
    off = 0
    for lc, lk in op.BCK:
        n = len(lc) * len(lk)
        D[np.ix_(lk, lc)] += F[off:off + n].reshape(len(lk), len(lc))
        off += n
    return D


def _rows64(t, ids):
    return t[ids].double().cpu().numpy()


@pytest.mark.parametrize("flags", [0, _lib.FLAG_FORCE_GENERIC], ids=["wgmma", "fma"])
def test_conv_past_2_31(flags):
    _need(30, "a bf16 conv of 2^31 + 2^20 elements with its fp32 pass accumulator")
    op = BlocksparseConv(BCK, (1,), (W,), padding="VALID")
    assert op.overlapC and op.overlapK
    g = torch.Generator(device="cuda").manual_seed(5)
    F = (torch.rand(op.sizeF, device="cuda", generator=g) * 2 - 1).to(BF16)
    x = (torch.rand((N, C, W), device="cuda", generator=g) * 2 - 1).to(BF16)
    assert x.numel() > 2 ** 31
    Fn = F.double().cpu().numpy()
    D = _dense(op, Fn)
    Da = _dense(op, np.abs(Fn))
    ids = sample_ids(N, 2 ** 31 // (C * W), np.random.default_rng(1))
    tc = not flags
    kernel = "wgmma" if tc else "fma"

    y = _on_poisoned_output(lambda: op._xprop(F, x, False, flags=flags))
    assert _lib.last_kernel() == kernel + "_conv_xprop"
    _no_nan(y, "fprop")
    xs = _rows64(x, ids)
    assert_close(y[ids], np.einsum("kc,ncw->nkw", D, xs), np.einsum("kc,ncw->nkw", Da, np.abs(xs)), C, BF16, tc,
                 "fprop")
    del y

    e = (torch.rand((N, K, W), device="cuda", generator=g) * 2 - 1).to(BF16)
    dx = _on_poisoned_output(lambda: op._xprop(F, e, True, flags=flags))
    _no_nan(dx, "bprop")
    es = _rows64(e, ids)
    assert_close(dx[ids], np.einsum("kc,nkw->ncw", D, es), np.einsum("kc,nkw->ncw", Da, np.abs(es)), K, BF16, tc,
                 "bprop")
    del dx

    df = _on_poisoned_output(lambda: op._updat(e, x, BF16, flags=flags))
    assert _lib.last_kernel() == kernel + "_conv_updat"
    _no_nan(df, "updat")
    # float64 (K, C) sums over every image and position, formed on the device in slices
    S, Sa = torch.zeros((K, C), dtype=torch.float64, device="cuda"), torch.zeros((K, C), dtype=torch.float64, device="cuda")
    for i in range(0, N, 1024):
        eb, xb = e[i:i + 1024].double(), x[i:i + 1024].double()
        S += torch.einsum("nkw,ncw->kc", eb, xb)
        Sa += torch.einsum("nkw,ncw->kc", eb.abs(), xb.abs())
    S, Sa = S.cpu().numpy(), Sa.cpu().numpy()
    ref = np.concatenate([S[np.ix_(lk, lc)].ravel() for lc, lk in op.BCK])
    mag = np.concatenate([Sa[np.ix_(lk, lc)].ravel() for lc, lk in op.BCK])
    assert_close(df, ref, mag, N * W // 8192 + 8192, BF16, tc, "updat")
