"""The float64 conv oracle (oracle/conv_oracle.py) and the package's host side against fixtures recorded from the
reference's own blocksparse/conv.py (tests/golden/make_golden_conv.py): shapes, padding, the l2 row table, and the
fprop / bprop / updat / l2 checkers on the fixtures' inputs."""
import os
import sys

import numpy as np
import pytest

from tests._util import GOLDEN, golden_files

sys.path.insert(0, GOLDEN)
from make_golden_conv import hash_values  # noqa: E402
from oracle import conv_oracle  # noqa: E402
from blocksparse_b200.conv import BlocksparseConv, BlocksparseDeconv  # noqa: E402

FILES = golden_files("conv_")


def load(name):
    z = np.load(os.path.join(GOLDEN, name))
    cs, ks = np.cumsum(np.r_[0, z["c_sizes"]]), np.cumsum(np.r_[0, z["k_sizes"]])
    BCK = [[z["c_lists"][cs[b]:cs[b + 1]].tolist(), z["k_lists"][ks[b]:ks[b + 1]].tolist()]
           for b in range(len(z["c_sizes"]))]
    pad = str(z["padding_spec"])
    kw = dict(strides=tuple(z["strides"]), dilates=tuple(z["dilates"]), padding=pad)
    return z, BCK, kw


def inputs(z, orc):
    N = int(z["N"])
    F = orc.split_filter(hash_values(int(z["sizeF"]), 1))
    U = orc.split_filter(hash_values(int(z["sizeF"]), 2))
    I = hash_values(int(np.prod(z["i_shape"])), 3).reshape(z["i_shape"]).astype(np.float64)
    E = hash_values(int(np.prod(z["o_shape"])), 4).reshape(z["o_shape"]).astype(np.float64)
    G = hash_values(int(z["C"] if str(z["kind"]) == "deconv" else z["K"]), 5).astype(np.float64)
    return N, F, U, I, E, G


def check(z, key, got):
    """fprop / bprop are float64 in the reference; updat and the l2 results come back rounded to float32."""
    ref = z[key]
    tol = 1e-9 if key in ("fprop", "bprop") else 2 ** -22
    np.testing.assert_allclose(np.asarray(got, dtype=np.float64).ravel()[z[key + "_idx"]], ref,
                               rtol=tol, atol=tol * max(1.0, np.abs(ref).max()), err_msg=key)


@pytest.mark.parametrize("name", FILES)
def test_oracle_matches_reference(name):
    z, BCK, kw = load(name)
    orc = conv_oracle.Conv(BCK, tuple(z["TRS"]), tuple(z["DHW"]), deconv=str(z["kind"]) == "deconv", **kw)
    assert orc.C == z["C"] and orc.K == z["K"] and orc.sizeF == z["sizeF"]
    assert list(orc.MPQ) == list(z["MPQ"]) and list(orc.padding) == list(z["padding"])
    assert orc.f_shape() == list(z["f_shape"])
    N, F, U, I, E, G = inputs(z, orc)
    check(z, "fprop", orc.fprop(F, I))
    check(z, "bprop", orc.bprop(F, E))
    check(z, "updat", orc.updat(E, I))
    check(z, "l2", orc.l2_normalize(F))
    check(z, "l2_grad", orc.l2_normalize_grad(F, U)[0])
    if "l2_gain" in z:
        check(z, "l2_gain", orc.l2_normalize(F, gain=G))
        d, dg = orc.l2_normalize_grad(F, U, gain=G)
        check(z, "l2_gain_grad", d)
        check(z, "l2_gain_dg", dg)


@pytest.mark.parametrize("name", FILES)
def test_package_host_side_matches_reference(name):
    z, BCK, kw = load(name)
    deconv = str(z["kind"]) == "deconv"
    cls = BlocksparseDeconv if deconv else BlocksparseConv
    op = cls(BCK, tuple(z["TRS"]), tuple(z["DHW"]), **kw)
    for attr in ("C", "K", "sizeF", "overlapC", "overlapK", "flops"):
        assert getattr(op, attr) == z[attr], attr
    assert list(op.MPQ) == list(z["MPQ"]) and list(op.padding) == list(z["padding"])
    assert op.i_shape(int(z["N"])) == list(z["i_shape"]) and op.o_shape(int(z["N"])) == list(z["o_shape"])
    assert op.f_shape() == list(z["f_shape"])
    # the reference's norm_lut: (offset, CTRS) per output channel, or (c, KTRS, CTRS, offset) per input channel
    nl = z["norm_lut"]
    if deconv:
        expect = np.stack([nl[:, 3] + nl[:, 0] * op.trs, nl[:, 1] // op.trs, nl[:, 2]], axis=1)
    else:
        expect = np.stack([nl[:, 0], nl[:, 1] // op.trs, np.full(len(nl), op.trs)], axis=1)
    np.testing.assert_array_equal(op._norm[:, :3], expect)
    # the checkers (API surface) on per-block filter lists
    orc = conv_oracle.Conv(BCK, tuple(z["TRS"]), tuple(z["DHW"]), deconv=deconv, **kw)
    N, F, U, I, E, G = inputs(z, orc)
    Fb = [f.reshape(op.f_shape(b)) for b, f in enumerate(F)]
    Ub = [u.reshape(op.f_shape(b)) for b, u in enumerate(U)]
    check(z, "fprop", op.fprop_test(Fb, I))
    check(z, "bprop", op.bprop_test(Fb, E))
    check(z, "updat", op.updat_test(E, I))
    check(z, "l2", op.l2_normalize_test(Fb))
    check(z, "l2_grad", op.l2_normalize_grad_test(Fb, Ub)[0])
    if "l2_gain" in z:
        check(z, "l2_gain", op.l2_normalize_test(Fb, gain=G))
        d, dg = op.l2_normalize_grad_test(Fb, Ub, gain=G)
        check(z, "l2_gain_grad", d)
        check(z, "l2_gain_dg", dg)
    np.testing.assert_array_equal(op.collapse_filter(Fb, np.float64), orc.collapse_filter(F))
