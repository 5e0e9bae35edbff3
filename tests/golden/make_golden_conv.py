"""Generate the block-sparse conv fixtures (conv_*.npz) from the REFERENCE implementation.

Needs a checkout of openai/blocksparse (the tests only read the committed .npz files):

    BLOCKSPARSE_REFERENCE=/path/to/blocksparse python tests/golden/make_golden_conv.py

The reference's blocksparse/conv.py is imported with TensorFlow mocked, as make_golden.py does; everything recorded is
computed by its own Python / NumPy code: the output shape and padding its __init__ resolves, norm_lut (through the
arguments it hands to tf.constant), and fprop_test / bprop_test / updat_test / l2_normalize_test /
l2_normalize_grad_test on seeded inputs. Configs: the nine of test/blocksparse_conv_test.py:45-55, plus one with
non-uniform block sizes and randomly permuted channel lists.

To keep the files small the inputs are not stored: hash_values() derives them from (size, salt), and the tests derive
them the same way. Each output is stored at up to 1024 positions (`<name>_idx`, `<name>`), the whole of it when smaller.
"""
import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, import_reference  # noqa: E402


def hash_values(n, salt):
    """n float32 values in [-1, 1) on a 1/128 grid: the top byte of a multiplicative hash of (index, salt)."""
    h = ((np.arange(n, dtype=np.uint64) + np.uint64(salt * 1000003)) * np.uint64(2654435761)) % np.uint64(2 ** 32)
    return ((h >> np.uint64(24)).astype(np.int64) - 128).astype(np.float32) / 128


def sample(a, salt):
    a = np.asarray(a, dtype=np.float64).ravel()
    if a.size <= 1024:
        return np.arange(a.size, dtype=np.int64), a
    idx = np.unique((np.arange(4096, dtype=np.int64) * 2654435761 + salt) % a.size)[:1024]
    return idx, a[idx]


def import_conv():
    import_reference()
    return importlib.import_module("blocksparse.conv")


def layouts(rng):
    diag = [[[b * 32 + c for c in range(32)], [b * 48 + k for k in range(48)]] for b in range(4)]
    over = [[[b * 8 + c for c in range(16)], [b * 16 + k for k in range(32)]] for b in range(8)]
    # non-uniform sizes, channel lists permuted at random, overlapping in C and K
    cp, kp = rng.permutation(40), rng.permutation(36)
    rand = [[cp[0:12].tolist(), kp[0:8].tolist()], [cp[10:40].tolist(), kp[8:36].tolist()],
            [cp[5:21].tolist(), kp[3:19].tolist()]]
    return diag, over, rand


def configs(rng):
    diag, over, rand = layouts(rng)
    return [
        ("cfg1", "conv", diag, (1, 1, 1), (1, 1, 32), (1, 1, 1), (1, 1, 1), "VALID"),
        ("cfg2", "conv", diag, (1, 1, 3), (1, 1, 32), (1, 1, 1), (1, 1, 2), "SAME"),
        ("cfg3", "conv", diag, (1, 1, 5), (1, 1, 32), (1, 1, 1), (1, 1, 2), "SAME"),
        ("cfg4", "conv", over, (1, 1, 3), (1, 1, 32), (1, 1, 2), (1, 1, 1), "SAME"),
        ("cfg5", "conv", diag, (1, 1, 3), (1, 1, 32), (1, 1, 1), (1, 1, 2), "SAME"),
        ("cfg6", "conv", diag, (1, 3, 3), (1, 8, 8), (1, 1, 1), (1, 1, 1), "SAME"),
        ("cfg7", "conv", over, (1, 3, 3), (1, 8, 8), (1, 1, 1), (1, 1, 1), "VALID"),
        ("cfg8", "conv", diag, (3, 3, 3), (4, 4, 4), (1, 1, 1), (1, 1, 1), "SAME"),
        ("cfg9", "deconv", diag, (1, 1, 3), (1, 1, 32), (1, 1, 1), (1, 1, 2), "SAME"),
        ("rand", "conv", rand, (1, 3, 3), (1, 6, 7), (1, 1, 1), (1, 2, 1), "SAME"),
    ]


def main():
    if not REF or not os.path.isfile(os.path.join(REF, "blocksparse", "conv.py")):
        sys.exit("set BLOCKSPARSE_REFERENCE to a checkout of openai/blocksparse")
    cv = import_conv()
    rng = np.random.default_rng(2024)
    for name, kind, BCK, TRS, DHW, dilates, strides, padding in configs(rng):
        clss = cv.BlocksparseDeconv if kind == "deconv" else cv.BlocksparseConv
        captured = {}
        real = cv.tf.constant

        def constant(value, name=None, **kw):
            captured[name] = np.array(value)
            return real(value, name=name, **kw)
        cv.tf.constant = constant
        op = clss(BCK, TRS, DHW, dilates=dilates, strides=strides, padding=padding)
        cv.tf.constant = real
        N = 2
        flatF, flatU = hash_values(op.sizeF, 1), hash_values(op.sizeF, 2)
        offs = np.cumsum([0] + [int(np.prod(op.f_shape(b))) for b in range(op.blocks)])
        F = [flatF[offs[b]:offs[b + 1]].reshape(op.f_shape(b)) for b in range(op.blocks)]
        U = [flatU[offs[b]:offs[b + 1]].reshape(op.f_shape(b)) for b in range(op.blocks)]
        I = hash_values(int(np.prod(op.i_shape(N))), 3).reshape(op.i_shape(N))
        E = hash_values(int(np.prod(op.o_shape(N))), 4).reshape(op.o_shape(N))
        G = hash_values(op.C if kind == "deconv" else op.K, 5)
        out = dict(kind=kind, TRS=np.array(TRS), DHW=np.array(DHW), dilates=np.array(dilates),
                   strides=np.array(strides), padding_spec=np.array(padding),
                   c_lists=np.concatenate([c for c, _ in BCK]).astype(np.int32),
                   k_lists=np.concatenate([k for _, k in BCK]).astype(np.int32),
                   c_sizes=np.array([len(c) for c, _ in BCK]), k_sizes=np.array([len(k) for _, k in BCK]),
                   C=op.C, K=op.K, MPQ=np.array(op.MPQ), padding=np.array(op.padding), sizeF=op.sizeF,
                   overlapC=op.overlapC, overlapK=op.overlapK, flops=op.flops,
                   i_shape=np.array(op.i_shape(N)), o_shape=np.array(op.o_shape(N)),
                   f_shape=np.array(op.f_shape()), norm_lut=captured["norm_lut"], N=N)
        res = dict(fprop=op.fprop_test(F, I), bprop=op.bprop_test(F, E), updat=op.updat_test(E, I),
                   l2=op.l2_normalize_test(F), l2_grad=op.l2_normalize_grad_test(F, U)[0])
        if not (op.overlapC if kind == "deconv" else op.overlapK):
            res["l2_gain"] = op.l2_normalize_test(F, gain=G)
            res["l2_gain_grad"], res["l2_gain_dg"] = op.l2_normalize_grad_test(F, U, gain=G)
        for i, (key, val) in enumerate(sorted(res.items())):
            out[key + "_idx"], out[key] = sample(val, 17 + i)
        np.savez_compressed(os.path.join(HERE, "conv_%s.npz" % name), **out)
        print("conv_%s.npz" % name)


if __name__ == "__main__":
    main()
