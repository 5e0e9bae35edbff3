"""Generate the conv edge bias and cwise_linear fixtures (edge_bias_*.npz, cwise_*.npz) from the REFERENCE
implementation.

Needs a checkout of openai/blocksparse (the tests only read the committed .npz files):

    BLOCKSPARSE_REFERENCE=/path/to/blocksparse python tests/golden/make_golden_conv_bias.py

The reference's blocksparse/conv.py is imported with TensorFlow mocked, as make_golden_conv.py does. Recorded from its
own Python / NumPy code: ConvEdgeBias's edgeBiasMap, edgeEntries and shape, the edge table it hands to tf.constant,
and edge_bias_test / edge_bias_grad_test on hash-derived inputs (N = 2); cwise_linear_test / cwise_linear_grad_test on
the shapes of test/cwise_linear_test.py plus a rank-2 one. Every edge config is at dilation 1, where the reference's
SAME padding is TensorFlow's. Inputs are not stored (hash_values() derives them); outputs are sampled as in
make_golden_conv.py.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF  # noqa: E402
from make_golden_conv import hash_values, import_conv, sample  # noqa: E402


def edge_configs():
    """(name, y_shape, x_shape, w_shape, strides, data_format, deconv): y = conv(x, w), or y = conv_transpose(x, w)
    for the deconv (its y the larger image), as conv_edge_bias_init / deconv_edge_bias_init take them."""
    cfgs = []
    for N, K, HW in ((1, 96, 8), (1, 24, 32)):                    # test/edge_bias_test.py's 3x3 shapes
        cfgs.append(("ref_k%d_nhwc" % K, [N, HW, HW, K], [N, HW, HW, K], [3, 3, K, K], None, "NHWC", False))
        cfgs.append(("ref_k%d_nchw" % K, [N, K, HW, HW], [N, K, HW, HW], [3, 3, K, K], None, "NCHW", False))
    cfgs += [
        ("stride2", [2, 5, 5, 8], [2, 9, 10, 6], [3, 3, 6, 8], [1, 2, 2, 1], "NHWC", False),
        ("even2x2", [2, 7, 7, 5], [2, 7, 7, 3], [2, 2, 3, 5], None, "NHWC", False),
        ("even4x4", [2, 6, 9, 8], [2, 6, 9, 8], [4, 4, 6, 6], None, "NCHW", False),
        ("conv1d", [2, 20, 7], [2, 20, 5], [5, 5, 7], None, "NWC", False),
        ("conv3d", [2, 4, 5, 6, 7], [2, 4, 5, 6, 7], [3, 3, 3, 4, 4], None, "NCDHW", False),
        ("deconv", [2, 8, 10, 3], [2, 4, 5, 6], [3, 3, 3, 6], [1, 2, 2, 1], "NHWC", True),
    ]
    return cfgs


CWISE_SHAPES = [(1, 32, 32), (8, 64, 4, 4), (3, 16), (2, 8, 3, 4, 5)]


def main():
    if not REF or not os.path.isfile(os.path.join(REF, "blocksparse", "conv.py")):
        sys.exit("set BLOCKSPARSE_REFERENCE to a checkout of openai/blocksparse")
    cv = import_conv()
    for name, y_shape, x_shape, w_shape, strides, fmt, deconv in edge_configs():
        captured = {}
        real = cv.tf.constant

        def constant(value, name=None, **kw):
            captured[name] = np.array(value)
            return real(value, name=name, **kw)
        cv.tf.constant = constant
        cv.ConvEdgeBias.Cache.clear()
        if deconv:      # deconv_edge_bias_init's swap
            eb = cv.ConvEdgeBias(x_shape, y_shape, w_shape, strides, "SAME", fmt, None, deconv=True)
        else:
            eb = cv.ConvEdgeBias(y_shape, x_shape, w_shape, strides, "SAME", fmt, None)
        io_shape = y_shape      # the op runs on y in both cases
        cv.tf.constant = real
        size = int(np.prod(io_shape))
        x = hash_values(size, 1).reshape(io_shape)
        dy = hash_values(size, 2).reshape(io_shape)
        g = hash_values(int(np.prod(eb.shape)), 3).reshape(eb.shape)
        b = hash_values(int(np.prod(eb.shape)), 4).reshape(eb.shape)
        dx, dg, db = eb.edge_bias_grad_test(dy, x, g)
        out = dict(y_shape=np.array(y_shape), x_shape=np.array(x_shape), w_shape=np.array(w_shape),
                   strides=np.array(strides if strides else []), data_format=np.array(fmt), deconv=deconv,
                   io_shape=np.array(io_shape), shape=np.array(eb.shape), entries=eb.edgeEntries,
                   map_sizes=np.array([len(m) for m in eb.edgeBiasMap]),
                   map=np.concatenate(eb.edgeBiasMap).astype(np.int32), lut=captured["edge_bias_lut"])
        res = dict(y=eb.edge_bias_test(x, g, b), dx=dx, dg=dg, db=db)
        for i, (key, val) in enumerate(sorted(res.items())):
            out[key + "_idx"], out[key] = sample(val, 31 + i)
        np.savez_compressed(os.path.join(HERE, "edge_bias_%s.npz" % name), **out)
        print("edge_bias_%s.npz" % name, eb.shape)
    for shape in CWISE_SHAPES:
        C = shape[1]
        x = hash_values(int(np.prod(shape)), 5).reshape(shape)
        dy = hash_values(int(np.prod(shape)), 6).reshape(shape)
        a, b = hash_values(C, 7), hash_values(C, 8)
        out = dict(shape=np.array(shape))
        res = {}
        for relu in (False, True):
            tag = "_relu" if relu else ""
            res["y" + tag] = cv.cwise_linear_test(x, a, b, relu=relu)
            res["dx" + tag], res["da" + tag], res["db" + tag] = cv.cwise_linear_grad_test(dy, x, a, b, relu=relu)
        for i, (key, val) in enumerate(sorted(res.items())):
            out[key + "_idx"], out[key] = sample(val, 41 + i)
        name = "cwise_" + "x".join(str(d) for d in shape)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
        print(name + ".npz")


if __name__ == "__main__":
    main()
