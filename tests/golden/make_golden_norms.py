"""Generate the layer norm fixtures (norms_*.npz) in this directory from the REFERENCE implementation.

Needs a checkout of openai/blocksparse (the tests only read the committed .npz files):

    BLOCKSPARSE_REFERENCE=/path/to/blocksparse python tests/golden/make_golden_norms.py

The reference is imported as make_golden.py does it (TensorFlow mocked, package __init__ bypassed). What the fixtures
record is computed by the reference's own NumPy checkers of blocksparse/norms.py: layer_norm_test and
layer_norm_grad_test, in float64.
"""
import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import import_reference  # noqa: E402

# (tag, x shape, axis, segments): both axes, segments 1 / 2 / 4 on the last axis, the odd widths 31 and 33 of the
# reference's layer norm test
CASES = [("ax1_k64_s1", (6, 64), 1, 1), ("ax1_k64_s2", (5, 64), 1, 2), ("ax1_k96_s4", (4, 96), 1, 4),
         ("ax1_k31_s1", (7, 31), 1, 1), ("ax1_k33_s1", (3, 2, 33), -1, 1), ("ax0_k33_s1", (33, 6), 0, 1),
         ("ax0_k31_s1", (31, 9), 0, 1), ("ax0_k48_s1", (48, 2, 4), 0, 1)]


def gen_norms(norms):
    rng = np.random.default_rng(20261017)
    for tag, shape, axis, segments in CASES:
        K = shape[axis]
        for relu in (False, True):
            x = rng.normal(0.5, 2.0, shape)
            g = rng.uniform(0.5, 1.5, K)
            b = rng.normal(0.0, 0.5, K)
            dy = rng.normal(0.0, 1.0, shape)
            eps = 1e-6 if relu else 1e-3
            y = norms.layer_norm_test(x, g, b, axis=axis, segments=segments, epsilon=eps, relu=relu)
            dx, dg, db = norms.layer_norm_grad_test(dy, x, g, b, axis=axis, segments=segments, epsilon=eps, relu=relu)
            name = "norms_%s_%s.npz" % (tag, "relu" if relu else "lin")
            np.savez_compressed(os.path.join(HERE, name), x=x, g=g, b=b, dy=dy, axis=axis, segments=segments,
                                epsilon=eps, relu=relu, y=y, dx=dx, dg=np.ravel(dg), db=np.ravel(db))
            print("wrote", name)


if __name__ == "__main__":
    import_reference()
    gen_norms(importlib.import_module("blocksparse.norms"))
