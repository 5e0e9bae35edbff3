"""Generate the dense softmax / top-k fixtures (dense_*.npz) in this directory from the REFERENCE implementation.

Needs a checkout of openai/blocksparse (the tests only read the committed .npz files):

    BLOCKSPARSE_REFERENCE=/path/to/blocksparse python tests/golden/make_golden_dense.py

The reference is imported as make_golden.py does it (TensorFlow mocked, package __init__ bypassed). Everything the
fixtures record is computed by the reference's own module-level NumPy checkers of blocksparse/transformer.py:
masked_softmax_test, masked_top_k_softmax_test, masked_softmax_grad_test (:609-656) and rectified_top_k_test (:536-549).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import import_reference  # noqa: E402


def gen_dense(tr):
    """The reference's checkers on seeded inputs -> dense_*.npz: ranks 2-4, no mask and the mask shapes its flattening
    checker gets right ((1, ..., 1, D3), (1, ..., D2, D3), x's trailing shape), non-binary mask values with zeros, k in
    {1, mid, D3}. x is continuous, so no row ties across its k boundary; every row keeps at least `mid` visible entries,
    so the masked entries (all -FLT_MAX) never straddle it either."""
    rng = np.random.default_rng(20261016)
    cases = [("r2", (6, 16), [None, (1, 16), (6, 16)]),
             ("r3", (3, 5, 24), [None, (1, 1, 24), (1, 5, 24)]),
             ("r4", (2, 3, 4, 20), [None, (1, 1, 1, 20), (1, 1, 4, 20), (1, 3, 4, 20)])]
    for name, shape, masks in cases:
        D3 = shape[-1]
        for mshape in masks:
            x = rng.normal(0, 2.0, shape).astype(np.float32)
            scale = float(rng.choice([0.5, -0.75, 1.25]))
            rec = dict(x=x, scale=scale)
            mask = None
            if mshape is not None:
                mask = (rng.uniform(0.5, 1.5, mshape) * (rng.random(mshape) >= 0.2)).astype(np.float32)
                mask[..., 0] = 1.0
                rec["mask"] = mask
            visible = D3 if mask is None else int((np.broadcast_to(mask, shape) != 0).sum(axis=-1).min())
            ks = np.array([1, min(D3 // 2, visible), D3])
            P = tr.masked_softmax_test(x.copy(), mask=mask, scale=scale)
            DY = rng.normal(0, 1, shape).astype(np.float32)
            rec.update(ks=ks, P=P, DY=DY, DX=tr.masked_softmax_grad_test(DY, P, mask=mask, scale=scale),
                       TK=np.stack([tr.masked_top_k_softmax_test(x.copy(), int(k), mask=mask, scale=scale) for k in ks]))
            if mask is None:       # rectified_top_k_test takes 2-D input
                x2 = x.reshape(-1, D3)
                rec["R_rebase"] = np.stack([tr.rectified_top_k_test(x2, int(k), rebase=True).reshape(shape) for k in ks])
                rec["R_plain"] = np.stack([tr.rectified_top_k_test(x2, int(k), rebase=False).reshape(shape) for k in ks])
            tag = "nomask" if mshape is None else "m" + "x".join(str(d) for d in mshape)
            np.savez_compressed(os.path.join(HERE, "dense_%s_%s.npz" % (name, tag)), **rec)
            print("wrote dense", name, tag, "ks", ks)


if __name__ == "__main__":
    _mm, tr = import_reference()
    gen_dense(tr)
