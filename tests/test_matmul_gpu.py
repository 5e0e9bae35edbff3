"""GPU parity: BlocksparseMatMul through the C ABI vs the oracle / reference fixtures.

Tolerances (BASELINE.json north_star): fp32 <= 1e-5, fp16/bf16 <= 1e-2 relative error, measured with the
reference's own metrics max|d|/mean|ref| and ||d||2/||ref||2 (test/blocksparse_matmul_test.py:408-418).
"""
import os

import numpy as np
import pytest
import torch

from tests._util import (GOLDEN, _on_poisoned_output, assert_within, assert_zero_filled, feature_terms, fma_gemm_bound,
                         golden_files, oracle_dense, ref_errors)
from blocksparse_b200 import BlocksparseMatMul, group_param_grads, _lib
from oracle.bsmm_oracle import MatmulOracle

pytestmark = pytest.mark.gpu

# (max|d|/mean|ref|, ||d||2/||ref||2).  The l2 bound is the north-star tolerance.  The max metric divides the
# worst element by the MEAN magnitude, so the output rounding alone (2^-9 of the largest bf16 element, 2^-12 for
# fp16) times max/mean (~5-8 for Gaussian data) is already 1-1.6e-2 for bf16: it gets 4e-2, fp16 keeps 1e-2.
TOL = {torch.float32: (1e-5, 1e-5), torch.float16: (1e-2, 1e-2), torch.bfloat16: (4e-2, 1e-2)}
DTYPES = [torch.float32, torch.float16, torch.bfloat16]


def rounded(a, dtype):
    """Round a float array through the storage dtype (blocksparse_matmul_test.py:313,345-346)."""
    t = torch.as_tensor(np.asarray(a, dtype=np.float32)).to(dtype)
    return t.cuda(), t.to(torch.float32).numpy()


def check(got, ref, dtype, what):
    mx, l2 = ref_errors(got.detach().to(torch.float32).cpu().numpy(), ref)
    tmx, tl2 = TOL[dtype]
    assert mx <= tmx and l2 <= tl2, "%s: max_err %.3e l2_err %.3e (dtype %s)" % (what, mx, l2, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fname", golden_files("bsmm_"))
def test_golden_fixture_parity(fname, dtype):
    g = np.load(os.path.join(GOLDEN, fname))
    bs, axis = int(g["bsize"]), int(g["axis"])
    bsmm = BlocksparseMatMul(g["layout"], block_size=bs, feature_axis=axis)
    orc = MatmulOracle(g["layout"], bs, axis)
    Wd, Wh = rounded(g["W"], dtype)
    Xd, Xh = rounded(g["X"], dtype)
    Ed, Eh = rounded(g["E"], dtype)
    if dtype == torch.float32:            # exact inputs -> compare with the reference's recorded outputs
        Y, DX, DW = g["Y"], g["DX"], g["DW"]
    else:
        Y, DX, DW = orc.fprop(Xh, Wh), orc.bprop(Eh, Wh), orc.updat(Xh, Eh)
    check(bsmm.fprop(Xd, Wd), Y, dtype, "fprop")
    check(bsmm.bprop(Ed, Wd), DX, dtype, "bprop")
    check(bsmm.updat([Xd], [Ed]), DW, dtype, "updat")
    if "gate" in g.files:
        gate = torch.as_tensor(g["gate"]).cuda()
        check(bsmm.fprop(Xd, Wd, gate=gate), orc.fprop(Xh, Wh, gate=g["gate"]), dtype, "fprop gated")
        check(bsmm.bprop(Ed, Wd, gate=gate), orc.bprop(Eh, Wh, gate=g["gate"]), dtype, "bprop gated")
        check(bsmm.updat([Xd], [Ed], gate=gate, dw_gated=True),
              orc.updat(Xh, Eh, gate=g["gate"], dw_gated=True), dtype, "updat gated")


def make_layout(rng, CB, KB, density):
    lay = (rng.random((CB, KB)) < density).astype(np.int32)
    for i in range(min(CB, KB)):
        lay[i, i] = 1
    return lay


@pytest.mark.parametrize("axis,bs", [(0, 32), (1, 32), (0, 8), (0, 16), (1, 64), (0, 64), (1, 8), (1, 16)])
@pytest.mark.parametrize("N", [1, 7, 64, 65, 200])
def test_ragged_minibatch_fp32(axis, bs, N):
    rng = np.random.default_rng(100 + N + bs)
    lay = make_layout(rng, 5, 7, 0.3)
    lay[:, 4] = 0                      # empty output column must be zero-filled
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=axis)
    orc = MatmulOracle(lay, bs, axis) if (axis, bs) in [(0, 8), (0, 16), (0, 32), (1, 32), (1, 64)] else None
    W = rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)
    X = rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)
    E = rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)
    if orc is None:                    # (axis, bs) pairs the reference rejects: use the dense einsum restatement
        orc = MatmulOracle.__new__(MatmulOracle)
        base = MatmulOracle(lay, 32, axis)
        orc.__dict__.update(base.__dict__)
        orc.bsize, orc.C, orc.K, orc.w_shape = bs, lay.shape[0] * bs, lay.shape[1] * bs, bsmm.w_shape
    Wd, Xd, Ed = (torch.as_tensor(a).cuda() for a in (W, X, E))
    # true fp32 FMA kernels, elementwise against float64 (fma_gemm_bound: bs x the LUT row length terms per output
    # block, N per dw element), each on NaN-poisoned output memory
    for op, inp, fn in [("fprop", X, bsmm.fprop), ("bprop", E, bsmm.bprop)]:
        ref, ref_abs = oracle_dense(orc, op, inp, W), oracle_dense(orc, op, np.abs(inp), np.abs(W))
        dev = torch.as_tensor(inp).cuda()
        got = _on_poisoned_output(lambda: fn(dev, Wd))
        assert _lib.last_kernel() == "fma_sdd_xn", _lib.last_kernel()
        assert_zero_filled(got, np.nonzero(lay.sum(axis=1 if op == "bprop" else 0) == 0)[0], bs, axis, op)
        assert_within(got, ref, fma_gemm_bound(ref, ref_abs, "float32", feature_terms(lay, bs, op == "bprop", axis)), op)
        check(got, ref, torch.float32, op)
        if op == "fprop":
            y = got
    ref, ref_abs = oracle_dense(orc, "updat", X, E), oracle_dense(orc, "updat", np.abs(X), np.abs(E))
    dw = _on_poisoned_output(lambda: bsmm.updat([Xd], [Ed]))
    assert _lib.last_kernel() == "fma_dds_nt", _lib.last_kernel()
    assert_within(dw, ref, fma_gemm_bound(ref, ref_abs, "float32", N), "updat")
    check(dw, ref, torch.float32, "updat")
    yv = y.reshape(bsmm.KB, bs, N) if axis == 0 else y.reshape(N, bsmm.KB, bs).permute(1, 2, 0)
    assert float(yv[4].abs().max()) == 0.0


def test_cfg1_reference_recipe_fp32():
    """BASELINE cfg 1: 256x256, bs=32, 25 %, N=64, fp32, both axes; values as in the reference test."""
    rng = np.random.default_rng(1235)
    lay = make_layout(rng, 8, 8, 0.25)
    for axis in (0, 1):
        bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=axis)
        orc = MatmulOracle(lay, 32, axis)
        W = rng.normal(0, 0.01, bsmm.w_shape).astype(np.float32)
        X = rng.normal(0, 0.1, bsmm.i_shape(64)).astype(np.float32)
        E = rng.normal(0, 0.1, bsmm.o_shape(64)).astype(np.float32)
        Wd, Xd, Ed = (torch.as_tensor(a).cuda() for a in (W, X, E))
        check(bsmm.fprop(Xd, Wd), orc.fprop(X, W), torch.float32, "fprop")
        check(bsmm.bprop(Ed, Wd), orc.bprop(E, W), torch.float32, "bprop")
        check(bsmm.updat([Xd], [Ed]), orc.updat(X, E), torch.float32, "updat")
        assert _lib.last_kernel().startswith("fma_")      # fp32 must run true-fp32 FMA, never TF32


@pytest.mark.parametrize("dtype", DTYPES)
def test_multi_pair_updat_and_accumulate(dtype):
    rng = np.random.default_rng(5)
    lay = make_layout(rng, 6, 6, 0.4)
    bsmm = BlocksparseMatMul(lay, block_size=16, feature_axis=0)
    orc = MatmulOracle(lay, 16, 0)
    N = 48
    xs, es, ref = [], [], np.zeros(bsmm.w_shape)
    for _ in range(8):
        xd, xh = rounded(rng.normal(0, 0.5, bsmm.i_shape(N)), dtype)
        ed, eh = rounded(rng.normal(0, 0.5, bsmm.o_shape(N)), dtype)
        xs.append(xd); es.append(ed)
        ref += orc.updat(xh, eh)
    dw = bsmm.updat(xs, es, dw_dtype=torch.float32)
    check(dw, ref, torch.float32 if dtype == torch.float32 else dtype, "8 pairs")
    dw2 = bsmm.updat(xs[:3], es[:3], dw=dw.clone())          # beta = 1: accumulate in place
    ref2 = ref + sum(orc.updat(x.float().cpu().numpy(), e.float().cpu().numpy()) for x, e in zip(xs[:3], es[:3]))
    check(dw2, ref2, torch.float32 if dtype == torch.float32 else dtype, "accumulate")
    with pytest.raises(ValueError):
        bsmm.updat(xs + xs[:1], es + es[:1])                # 9 pairs: reference limit is 8 (op.cc:233-234)
    check(bsmm.updat(xs[:2], es[:2], alpha=0.5, dw_dtype=torch.float32),
          0.5 * (orc.updat(xs[0].float().cpu().numpy(), es[0].float().cpu().numpy())
                 + orc.updat(xs[1].float().cpu().numpy(), es[1].float().cpu().numpy())),
          torch.float32 if dtype == torch.float32 else dtype, "alpha")


@pytest.mark.parametrize("axis", [0, 1])
def test_autograd_matches_oracle(axis):
    rng = np.random.default_rng(9)
    lay = make_layout(rng, 4, 6, 0.5)
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=axis)
    orc = MatmulOracle(lay, 32, axis)
    N = 40
    W = rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)
    X = rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)
    E = rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)
    w = torch.as_tensor(W).cuda().requires_grad_()
    x = torch.as_tensor(X).cuda().requires_grad_()
    y = bsmm(x, w)
    y.backward(torch.as_tensor(E).cuda())
    check(y, orc.fprop(X, W), torch.float32, "y")
    check(x.grad, orc.bprop(E, W), torch.float32, "dx")
    check(w.grad, orc.updat(X, E), torch.float32, "dw")


def test_gate_grad_and_group_param_grads():
    rng = np.random.default_rng(11)
    lay = make_layout(rng, 5, 5, 0.5)
    bsmm = BlocksparseMatMul(lay, block_size=8, feature_axis=0)
    orc = MatmulOracle(lay, 8, 0)
    N, T = 16, 11
    W = rng.normal(0, 0.3, bsmm.w_shape).astype(np.float32)
    w = torch.as_tensor(W).cuda().requires_grad_()
    # a depth-T chain through the same weight (blocksparse_matmul_test.py:363-374)
    X0 = rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)
    E = rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)

    def run():
        h = torch.as_tensor(X0).cuda()
        for _ in range(T):
            h = bsmm(h, w)
        return h

    w.grad = None
    run().backward(torch.as_tensor(E).cuda())
    plain = w.grad.clone()
    w.grad = None
    with group_param_grads(bsmm, w, group_size=8) as pend:
        run().backward(torch.as_tensor(E).cuda())
    assert pend.launches == 2                      # ceil(11 / 8) multi-pair launches
    check(w.grad, plain.cpu().numpy().astype(np.float64), torch.float32, "grouped dw == per-use dw")
    # oracle value of the chained gradient
    hs, h = [X0], X0
    for _ in range(T):
        h = orc.fprop(h, W).astype(np.float32); hs.append(h)
    e, ref = E, np.zeros(bsmm.w_shape)
    for t in reversed(range(T)):
        ref += orc.updat(hs[t], e)
        e = orc.bprop(e, W).astype(np.float32)
    mx, l2 = ref_errors(plain.cpu().numpy(), ref)
    assert l2 < 1e-4                                # 11 chained fp32 matmuls

    gate = torch.as_tensor(rng.uniform(0.5, 1.5, bsmm.blocks).astype(np.float32)).cuda().requires_grad_()
    w.grad = None
    x = torch.as_tensor(X0).cuda()
    y = bsmm(x, w, gate=gate, gate_grad=True, dw_gated=True)
    y.backward(torch.as_tensor(E).cuda())
    dw_ref = orc.updat(X0, E, gate=gate.detach().cpu().numpy(), dw_gated=True)
    check(w.grad, dw_ref, torch.float32, "gated dw")
    check(gate.grad, (orc.updat(X0, E) * W).sum(axis=(1, 2)), torch.float32, "dg")


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_full_size_properties(axis, dtype):
    """BASELINE cfg 2 size (4096x4096, bs 32, N 4096): too big for the NumPy loops, so check
    (a) a dense torch fp32 matmul of the scattered weight on sampled rows/columns and
    (b) linearity  f(x1 + x2) = f(x1) + f(x2)  up to rounding."""
    rng = np.random.default_rng(1236)
    lay = make_layout(rng, 128, 128, 0.10)
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=axis)
    N = 4096
    gen = torch.Generator(device="cuda").manual_seed(3)
    W = (torch.randn(bsmm.w_shape, generator=gen, device="cuda") * 0.01).to(dtype)
    X = (torch.randn(bsmm.i_shape(N), generator=gen, device="cuda") * 0.1).to(dtype)
    E = (torch.randn(bsmm.o_shape(N), generator=gen, device="cuda") * 0.1).to(dtype)
    D = torch.zeros(bsmm.C, bsmm.K, device="cuda")
    cs = torch.as_tensor(bsmm.updat_lut[:, 0].astype(np.int64)).cuda()
    ks = torch.as_tensor(bsmm.updat_lut[:, 1].astype(np.int64)).cuda()
    Dv = D.view(bsmm.CB, 32, bsmm.KB, 32)
    Dv[cs, :, ks, :] = W.float()
    torch.backends.cuda.matmul.allow_tf32 = False
    Xf, Ef = X.float(), E.float()
    y_ref = (Xf @ D) if axis else (D.t() @ Xf)
    dx_ref = (Ef @ D.t()) if axis else (D @ Ef)
    full = (Xf.t() @ Ef) if axis else (Xf @ Ef.t())
    dw_ref = full.view(bsmm.CB, 32, bsmm.KB, 32)[cs, :, ks, :]
    for got, ref, what in [(bsmm.fprop(X, W), y_ref, "fprop"), (bsmm.bprop(E, W), dx_ref, "bprop"),
                           (bsmm.updat([X], [E]), dw_ref, "updat")]:
        d = (got.float() - ref)
        mx = float(d.abs().max() / ref.abs().mean())
        l2 = float(d.norm() / ref.norm())
        assert l2 <= 1e-2 and mx <= 5e-2, "%s max %.3e l2 %.3e" % (what, mx, l2)
    X2 = (torch.randn(bsmm.i_shape(N), generator=gen, device="cuda") * 0.1).to(dtype)
    lhs = bsmm.fprop((X.float() + X2.float()).to(dtype), W).float()
    rhs = bsmm.fprop(X, W).float() + bsmm.fprop(X2, W).float()
    assert float((lhs - rhs).norm() / rhs.norm()) < 2e-2
