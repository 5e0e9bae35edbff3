"""GPU parity AT THE SIZES BASELINE.json NAMES (the benchmarked configurations), against the oracle.

The oracle's NumPy loops cannot run a 4096 x 4096 x 4096 problem in seconds, so every case compares
  * fprop / bprop on a strided SAMPLE of minibatch rows (48 rows that touch every 128-row tile) -- the oracle's
    `fprop` / `bprop` restatement of matmul.py:353-399 evaluated on exactly those rows, all features;
  * updat on a SAMPLE of weight blocks over the FULL minibatch (`updat_blocks`, matmul.py:401-419);
with the reference's two error metrics, and asserts which kernel family ran and that no bounded wait timed out.
The same samples are also checked elementwise against float64, with the error bound of the kernel that ran. Every
density of cfg 2 runs the same wgmma kernels; what changes is the LUT row length, up to 128 entries (4096 accumulated
terms) at density 1.0.
"""
import numpy as np
import pytest
import torch

from tests._util import (U_OUT, assert_within, dtype_name, fma_gemm_bound, mma_gemm_bound, ref_errors, softmax_grad_bound,
                         softmax_row_sums)
from blocksparse_b200 import BlocksparseMatMul, BlocksparseTransformer, _lib
from blocksparse_b200.layouts import bernoulli_layout, barabasi_albert_layout, local_strided_layout
from oracle.bsmm_oracle import MatmulOracle
from oracle.bst_oracle import TransformerOracle

pytestmark = pytest.mark.gpu

TOL16 = (4e-2, 1e-2)     # (max|d|/mean|ref|, l2): see tests/test_matmul_gpu.py for why the max metric gets 4e-2 in bf16


def _case(layout, bs, axis, N, dtype, seed, n_rows=48, n_blocks=96, expect=None, tol=TOL16):
    bsmm = BlocksparseMatMul(layout, block_size=bs, feature_axis=axis)
    orc = MatmulOracle(layout, bs, axis)
    gen = torch.Generator(device="cuda").manual_seed(seed)
    W = (torch.randn(bsmm.w_shape, generator=gen, device="cuda") * 0.01).to(dtype)
    X = (torch.randn(bsmm.i_shape(N), generator=gen, device="cuda") * 0.1).to(dtype)
    E = (torch.randn(bsmm.o_shape(N), generator=gen, device="cuda") * 0.1).to(dtype)
    rows = torch.as_tensor((np.arange(n_rows) * (N // n_rows) + np.arange(n_rows) % 7) % N, device="cuda")
    Wh = W.float().cpu().numpy()

    def sample(t):           # minibatch sample, in the op's own layout
        return (t.index_select(0, rows) if axis else t.index_select(1, rows)).float().cpu().numpy()

    kernels = {}
    y = bsmm.fprop(X, W); kernels["fprop"] = _lib.last_kernel()
    dx = bsmm.bprop(E, W); kernels["bprop"] = _lib.last_kernel()
    dw = bsmm.updat([X], [E]); kernels["updat"] = _lib.last_kernel()
    assert _lib.device_error() == 0, _lib.device_error_text()
    if expect:
        for op, k in kernels.items():
            assert k.startswith(expect), "%s ran %s, expected %s*" % (op, k, expect)
    errs = {}
    errs["fprop"] = ref_errors(sample(y), orc.fprop(sample(X), Wh))
    errs["bprop"] = ref_errors(sample(dx), orc.bprop(sample(E), Wh))
    rng = np.random.default_rng(seed)
    blk = np.sort(rng.choice(bsmm.blocks, size=min(n_blocks, bsmm.blocks), replace=False))
    ref_dw = orc.updat_blocks(X.float().cpu().numpy(), E.float().cpu().numpy(), blk)
    errs["updat"] = ref_errors(dw.index_select(0, torch.as_tensor(blk, device="cuda")).float().cpu().numpy(), ref_dw)
    for op, (mx, l2) in errs.items():
        assert mx <= tol[0] and l2 <= tol[1], "%s: max_err %.3e l2_err %.3e (%s)" % (op, mx, l2, kernels[op])
    # elementwise, against float64, with the bound of the kernel that ran: bs x the LUT row length terms per output
    # block of the layout the kernel walks (the 16 x 16 super-blocks for padded 8 x 8 blocks), N per dw element
    name = dtype_name(dtype)
    walked = bsmm._shadow if bsmm._shadow is not None else bsmm
    lay_w = walked.layout.astype(np.int64)
    W64, rows_x, rows_e = Wh.astype(np.float64), sample(X).astype(np.float64), sample(E).astype(np.float64)
    for op, got, a, fn in [("fprop", y, rows_x, orc.fprop), ("bprop", dx, rows_e, orc.bprop)]:
        counts = lay_w.sum(axis=1 if op == "bprop" else 0) * walked.bsize
        k = np.repeat(counts, walked.bsize).astype(np.float64)
        k = k[None, :] if axis else k[:, None]
        ref, ref_abs = fn(a, W64), fn(np.abs(a), np.abs(W64))
        bound_fn = fma_gemm_bound if kernels[op].startswith("fma_") else mma_gemm_bound
        assert_within(sample(got), ref, bound_fn(ref, ref_abs, name, k), "%s (%s)" % (op, kernels[op]), ref_abs, k, name,
                      kernels[op].split("_bs")[0])
    abs_dw = orc.updat_blocks(np.abs(X.float().cpu().numpy()), np.abs(E.float().cpu().numpy()), blk)
    bound_fn = fma_gemm_bound if kernels["updat"].startswith("fma_") else mma_gemm_bound
    got_dw = dw.index_select(0, torch.as_tensor(blk, device="cuda")).float().cpu().numpy()
    assert_within(got_dw, ref_dw, bound_fn(ref_dw, abs_dw, name, N), "updat (%s)" % kernels["updat"], abs_dw, N, name,
                  kernels["updat"].split("_bs")[0])
    # rows of Y that belong to empty output block-columns must be exactly zero (cn_64.cu:243-253)
    empty = np.nonzero(np.asarray(layout).sum(axis=0) == 0)[0]
    if len(empty):
        yv = y.reshape(bsmm.KB, bs, N) if axis == 0 else y.reshape(N, bsmm.KB, bs).permute(1, 2, 0)
        assert float(yv[torch.as_tensor(empty, device="cuda")].abs().max()) == 0.0
    return errs


@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("density", [0.05, 0.10, 0.25, 0.50, 1.00])
def test_cfg2_every_density_bf16(density, axis):
    """BASELINE configs[1]: 4096 x 4096, bs 32, N 4096, bf16, all five densities, both feature axes."""
    rng = np.random.default_rng(1236)
    lay = bernoulli_layout(rng, 128, 128, density)
    _case(lay, 32, axis, 4096, torch.bfloat16, seed=int(density * 100) + axis, expect="wgmma_")


def test_cfg2_fp16_headline_density():
    rng = np.random.default_rng(1236)
    _case(bernoulli_layout(rng, 128, 128, 0.25), 32, 1, 4096, torch.float16, seed=7, expect="wgmma_", tol=(1e-2, 1e-2))


@pytest.mark.parametrize("density", [0.10, 0.25])
def test_cfg2_skewed_barabasi_albert(density):
    """The reference benchmark's power-law layout (test/blocksparse_matmul_bench.py:53-68): a few block rows and
    columns hold most of the blocks, the case that made the reference segment its LUT."""
    rng = np.random.default_rng(1237)
    lay = barabasi_albert_layout(128, density, rng)
    assert lay.sum(axis=0).max() >= 3 * lay.sum(axis=0).mean() * 0.6
    _case(lay, 32, 1, 4096, torch.bfloat16, seed=11, expect="wgmma_")


@pytest.mark.parametrize("bs,axis", [(8, 0), (16, 0), (32, 0), (32, 1), (64, 1)])
def test_cfg4_block_size_sweep(bs, axis):
    """BASELINE configs[3]: 4096 x 4096, 20 % density, N 2048, block size 8 / 16 / 32 / 64."""
    rng = np.random.default_rng(1238)
    nb = 4096 // bs
    _case(bernoulli_layout(rng, nb, nb, 0.20), bs, axis, 2048, torch.bfloat16, seed=bs + axis, n_blocks=64)


def test_cfg3_full_heads_and_batch():
    """BASELINE configs[2]: heads 16, ctx 4096, bs 64, batch 4, head_state 64, fp16, causal local+strided layout.
    Forward chain and the whole backward (dv, the softmax gradient, dq, dk) against the oracle on (batch 3, heads 0
    and 15), and which kernel ran each backward op."""
    nb, bs, heads, hs, batch = 64, 64, 16, 64, 4
    lay = local_strided_layout(nb)

    def causal(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
        m = np.ones(blk_shape, dtype=bool)
        if qry_idx == key_idx:
            m = np.tril(m)
        return m

    bst = BlocksparseTransformer(lay, bs, heads=heads, mask_callback=causal)
    assert (bst.blocks, bst.nn_max, bst.tn_max) == (453, 11, 57)
    # record the kernel behind every raw op of the backward, with its operand dtypes
    seen = []

    def logged(fn, op):
        def run(*args, **kw):
            out = fn(*args, **kw)
            seen.append((op, args[0].dtype, args[1].dtype, _lib.last_kernel()))
            return out
        return run
    gen = torch.Generator(device="cuda").manual_seed(5)
    Q, K, V, E = ((torch.rand((batch, nb * bs, heads * hs), generator=gen, device="cuda") * 2 - 1).half() for _ in range(4))
    scale = 1.0 / np.sqrt(hs)
    Q.requires_grad_(); K.requires_grad_(); V.requires_grad_()
    w = bst.query_key_op(Q, K)
    k_nt = _lib.last_kernel()
    p = bst.masked_softmax(w, scale=scale)
    k_sm = _lib.last_kernel()
    y = bst.weight_value_op(p, V)
    k_nn = _lib.last_kernel()
    grads = {}
    w.register_hook(lambda g: grads.__setitem__("ds", g))       # softmax grad, cast back to the scores' bf16
    p.register_hook(lambda g: grads.__setitem__("dp", g))       # upstream gradient of the probabilities (fp16)
    bst._xn, bst._softmax_grad = logged(bst._xn, "xn"), logged(bst._softmax_grad, "softmax_grad")
    y.backward(E)
    assert _lib.device_error() == 0, _lib.device_error_text()
    assert k_nt.startswith("wgmma_bst") and k_nn.startswith("wgmma_bst")
    assert k_sm == "bst_softmax_staged"                                         # rows of <= 11 blocks: MAXE 12
    assert grads["ds"].dtype == torch.bfloat16 and grads["dp"].dtype == torch.float16
    # dv: fp16 x fp16 on wgmma; the softmax grad on the staged kernel (MAXE 12); dq / dk: bf16 dS x fp16 Q / K, which
    # the wgmma kernels refuse, on the CUDA-core kernel
    f16, b16 = torch.float16, torch.bfloat16
    assert seen == [("xn", f16, f16, "wgmma_bst_tn"), ("softmax_grad", f16, f16, "bst_softmax_grad_staged"),
                    ("xn", b16, f16, "fma_sdd_xn"), ("xn", b16, f16, "fma_sdd_xn")], seen
    b = batch - 1
    for h in (0, heads - 1):
        sl = slice(h * hs, (h + 1) * hs)
        orc = TransformerOracle(lay, bs, heads=1, mask_callback=causal)
        Qh, Kh, Vh, Eh = (t[b:b + 1, :, sl].detach().float().cpu().numpy() for t in (Q, K, V, E))
        S = orc.nt(Qh, Kh)
        S16 = torch.as_tensor(S).to(torch.bfloat16).float().numpy()          # the op stores scores in bf16
        P = orc.masked_softmax(S16, scale=scale)
        P16 = torch.as_tensor(P).half().float().numpy()
        Y = orc.nn(P16, Vh)
        DV = orc.tn(P16, Eh)
        for got, ref, what, tol in [(w[b:b + 1, h:h + 1], S, "scores", (4e-2, 1e-2)),
                                    (p[b:b + 1, h:h + 1], P, "probs", (1e-1, 1e-2)),
                                    (y[b:b + 1, :, sl], Y, "y", (1.5e-1, 1e-2)),
                                    (V.grad[b:b + 1, :, sl], DV, "dv", (1.5e-1, 1e-2))]:
            mx, l2 = ref_errors(got.detach().float().cpu().numpy().reshape(ref.shape), ref)
            assert mx <= tol[0] and l2 <= tol[1], "head %d %s: max %.3e l2 %.3e" % (h, what, mx, l2)

        # backward through the softmax, elementwise, at the op's own intermediates of this slice
        Pk = p[b:b + 1, h:h + 1].detach().double().cpu().numpy()
        dPk = grads["dp"][b:b + 1, h:h + 1].double().cpu().numpy()
        dSk = grads["ds"][b:b + 1, h:h + 1].double().cpu().numpy()
        DSk = orc.masked_softmax_grad(dPk, Pk, scale=scale)                    # float64
        bound = softmax_grad_bound(DSk, dPk, Pk, softmax_row_sums(np.abs(dPk * Pk), orc), "float16", scale, bst.nn_max)
        bound += U_OUT["bfloat16"] * (np.abs(DSk) + bound)                     # fp16 result cast to bf16 for the NT backward
        err = np.abs(dSk - DSk)
        assert np.all(err <= bound), "head %d softmax grad: %d out of bound" % (h, int((err > bound).sum()))
        dS32 = dSk.astype(np.float32)
        for got, op, dense, k_terms, what in [(Q.grad, orc.nn, Kh, bst.nn_max * bs, "dq"), (K.grad, orc.tn, Qh, bst.tn_max * bs, "dk")]:
            ref = op(dS32, dense)
            g = got[b:b + 1, :, sl].double().cpu().numpy()
            bound = fma_gemm_bound(ref.astype(np.float64), op(np.abs(dS32), np.abs(dense)).astype(np.float64), "float16", k_terms)
            err = np.abs(g - ref)
            assert np.all(err <= bound), "head %d %s: %d out of bound" % (h, what, int((err > bound).sum()))
        # and the whole backward against the oracle chain on its own 16-bit-rounded intermediates
        DP16 = torch.as_tensor(orc.nt(Eh, Vh)).half().float().numpy()
        DS16 = torch.as_tensor(orc.masked_softmax_grad(DP16, P16, scale=scale)).to(torch.bfloat16).float().numpy()
        # probabilities and their gradients are peaked per row, so the max metric (over the MEAN magnitude) says little
        # about dS: its l2 only; dq / dk are three 16-bit roundings deep, as in the golden chain test
        for got, ref, what, tol in [(grads["ds"][b:b + 1, h:h + 1], DS16, "ds", (np.inf, 1e-2)),
                                    (Q.grad[b:b + 1, :, sl], orc.nn(DS16, Kh), "dq", (2e-1, 2e-2)),
                                    (K.grad[b:b + 1, :, sl], orc.tn(DS16, Qh), "dk", (2e-1, 2e-2))]:
            mx, l2 = ref_errors(got.float().cpu().numpy().reshape(ref.shape), ref)
            assert mx <= tol[0] and l2 <= tol[1], "head %d %s: max %.3e l2 %.3e" % (h, what, mx, l2)
