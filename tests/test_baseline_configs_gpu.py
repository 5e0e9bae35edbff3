"""GPU parity AT THE SIZES BASELINE.json NAMES (the benchmarked configurations), against the oracle.

The oracle's NumPy loops cannot run a 4096 x 4096 x 4096 problem in seconds, so every case compares
  * fprop / bprop on a strided SAMPLE of minibatch rows (48 rows that touch every 128-row tile) -- the oracle's
    `fprop` / `bprop` restatement of matmul.py:353-399 evaluated on exactly those rows, all features;
  * updat on a SAMPLE of weight blocks over the FULL minibatch (`updat_blocks`, matmul.py:401-419);
with the reference's two error metrics, and asserts which kernel family ran and that no bounded wait timed out.
Each density of cfg 2 selects a different xprop kernel variant (matmul.py picks the stage shape from the density).
"""
import numpy as np
import pytest
import torch

from tests._util import ref_errors
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
    Forward chain and both backward GEMMs against the oracle on (batch 3, heads 0 and 15)."""
    nb, bs, heads, hs, batch = 64, 64, 16, 64, 4
    lay = local_strided_layout(nb)

    def causal(blk_shape, head_idx, qry_idx, key_idx, blk_idx):
        m = np.ones(blk_shape, dtype=bool)
        if qry_idx == key_idx:
            m = np.tril(m)
        return m

    bst = BlocksparseTransformer(lay, bs, heads=heads, mask_callback=causal)
    assert (bst.blocks, bst.nn_max, bst.tn_max) == (453, 11, 57)
    gen = torch.Generator(device="cuda").manual_seed(5)
    Q, K, V, E = ((torch.rand((batch, nb * bs, heads * hs), generator=gen, device="cuda") * 2 - 1).half() for _ in range(4))
    scale = 1.0 / np.sqrt(hs)
    Q.requires_grad_(); K.requires_grad_(); V.requires_grad_()
    w = bst.query_key_op(Q, K)
    k_nt = _lib.last_kernel()
    p = bst.masked_softmax(w, scale=scale)
    y = bst.weight_value_op(p, V)
    k_nn = _lib.last_kernel()
    y.backward(E)
    assert _lib.device_error() == 0, _lib.device_error_text()
    assert k_nt.startswith("wgmma_bst") and k_nn.startswith("wgmma_bst")
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
