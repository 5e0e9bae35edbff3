"""GPU parity of the wgmma kernel families (forced with BSMM_FLAG_FORCE_TC so a silent fall-back to the
CUDA-core kernels cannot pass) against the oracle, at sizes the NumPy loops finish in seconds."""
import numpy as np
import pytest
import torch

from tests._util import fma_gemm_bound, ref_errors
from blocksparse_b200 import BlocksparseMatMul, _lib
from oracle.bsmm_oracle import MatmulOracle

pytestmark = pytest.mark.gpu


def layout(rng, CB, KB, density, empty_col=None, empty_row=None):
    lay = (rng.random((CB, KB)) < density).astype(np.int32)
    lay[rng.integers(CB), rng.integers(KB)] = 1
    if empty_col is not None:
        lay[:, empty_col] = 0
    if empty_row is not None:
        lay[empty_row, :] = 0
    if lay.sum() == 0:
        lay[0, 0] = 1
    return lay


CASES = [
    # CB, KB, density, N, bs
    (8, 8, 0.3, 128, 32),
    (5, 37, 0.5, 200, 32),        # ragged N, more than two output tiles (16 blocks each), rectangular
    (40, 33, 0.08, 1, 32),        # single row
    (20, 20, 1.0, 257, 32),       # dense layout: 16 pairs per group
    (64, 64, 0.2, 640, 32),       # many tiles per CTA
    (9, 40, 0.3, 200, 16),        # 16 x 16 blocks: 16-block tiles, 32-byte swizzle
    (33, 17, 0.15, 64, 16),
    (12, 12, 1.0, 130, 16),
    (6, 9, 0.5, 130, 64),
    (16, 17, 0.3, 64, 64),
    (12, 12, 1.0, 300, 64),
]


@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", CASES)
def test_tc_xprop_matches_oracle(case, dtype, axis):
    CB, KB, density, N, bs = case
    if axis == 0:
        N = max(8, (N + 7) // 8 * 8)          # TMA needs a 16-byte row pitch when the minibatch is the inner dim
    rng = np.random.default_rng(CB * 1000 + KB * 10 + N)
    lay = layout(rng, CB, KB, density, empty_col=KB // 2 if density < 1 else None, empty_row=1 if density < 1 and CB > 2 else None)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=axis)
    orc = MatmulOracle(lay, 32, axis)         # (axis 0, bs 64) is outside the reference's pairs: reuse the dense restatement
    orc.bsize, orc.C, orc.K, orc.w_shape = bs, CB * bs, KB * bs, bsmm.w_shape
    W = torch.as_tensor(rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)).to(dtype)
    X = torch.as_tensor(rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)).to(dtype)
    E = torch.as_tensor(rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)).to(dtype)
    Wn, Xn, En = W.float().numpy(), X.float().numpy(), E.float().numpy()
    for name, got_fn, ref in [("fprop", lambda: bsmm.fprop(X.cuda(), W.cuda(), flags=_lib.FLAG_FORCE_TC), orc.fprop_dense(Xn, Wn)),
                              ("bprop", lambda: bsmm.bprop(E.cuda(), W.cuda(), flags=_lib.FLAG_FORCE_TC), orc.bprop_dense(En, Wn))]:
        got = got_fn()
        assert _lib.device_error() == 0, "a wgmma kernel hit its bounded-wait timeout or faulted: " + _lib.device_error_text()
        assert _lib.last_kernel().startswith("wgmma_xprop"), _lib.last_kernel()
        mx, l2 = ref_errors(got.float().cpu().numpy(), ref)
        assert l2 <= (4e-3 if dtype == torch.bfloat16 else 1e-3), "%s l2 %.3e max %.3e" % (name, l2, mx)
        assert mx <= (4e-2 if dtype == torch.bfloat16 else 1e-2), "%s l2 %.3e max %.3e" % (name, l2, mx)
        # agrees with the fp32-accumulating CUDA-core path up to one output rounding
        gen = bsmm.fprop(X.cuda(), W.cuda(), flags=_lib.FLAG_FORCE_GENERIC) if name == "fprop" else \
            bsmm.bprop(E.cuda(), W.cuda(), flags=_lib.FLAG_FORCE_GENERIC)
        diff = (got.float() - gen.float()).abs().max().item()
        scale = gen.float().abs().max().item()
        assert diff <= scale * 2.0 ** -7, "wgmma vs FMA path differ by %g (scale %g)" % (diff, scale)


def test_tc_xprop_repeatable_and_stream_ordered():
    rng = np.random.default_rng(3)
    lay = layout(rng, 32, 32, 0.25)
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=1)
    W = (torch.randn(bsmm.w_shape, device="cuda") * 0.1).bfloat16()
    X = torch.randn(bsmm.i_shape(1024), device="cuda").bfloat16()
    y0 = bsmm.fprop(X, W, flags=_lib.FLAG_FORCE_TC)
    for _ in range(5):
        y = bsmm.fprop(X, W, flags=_lib.FLAG_FORCE_TC)
        assert torch.equal(y, y0)          # no atomics, no races: bit-identical run to run


@pytest.mark.parametrize("bs", [32, 64])
def test_gated_xprop_runs_on_tcgen05(bs):
    """gate folded into a scaled weight copy (bsmm_gate_weights) + wgmma kernel == oracle's gated product;
    zero gates drop their blocks exactly."""
    rng = np.random.default_rng(11)
    lay = layout(rng, 12, 10, 0.4)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=1)
    orc = MatmulOracle(lay, 32, 1)
    orc.bsize, orc.C, orc.K, orc.w_shape = bs, 12 * bs, 10 * bs, bsmm.w_shape
    N = 200
    W = torch.as_tensor(rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)).bfloat16()
    X = torch.as_tensor(rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)).bfloat16()
    E = torch.as_tensor(rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)).bfloat16()
    gate = rng.uniform(0.5, 1.5, bsmm.blocks).astype(np.float32)
    gate[rng.random(bsmm.blocks) < 0.3] = 0.0
    Wg = (W.float().numpy() * gate[:, None, None])
    g = torch.as_tensor(gate).cuda()
    y = bsmm.fprop(X.cuda(), W.cuda(), gate=g)
    assert _lib.last_kernel().startswith("wgmma_xprop")
    dx = bsmm.bprop(E.cuda(), W.cuda(), gate=g)
    assert _lib.last_kernel().startswith("wgmma_xprop") and _lib.device_error() == 0
    for got, ref in [(y, orc.fprop_dense(X.float().numpy(), Wg)), (dx, orc.bprop_dense(E.float().numpy(), Wg))]:
        err = np.abs(got.float().cpu().numpy() - ref)
        assert err.max() <= 4e-2 * np.abs(ref).max() and np.sqrt((err ** 2).sum() / (ref ** 2).sum()) <= 1e-2
    yg = bsmm.fprop(X.cuda(), W.cuda(), gate=g, flags=_lib.FLAG_FORCE_GENERIC)      # CUDA-core gated path agrees
    assert (y.float() - yg.float()).abs().max().item() <= 2.0 ** -6 * yg.float().abs().max().item()


UPDAT_CASES = [
    # CB, KB, density, N, bs, pairs
    (8, 8, 0.3, 128, 32, 1),
    (5, 37, 0.5, 200, 32, 2),      # group of 4 input blocks is ragged (5 = 4 + 1), N not a multiple of 64
    (40, 33, 0.08, 1, 32, 1),
    (20, 20, 1.0, 257, 32, 3),
    (64, 64, 0.2, 640, 32, 8),     # 8 (x, dy) pairs in one launch
    (9, 40, 0.3, 200, 16, 2),      # 16 x 16 blocks: 8 input blocks per group, 16 slots per tile, two blocks per epilogue warp
    (33, 17, 0.15, 64, 16, 1),
    (12, 12, 1.0, 130, 16, 8),
    (6, 9, 0.5, 130, 64, 1),
    (16, 17, 0.3, 64, 64, 2),
    (12, 12, 1.0, 300, 64, 1),
]


@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", UPDAT_CASES)
def test_tc_updat_matches_oracle(case, dtype, axis):
    CB, KB, density, N, bs, pairs = case
    if axis == 0:
        N = max(8, (N + 7) // 8 * 8)
    rng = np.random.default_rng(CB * 1000 + KB * 10 + N + 7)
    lay = layout(rng, CB, KB, density, empty_col=KB // 2 if density < 1 else None, empty_row=1 if density < 1 and CB > 2 else None)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=axis)
    orc = MatmulOracle(lay, 32, axis)
    orc.bsize, orc.C, orc.K, orc.w_shape = bs, CB * bs, KB * bs, bsmm.w_shape
    xs, es, ref = [], [], np.zeros(bsmm.w_shape)
    for _ in range(pairs):
        X = torch.as_tensor(rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)).to(dtype)
        E = torch.as_tensor(rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)).to(dtype)
        xs.append(X.cuda()); es.append(E.cuda())
        ref += orc.updat_dense(X.float().numpy(), E.float().numpy())
    # fp32 output: only the 16-bit INPUT rounding separates us from the oracle (which sees the same rounded inputs)
    dw32 = bsmm.updat(xs, es, dw_dtype=torch.float32, flags=_lib.FLAG_FORCE_TC)
    assert _lib.device_error() == 0, "a wgmma kernel hit its bounded-wait timeout or faulted: " + _lib.device_error_text()
    assert _lib.last_kernel().startswith("wgmma_updat"), _lib.last_kernel()
    mx, l2 = ref_errors(dw32.cpu().numpy(), ref)
    assert l2 <= 1e-5 and mx <= 1e-4, "fp32-out updat l2 %.3e max %.3e" % (l2, mx)
    # native-dtype output, alpha, and in-place accumulation (beta = 1)
    dw = bsmm.updat(xs, es, alpha=0.5, flags=_lib.FLAG_FORCE_TC)
    mx, l2 = ref_errors(dw.float().cpu().numpy(), 0.5 * ref)
    assert l2 <= (4e-3 if dtype == torch.bfloat16 else 1e-3), "updat l2 %.3e max %.3e" % (l2, mx)
    acc = dw32.clone()
    bsmm.updat(xs[:1], es[:1], dw=acc, flags=_lib.FLAG_FORCE_TC)
    ref2 = ref + orc.updat_dense(xs[0].float().cpu().numpy(), es[0].float().cpu().numpy())
    mx, l2 = ref_errors(acc.cpu().numpy(), ref2)
    assert l2 <= 1e-5, "accumulate l2 %.3e" % l2
    gate = torch.as_tensor((rng.random(bsmm.blocks) < 0.7).astype(np.float32) * 1.5).cuda()
    dwg = bsmm.updat(xs, es, gate=gate, dw_gated=True, dw_dtype=torch.float32, flags=_lib.FLAG_FORCE_TC)
    mx, l2 = ref_errors(dwg.cpu().numpy(), ref * gate.cpu().numpy()[:, None, None])
    assert l2 <= 1e-5, "gated l2 %.3e" % l2
    assert _lib.device_error() == 0


# ------------------------------------------------------------------------------------------------------------
# block-sparse transformer GEMMs on wgmma (block size 64)
from blocksparse_b200 import BlocksparseTransformer          # noqa: E402
from oracle.bst_oracle import TransformerOracle               # noqa: E402


def _bst_layout(rng, heads_l, qb, kb, density, empty_q=(), empty_k=()):
    """Random per-head layouts with equal block counts (reference requirement); query blocks `empty_q` hold no key
    block and key blocks `empty_k` no query block in any head."""
    lay = (rng.random((heads_l, qb, kb)) < density).astype(np.int32)
    for h in range(heads_l):
        for q in range(qb):
            lay[h, q, (q + h) % kb] = 1
    lay[:, list(empty_q), :] = 0
    lay[:, :, list(empty_k)] = 0
    # equal block count across heads: top up the sparser heads, outside the empty rows and columns
    target = int(lay.reshape(heads_l, -1).sum(1).max())
    for h in range(heads_l):
        free = np.argwhere(lay[h] == 0)
        free = free[~np.isin(free[:, 0], list(empty_q)) & ~np.isin(free[:, 1], list(empty_k))]
        rng.shuffle(free)
        for q, k in free[: target - int(lay[h].sum())]:
            lay[h, q, k] = 1
    return lay


def _on_poisoned_output(fn, shape, dtype, tries=8):
    """Run fn(), whose output is a fresh torch.empty(shape, dtype), on memory just filled with NaN: a tensor of that
    size is filled and freed, and the caching allocator hands the block back to the next allocation of that size, so
    an element the kernel never writes shows up as NaN. Should the allocator pick another free block instead (it
    prefers the best fit, and the freed block may have merged with a neighbour), that output is kept alive, so the
    next try cannot get it again."""
    held = []
    for _ in range(tries):
        t = torch.full(shape, float("nan"), dtype=dtype, device="cuda")
        ptr = t.data_ptr()
        del t
        c = fn()
        if c.data_ptr() == ptr:
            return c
        held.append(c)
    raise AssertionError("the output never landed on the NaN-filled block")


def _assert_zero_blocks(c, empty, bs, what):
    """rows of the dense output that belong to the given context blocks are exactly 0 (no NaN left from _poison_next)"""
    for blk in empty:
        v = c[:, blk * bs:(blk + 1) * bs]
        assert bool((v == 0).all()), "%s: output block %d is not zero-filled (max %s)" % (what, blk, v.float().abs().max().item())


BST_CASES = [
    # lut_heads, heads, q_blks, k_blks, density, head_state, batch, (empty query blocks, empty key blocks)
    (1, 2, 4, 4, 0.6, 64, 2, None),
    (1, 3, 5, 7, 0.4, 64, 1, None),        # rectangular, odd number of blocks per key column
    (2, 2, 6, 5, 0.5, 128, 2, None),       # per-head layouts, head_state 128 (two column atoms)
    (1, 4, 16, 16, 0.3, 64, 1, None),
    (4, 4, 6, 7, 0.4, 64, 2, None),        # a layout per head at head_state 64
    (1, 2, 5, 6, 0.5, 128, 1, None),       # shared layout at head_state 128
    (1, 2, 12, 12, 0.85, 64, 1, None),     # rows of 9+ blocks: the 4-stage ring wraps more than twice
    (2, 2, 7, 6, 0.5, 64, 2, ((1, 4), (2,))),   # empty query rows (NN zero-fill) and an empty key column (TN zero-fill)
]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("case", BST_CASES)
def test_tc_bst_gemms_match_oracle(case, dtype):
    lh, heads, qb, kb, density, hs, batch, holes = case
    rng = np.random.default_rng(lh * 100 + heads * 10 + qb)
    empty_q, empty_k = holes or ((), ())
    lay = _bst_layout(rng, lh, qb, kb, density, empty_q, empty_k)
    bst = BlocksparseTransformer(lay if lh > 1 else lay[0], 64, heads=heads)
    if density > 0.8:
        assert bst.nn_max > 8 and bst.tn_max > 8
    orc = TransformerOracle(lay if lh > 1 else lay[0], 64, heads=heads)
    S = heads * hs
    mk = lambda *shape: torch.as_tensor(rng.uniform(-1, 1, shape).astype(np.float32)).to(dtype)
    Q, K, V = mk(batch, qb * 64, S), mk(batch, kb * 64, S), mk(batch, kb * 64, S)
    DY = mk(batch, qb * 64, S)
    P = torch.as_tensor(rng.uniform(0, 1, (batch, heads, bst.blocks, 64, 64)).astype(np.float32)).to(dtype)
    Qn, Kn, Vn, DYn, Pn = (t.float().numpy() for t in (Q, K, V, DY, P))
    F = _lib.FLAG_FORCE_TC
    tol = 4e-3 if dtype == torch.bfloat16 else 1e-3
    for c_dtype in (torch.float32, torch.bfloat16):
        got = bst._nt(Q.cuda(), K.cuda(), c_dtype, flags=F)
        assert _lib.device_error() == 0 and _lib.last_kernel() == "wgmma_bst_nt"
        mx, l2 = ref_errors(got.float().cpu().numpy(), orc.nt(Qn, Kn))
        assert l2 <= (1e-5 if c_dtype == torch.float32 else 4e-3), "nt l2 %.3e" % l2
    got = bst._xn(P.cuda(), V.cuda(), False, flags=F)
    assert _lib.device_error() == 0 and _lib.last_kernel() == "wgmma_bst_nn"
    mx, l2 = ref_errors(got.float().cpu().numpy(), orc.nn(Pn, Vn))
    assert l2 <= tol, "nn l2 %.3e" % l2
    got = bst._xn(P.cuda(), DY.cuda(), True, flags=F)
    assert _lib.device_error() == 0 and _lib.last_kernel() == "wgmma_bst_tn"
    mx, l2 = ref_errors(got.float().cpu().numpy(), orc.tn(Pn, DYn))
    assert l2 <= tol, "tn l2 %.3e" % l2
    if holes:
        Pd, Vd, DYd = P.cuda(), V.cuda(), DY.cuda()
        for transpose, dense, empty, what in [(False, Vd, empty_q, "nn"), (True, DYd, empty_k, "tn")]:
            shape = (batch, (kb if transpose else qb) * 64, S)
            c = _on_poisoned_output(lambda: bst._xn(Pd, dense, transpose, flags=F), shape, dtype)
            assert _lib.device_error() == 0 and _lib.last_kernel() == "wgmma_bst_" + what
            _assert_zero_blocks(c, empty, 64, what)


FMA_CASES = [
    # bs, head_state, flags, sparse dtype, dense dtype: the CUDA-core NT / NN / TN kernels in 16-bit
    (8, 32, 0, torch.bfloat16, torch.bfloat16),
    (16, 64, 0, torch.float16, torch.float16),
    (32, 64, 0, torch.bfloat16, torch.bfloat16),
    (64, 32, 0, torch.float16, torch.float16),
    (64, 96, 0, torch.bfloat16, torch.bfloat16),
    (64, 256, 0, torch.float16, torch.float16),
    (64, 64, _lib.FLAG_FORCE_GENERIC, torch.bfloat16, torch.bfloat16),
    (64, 64, 0, torch.bfloat16, torch.float16),    # bf16 scores x fp16 Q / K: the fp16 attention backward's dq / dk
]


@pytest.mark.parametrize("case", FMA_CASES)
def test_fma_bst_gemms_match_oracle(case):
    """The CUDA-core attention GEMMs, elementwise against the oracle: NT (fma_dds_nt) and NN / TN (fma_sdd_xn),
    with empty query rows and an empty key column whose output rows must be zero-filled."""
    bs, hs, flags, a_dtype, dtype = case
    heads, batch, qb, kb = 2, 2, 7, 6
    rng = np.random.default_rng(bs * 1000 + hs)
    empty_q, empty_k = (1, 4), (2,)
    lay = _bst_layout(rng, 2, qb, kb, 0.5, empty_q, empty_k)
    bst = BlocksparseTransformer(lay, bs, heads=heads)
    orc = TransformerOracle(lay, bs, heads=heads)
    S = heads * hs
    mk = lambda dt, *shape: torch.as_tensor(rng.uniform(-1, 1, shape).astype(np.float32)).to(dt)
    Q, K, DY = mk(dtype, batch, qb * bs, S), mk(dtype, batch, kb * bs, S), mk(dtype, batch, qb * bs, S)
    P = mk(a_dtype, batch, heads, bst.blocks, bs, bs)
    Qn, Kn, DYn, Pn = (t.float().numpy() for t in (Q, K, DY, P))
    Qd, Kd, DYd, Pd = Q.cuda(), K.cuda(), DY.cuda(), P.cuda()
    name = lambda dt: str(dt).replace("torch.", "")

    def check(got, ref, ref_abs, k_terms, what):
        g = got.double().cpu().numpy().reshape(ref.shape)
        bound = fma_gemm_bound(ref.astype(np.float64), ref_abs.astype(np.float64), name(got.dtype), k_terms)
        err = np.abs(g - ref)
        assert np.all(err <= bound), "%s: %d elements out of bound, worst excess %.3e" % (
            what, int((err > bound).sum()), float((err - bound).max()))

    if a_dtype == dtype:            # NT takes one dtype for both dense operands
        for c_dtype in (torch.float32, torch.bfloat16):
            got = bst._nt(Qd, Kd, c_dtype, flags=flags)
            assert _lib.device_error() == 0 and _lib.last_kernel() == "fma_dds_nt", _lib.last_kernel()
            check(got, orc.nt(Qn, Kn), orc.nt(np.abs(Qn), np.abs(Kn)), hs, "nt")
    for transpose, dense, dn, empty, lmax, what in [(False, Kd, Kn, empty_q, bst.nn_max, "nn"),
                                                    (True, DYd, DYn, empty_k, bst.tn_max, "tn")]:
        bst._xn(Pd, dense, transpose, flags=flags)              # first call builds the device LUTs
        got = _on_poisoned_output(lambda: bst._xn(Pd, dense, transpose, flags=flags),
                                  (batch, (kb if transpose else qb) * bs, S), dtype)
        assert _lib.device_error() == 0 and _lib.last_kernel() == "fma_sdd_xn", _lib.last_kernel()
        assert got.dtype == dtype
        op = orc.tn if transpose else orc.nn
        ref, ref_abs = op(Pn, dn), op(np.abs(Pn), np.abs(dn))
        check(got, ref, ref_abs, lmax * bs, what)
        _assert_zero_blocks(got, empty, bs, what)


X2_CASES = [
    # CB, KB, density, N            (32 x 32 blocks; csrc/tc_xprop2.cuh wide tiles)
    (8, 8, 0.3, 128),
    (5, 37, 0.5, 200),            # odd number of input blocks (last pair is half out of range), ragged N
    (7, 20, 1.0, 257),            # dense: every pair-group overflows its W slots and is split
    (40, 33, 0.08, 1),
    (6, 32, -1, 136),             # checkerboard: 8 isolated runs per half (the record's run limit)
    (64, 64, 0.2, 640),
]


@pytest.mark.parametrize("variant", [1, 2, 3])
@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", X2_CASES)
def test_tc_xprop2_variants_match_oracle(case, dtype, axis, variant, monkeypatch):
    """Every variant of the wide-activation-tile kernel (forced through matmul._X2_FORCE), both feature axes."""
    import blocksparse_b200.matmul as mm
    monkeypatch.setattr(mm, "_X2_FORCE", variant)
    CB, KB, density, N = case
    if axis == 0:
        N = max(8, (N + 7) // 8 * 8)
    rng = np.random.default_rng(CB * 1000 + KB * 10 + N)
    if density < 0:
        lay = ((np.arange(CB)[:, None] + np.arange(KB)[None, :]) % 2).astype(np.int32)
    else:
        lay = layout(rng, CB, KB, density, empty_col=KB // 2 if density < 1 else None, empty_row=1 if density < 1 and CB > 2 else None)
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=axis)
    orc = MatmulOracle(lay, 32, axis)
    W = torch.as_tensor(rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)).to(dtype)
    X = torch.as_tensor(rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)).to(dtype)
    E = torch.as_tensor(rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)).to(dtype)
    Wn, Xn, En = W.float().numpy(), X.float().numpy(), E.float().numpy()
    for name, fn, inp, ref in [("fprop", bsmm.fprop, X, orc.fprop_dense(Xn, Wn)), ("bprop", bsmm.bprop, E, orc.bprop_dense(En, Wn))]:
        got = fn(inp.cuda(), W.cuda(), flags=_lib.FLAG_FORCE_TC)
        assert _lib.device_error() == 0, _lib.device_error_text()
        assert _lib.last_kernel() == "wgmma_xprop2_bs32", _lib.last_kernel()
        mx, l2 = ref_errors(got.float().cpu().numpy(), ref)
        # max metric = worst element over MEAN magnitude: the bf16 output rounding alone (2^-9 of the largest element,
        # max/mean ~ 20 for these N(0,1) inputs at 4-10 terms per sum) reaches ~4e-2; the l2 bound is the meaningful one
        assert l2 <= (4e-3 if dtype == torch.bfloat16 else 1e-3) and mx <= (6e-2 if dtype == torch.bfloat16 else 1e-2), \
            "%s variant %d: l2 %.3e max %.3e" % (name, variant, l2, mx)
        again = fn(inp.cuda(), W.cuda(), flags=_lib.FLAG_FORCE_TC)
        assert torch.equal(got, again)            # deterministic accumulation order


def test_cuda_graph_capture_and_replay():
    """The launches take their tensor maps by value and read schedules from device memory, so a step can be captured in a
    CUDA graph: replaying it (no Python, no host-side descriptor work) reproduces the eager results bit for bit."""
    rng = np.random.default_rng(21)
    lay = layout(rng, 32, 32, 0.25)
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=1)
    N = 512
    W = (torch.randn(bsmm.w_shape, device="cuda") * 0.1).bfloat16()
    X = torch.randn(bsmm.i_shape(N), device="cuda").bfloat16()
    E = torch.randn(bsmm.o_shape(N), device="cuda").bfloat16()
    ref = (bsmm.fprop(X, W), bsmm.bprop(E, W), bsmm.updat([X], [E]))      # also warms the schedule / tensor-map caches
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            bsmm.fprop(X, W); bsmm.bprop(E, W); bsmm.updat([X], [E])
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = bsmm.fprop(X, W)
        dx = bsmm.bprop(E, W)
        dw = bsmm.updat([X], [E])
    for _ in range(3):
        y.zero_(); dx.zero_(); dw.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, ref[0]) and torch.equal(dx, ref[1]) and torch.equal(dw, ref[2])
    # new data in the captured input buffers
    X.copy_(torch.randn_like(X.float()).bfloat16())
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, bsmm.fprop(X, W))
    assert _lib.device_error() == 0


@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", [(8, 8, 0.3, 128), (40, 33, 0.08, 1), (64, 64, 0.2, 640), (9, 47, 0.3, 200), (128, 128, 0.25, 1024)])
def test_tc_xprop_pair_tiles_match_oracle(case, dtype, axis, monkeypatch):
    """2-CTA clusters sharing every W block by TMA multicast (BSMM_PAIR_TILES, csrc/tc.cuh CL = 2): same results, bit for
    bit, as the single-CTA kernel (each output block still sees its MMAs in LUT order)."""
    import blocksparse_b200.matmul as mm
    CB, KB, density, N = case
    if axis == 0:
        N = max(8, (N + 7) // 8 * 8)
    rng = np.random.default_rng(CB * 1000 + KB * 10 + N)
    lay = layout(rng, CB, KB, density, empty_col=KB // 2, empty_row=1)
    W = torch.as_tensor(rng.normal(0, 0.1, (int(lay.sum()), 32, 32)).astype(np.float32)).to(dtype).cuda()
    res = {}
    for pair in (0, 1):
        monkeypatch.setattr(mm, "_PAIR_TILES", pair)
        bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=axis)
        X = torch.as_tensor(np.random.default_rng(1).normal(0, 1, bsmm.i_shape(N)).astype(np.float32)).to(dtype).cuda()
        E = torch.as_tensor(np.random.default_rng(2).normal(0, 1, bsmm.o_shape(N)).astype(np.float32)).to(dtype).cuda()
        y = bsmm.fprop(X, W, flags=_lib.FLAG_FORCE_TC); k1 = _lib.last_kernel()
        dx = bsmm.bprop(E, W, flags=_lib.FLAG_FORCE_TC); k2 = _lib.last_kernel()
        assert _lib.device_error() == 0, _lib.device_error_text()
        assert k1 == k2 == ("wgmma_xprop_bs32_pair" if pair else "wgmma_xprop_bs32"), (k1, k2)
        res[pair] = (y, dx)
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    orc = MatmulOracle(lay, 32, axis)
    mx, l2 = ref_errors(res[1][0].float().cpu().numpy(), orc.fprop_dense(X.float().cpu().numpy(), W.float().cpu().numpy()))
    assert l2 <= (4e-3 if dtype == torch.bfloat16 else 1e-3), "pair-tile fprop l2 %.3e" % l2


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_bs8_runs_padded_on_tcgen05(dtype, axis):
    """8 x 8 blocks: 2 x 2 neighbourhoods padded into 16 x 16 super-blocks (csrc/wutil.cuh pad/unpad) and run by the wgmma
    kernels; fprop / bprop / updat (alpha, accumulate, gate) against the oracle and against the CUDA-core path."""
    rng = np.random.default_rng(8 + axis)
    lay = layout(rng, 20, 14, 0.3, empty_col=3, empty_row=5)
    bsmm = BlocksparseMatMul(lay, block_size=8, feature_axis=axis)
    assert bsmm._shadow is not None and bsmm._shadow.bsize == 16
    orc = MatmulOracle(lay, 8, 0)
    orc.axis = axis
    N = 136
    W = torch.as_tensor(rng.normal(0, 0.2, bsmm.w_shape).astype(np.float32)).to(dtype)
    X = torch.as_tensor(rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)).to(dtype)
    E = torch.as_tensor(rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)).to(dtype)
    Wn, Xn, En = W.float().numpy(), X.float().numpy(), E.float().numpy()
    gate = (rng.random(bsmm.blocks) < 0.7).astype(np.float32) * 1.5
    g = torch.as_tensor(gate).cuda()
    tol = 4e-3 if dtype == torch.bfloat16 else 1e-3
    for name, got, ref in [("fprop", bsmm.fprop(X.cuda(), W.cuda()), orc.fprop_dense(Xn, Wn)),
                           ("bprop", bsmm.bprop(E.cuda(), W.cuda()), orc.bprop_dense(En, Wn)),
                           ("fprop gated", bsmm.fprop(X.cuda(), W.cuda(), gate=g), orc.fprop_dense(Xn, Wn * gate[:, None, None]))]:
        assert _lib.last_kernel() == "wgmma_xprop_bs16", _lib.last_kernel()
        mx, l2 = ref_errors(got.float().cpu().numpy(), ref)
        assert l2 <= tol, "%s l2 %.3e" % (name, l2)
    ref_dw = orc.updat_dense(Xn, En)
    dw = bsmm.updat([X.cuda()], [E.cuda()], dw_dtype=torch.float32)
    assert _lib.last_kernel() == "unpad_blocks"
    mx, l2 = ref_errors(dw.cpu().numpy(), ref_dw)
    assert l2 <= 1e-5, "updat l2 %.3e" % l2
    bsmm.updat([X.cuda()], [E.cuda()], dw=dw, alpha=0.5)                           # in-place accumulate
    mx, l2 = ref_errors(dw.cpu().numpy(), 1.5 * ref_dw)
    assert l2 <= 1e-5, "accumulate l2 %.3e" % l2
    dwg = bsmm.updat([X.cuda()], [E.cuda()], gate=g, dw_gated=True, dw_dtype=torch.float32)
    mx, l2 = ref_errors(dwg.cpu().numpy(), ref_dw * gate[:, None, None])
    assert l2 <= 1e-5
    fma = bsmm.fprop(X.cuda(), W.cuda(), flags=_lib.FLAG_FORCE_GENERIC)
    assert _lib.last_kernel().startswith("fma_")
    assert (fma.float() - bsmm.fprop(X.cuda(), W.cuda()).float()).abs().max().item() <= 2.0 ** -7 * fma.float().abs().max().item()
    assert _lib.device_error() == 0
