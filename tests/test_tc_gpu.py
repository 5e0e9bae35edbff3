"""GPU parity of the wgmma kernel families (forced with BSMM_FLAG_FORCE_TC so a silent fall-back to the
CUDA-core kernels cannot pass) against the oracle, at sizes the NumPy loops finish in seconds.

The matmul results are checked elementwise against the float64 oracle with mma_gemm_bound (tests/_util.py), each on
memory filled with NaN first, so an element the kernel never writes fails too. Every family also has a case with
operands uniform in (0, 1): there the bound is within a few eps32 of one output rounding, tight enough to tell
round-to-nearest from truncation, which sign-mixed data hides behind cancellation."""
import numpy as np
import pytest
import torch

from tests._util import (_on_poisoned_output, assert_within, assert_zero_filled, bst_dense, bst_terms, dtype_name,
                         feature_terms, fma_gemm_bound, mma_gemm_bound, oracle_dense, record_kernels, ref_errors)
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
    # CB, KB, density, N, bs[, "pos": operands uniform in (0, 1)]
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
    (10, 12, 0.4, 136, 32, "pos"),
    (9, 14, 0.4, 128, 16, "pos"),
    (6, 9, 0.5, 130, 64, "pos"),
]


def operands(rng, bsmm, N, dtype, positive=False):
    """W, X, E on the host in dtype: N(0, 0.1) weights and N(0, 1) activations, or all uniform in (0, 1)."""
    draw = (lambda shape, s: rng.uniform(0, 1, shape)) if positive else (lambda shape, s: rng.normal(0, s, shape))
    return tuple(torch.as_tensor(draw(shape, s).astype(np.float32)).to(dtype)
                 for shape, s in ((bsmm.w_shape, 0.1), (bsmm.i_shape(N), 1), (bsmm.o_shape(N), 1)))


def check_xprop(orc, lay, bs, bprop, inp, W, run, what, k=None, family="wgmma_xprop"):
    """run() (an fprop / bprop of inp and W, already on the device) on NaN-poisoned output memory: every element is
    written, the output blocks of lay (block size bs) with an empty LUT row are exactly zero, and the result is within
    mma_gemm_bound of the float64 oracle. k: k_terms (default: bs x the LUT row length of each output block of lay).
    Returns the output and the kernel that ran."""
    name = dtype_name(inp.dtype)
    inp_n, Wn = inp.float().numpy(), W.float().numpy()
    op = "bprop" if bprop else "fprop"
    ref, ref_abs = oracle_dense(orc, op, inp_n, Wn), oracle_dense(orc, op, np.abs(inp_n), np.abs(Wn))
    got = _on_poisoned_output(run)
    assert _lib.device_error() == 0, "a wgmma kernel hit its bounded-wait timeout or faulted: " + _lib.device_error_text()
    kern = _lib.last_kernel()
    if k is None:
        k = feature_terms(lay, bs, bprop, orc.axis)
    empty = np.nonzero((np.asarray(lay) != 0).sum(axis=1 if bprop else 0) == 0)[0]
    assert_zero_filled(got, empty, bs, orc.axis, "%s (%s)" % (what, kern))
    assert_within(got, ref, mma_gemm_bound(ref, ref_abs, name, k), "%s (%s)" % (what, kern), ref_abs, k, name, family)
    mx, l2 = ref_errors(got.double().cpu().numpy(), ref)
    assert l2 <= (4e-3 if inp.dtype == torch.bfloat16 else 1e-3), "%s (%s) l2 %.3e" % (what, kern, l2)
    return got, kern


@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", CASES)
def test_tc_xprop_matches_oracle(case, dtype, axis):
    CB, KB, density, N, bs, *opt = case
    if axis == 0:
        N = max(8, (N + 7) // 8 * 8)          # TMA needs a 16-byte row pitch when the minibatch is the inner dim
    rng = np.random.default_rng(CB * 1000 + KB * 10 + N)
    lay = layout(rng, CB, KB, density, empty_col=KB // 2 if density < 1 else None, empty_row=1 if density < 1 and CB > 2 else None)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=axis)
    orc = MatmulOracle(lay, 32, axis)         # (axis 0, bs 64) is outside the reference's pairs: reuse the dense restatement
    orc.bsize, orc.C, orc.K, orc.w_shape = bs, CB * bs, KB * bs, bsmm.w_shape
    W, X, E = operands(rng, bsmm, N, dtype, "pos" in opt)
    Wd = W.cuda()
    for bprop, inp in [(False, X), (True, E)]:
        fn = bsmm.bprop if bprop else bsmm.fprop
        xd = inp.cuda()
        got, kern = check_xprop(orc, lay, bs, bprop, inp, W, lambda: fn(xd, Wd, flags=_lib.FLAG_FORCE_TC),
                                "bprop" if bprop else "fprop")
        assert kern.startswith("wgmma_xprop"), kern
        # agrees with the fp32-accumulating CUDA-core path up to one output rounding
        gen = fn(xd, Wd, flags=_lib.FLAG_FORCE_GENERIC)
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
    """gate folded into a scaled weight copy (bsmm_gate_weights) + wgmma kernel == oracle's product with that copy
    (tests/test_bsmm_paths_gpu.py checks the copy bit for bit); zero gates drop their blocks exactly."""
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
    Wg = (W.float() * torch.as_tensor(gate)[:, None, None]).bfloat16()
    g = torch.as_tensor(gate).cuda()
    Xd, Ed, Wd = X.cuda(), E.cuda(), W.cuda()
    y, kern = check_xprop(orc, lay, bs, False, X, Wg, lambda: bsmm.fprop(Xd, Wd, gate=g), "gated fprop")
    assert kern.startswith("wgmma_xprop"), kern
    _, kern = check_xprop(orc, lay, bs, True, E, Wg, lambda: bsmm.bprop(Ed, Wd, gate=g), "gated bprop")
    assert kern.startswith("wgmma_xprop"), kern
    yg = bsmm.fprop(Xd, Wd, gate=g, flags=_lib.FLAG_FORCE_GENERIC)      # CUDA-core gated path agrees
    assert (y.float() - yg.float()).abs().max().item() <= 2.0 ** -6 * yg.float().abs().max().item()


UPDAT_CASES = [
    # CB, KB, density, N, bs, pairs[, "pos": operands uniform in (0, 1) | "sms3": host schedule balanced for 3 SMs]
    (8, 8, 0.3, 128, 32, 1),
    (5, 37, 0.5, 200, 32, 2),      # group of 4 input blocks is ragged (5 = 4 + 1), N not a multiple of 64
    (40, 33, 0.08, 1, 32, 1),
    (20, 20, 1.0, 257, 32, 3),     # 20 kept output blocks per group: three windows of <= 8 slots
    (64, 64, 0.2, 640, 32, 8),     # 8 (x, dy) pairs in one launch
    (9, 40, 0.3, 200, 16, 2),      # 16 x 16 blocks: 8 input blocks per group, 16 slots per tile, two blocks per epilogue warp
    (33, 17, 0.15, 64, 16, 1),
    (12, 12, 1.0, 130, 16, 8),
    (6, 9, 0.5, 130, 64, 1),
    (16, 17, 0.3, 64, 64, 2),
    (12, 12, 1.0, 300, 64, 1),     # 12 kept output blocks per group: three windows of 4 slots
    (10, 12, 0.4, 136, 32, 3, "pos"),
    (9, 14, 0.4, 128, 16, 2, "pos"),
    (6, 9, 0.5, 130, 64, 1, "pos"),
    # "sms3" checks _balance_windows' extra windows only: the launch grid stays the device's (BSMM_SM_MARGIN), so each
    # CTA still runs one tile. tests/test_updat_persistent_gpu.py runs CTAs over several tiles.
    (9, 40, 0.3, 200, 16, 2, "sms3"),
    (64, 64, 0.2, 256, 32, 2, "sms3"),
]


@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", UPDAT_CASES)
def test_tc_updat_matches_oracle(case, dtype, axis, monkeypatch):
    CB, KB, density, N, bs, pairs, *opt = case
    if axis == 0:
        N = max(8, (N + 7) // 8 * 8)
    rng = np.random.default_rng(CB * 1000 + KB * 10 + N + 7)
    lay = layout(rng, CB, KB, density, empty_col=KB // 2 if density < 1 else None, empty_row=1 if density < 1 and CB > 2 else None)
    dev = torch.device("cuda", torch.cuda.current_device())
    if "sms3" in opt:               # the schedule is cached per object: build a fresh one for 3 SMs
        default_tiles = BlocksparseMatMul(lay, block_size=bs, feature_axis=axis)._device_luts(dev)["updat_tiles"]
        monkeypatch.setattr(_lib, "grid_sms", lambda d: 3)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=axis)
    if "sms3" in opt:
        assert bsmm._device_luts(dev)["updat_tiles"] > default_tiles
    orc = MatmulOracle(lay, 32, axis)
    orc.bsize, orc.C, orc.K, orc.w_shape = bs, CB * bs, KB * bs, bsmm.w_shape
    draw = (lambda shape: rng.uniform(0, 1, shape)) if "pos" in opt else (lambda shape: rng.normal(0, 1, shape))
    xs, es, ref, ref_abs = [], [], 0.0, 0.0
    for _ in range(pairs):
        X = torch.as_tensor(draw(bsmm.i_shape(N)).astype(np.float32)).to(dtype)
        E = torch.as_tensor(draw(bsmm.o_shape(N)).astype(np.float32)).to(dtype)
        xs.append(X.cuda()); es.append(E.cuda())
        Xn, En = X.float().numpy(), E.float().numpy()
        ref = ref + oracle_dense(orc, "updat", Xn, En)
        ref_abs = ref_abs + oracle_dense(orc, "updat", np.abs(Xn), np.abs(En))
    k, name, F = N * pairs, dtype_name(dtype), _lib.FLAG_FORCE_TC

    def check(got, r, a, k_terms, extra, what, max_tol=np.inf):
        assert _lib.device_error() == 0, "a wgmma kernel hit its bounded-wait timeout or faulted: " + _lib.device_error_text()
        assert _lib.last_kernel().startswith("wgmma_updat"), _lib.last_kernel()
        assert not bool(torch.isnan(got).any()), "%s: %d dw elements never written" % (what, int(torch.isnan(got).sum()))
        out = dtype_name(got.dtype)
        assert_within(got, r, mma_gemm_bound(r, a, out, k_terms, extra), what, a, k_terms, out, "wgmma_updat")
        # the aggregate metrics too: on sign-mixed data the linear worst-case bound is loose, and l2 is the tighter
        # statistical guard for an fp32 dw (only the 16-bit input rounding separates it from the oracle)
        mx, l2 = ref_errors(got.double().cpu().numpy(), r)
        assert l2 <= {"float32": 1e-5, "bfloat16": 4e-3, "float16": 1e-3}[out] and mx <= max_tol, \
            "%s l2 %.3e max %.3e" % (what, l2, mx)

    # fresh outputs on NaN-poisoned memory: every dw element is written. fp32 dw, then 16-bit dw with alpha.
    dw32 = _on_poisoned_output(lambda: bsmm.updat(xs, es, dw_dtype=torch.float32, flags=F))
    check(dw32, ref, ref_abs, k, 0, "fp32 dw", max_tol=1e-4)
    dw = _on_poisoned_output(lambda: bsmm.updat(xs, es, alpha=0.5, flags=F))
    check(dw, 0.5 * ref, 0.5 * ref_abs, k, 1, "%s dw, alpha 0.5" % name)
    # in-place accumulation (beta = 1), into an fp32 and into a 16-bit dw
    X0, E0 = xs[0].float().cpu().numpy(), es[0].float().cpu().numpy()
    ref0, abs0 = oracle_dense(orc, "updat", X0, E0), oracle_dense(orc, "updat", np.abs(X0), np.abs(E0))
    for base in (dw32, dw):
        acc = base.clone()
        old = base.double().cpu().numpy()
        bsmm.updat(xs[:1], es[:1], dw=acc, flags=F)
        check(acc, old + ref0, np.abs(old) + abs0, N, 1, "accumulate into %s dw" % dtype_name(base.dtype))
    # gated dw with alpha != 1, accumulated: g = alpha * gate, then a * g + old (zero gates leave old untouched)
    gate = ((rng.random(bsmm.blocks) < 0.7) * rng.uniform(0.5, 1.5, bsmm.blocks)).astype(np.float32)
    g, gn = torch.as_tensor(gate).cuda(), gate.astype(np.float64)[:, None, None]
    for base in (dw32, dw):
        acc = base.clone()
        old = base.double().cpu().numpy()
        bsmm.updat(xs, es, dw=acc, alpha=0.75, gate=g, dw_gated=True, flags=F)
        check(acc, old + 0.75 * gn * ref, np.abs(old) + 0.75 * gn * ref_abs, k, 3,
              "gated, alpha 0.75, accumulate into %s dw" % dtype_name(base.dtype))


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


def _assert_zero_blocks(c, empty, bs, what):
    """rows of the dense output that belong to the given context blocks are exactly 0 (no NaN left from _poison_next)"""
    for blk in empty:
        v = c[:, blk * bs:(blk + 1) * bs]
        assert bool((v == 0).all()), "%s: output block %d is not zero-filled (max %s)" % (what, blk, v.float().abs().max().item())


BST_CASES = [
    # lut_heads, heads, q_blks, k_blks, density, head_state, batch, (empty query blocks, empty key blocks)
    # [, "pos": operands uniform in (0, 1)]. density "tril": the causal block layout, rows and columns of 1 .. q_blks.
    (1, 2, 4, 4, 0.6, 64, 2, None),
    (1, 3, 5, 7, 0.4, 64, 1, None),        # rectangular, odd number of blocks per key column
    (2, 2, 6, 5, 0.5, 128, 2, None),       # per-head layouts, head_state 128 (two column atoms)
    (1, 4, 16, 16, 0.3, 64, 1, None),
    (4, 4, 6, 7, 0.4, 64, 2, None),        # a layout per head at head_state 64
    (1, 2, 5, 6, 0.5, 128, 1, None),       # shared layout at head_state 128
    (1, 2, 12, 12, 0.85, 64, 1, None),     # rows of 9+ blocks: the 4-stage ring wraps more than twice
    (2, 2, 7, 6, 0.5, 64, 2, ((1, 4), (2,))),   # empty query rows (NN zero-fill) and an empty key column (TN zero-fill)
    (1, 2, 6, 6, "tril", 64, 2, None),     # rows of exactly 1, 4 and 5 entries: the ring's first refill is entry 4
    (1, 1, 24, 24, 1.0, 64, 1, None),      # dense: rows of 24, the ring wraps six times
    (3, 3, 5, 8, 0.4, 64, 3, None),        # batch 3, ctx_q != ctx_k, a layout per head: offsets cannot cancel
    (2, 2, 7, 6, 0.5, 128, 2, ((1, 4), (2,))),  # head_state 128 with per-head layouts and holes
    (1, 2, 5, 5, 0.6, 64, 2, None, "pos"),
    (2, 2, 6, 5, 0.5, 128, 2, None, "pos"),
]


def bst_case_layout(case):
    """The layout of a BST_CASES entry ((lut_heads, q_blks, k_blks) array) and the rng that drew it, which then draws
    the operands."""
    lh, heads, qb, kb, density, hs, batch, holes, *opt = case
    rng = np.random.default_rng(lh * 100 + heads * 10 + qb)
    if density == "tril":
        return np.tril(np.ones((lh, qb, kb), np.int32)), rng
    empty_q, empty_k = holes or ((), ())
    return _bst_layout(rng, lh, qb, kb, density, empty_q, empty_k), rng


BST_DTYPES = (torch.float16, torch.bfloat16)               # dense operands, and the sparse one of NN / TN
BST_NT_OUT = ((torch.float32, 1e-5), (torch.bfloat16, 4e-3), (torch.float16, 1e-3))   # NT output dtype, l2 limit


@pytest.mark.parametrize("dtype", BST_DTYPES)
@pytest.mark.parametrize("case", BST_CASES)
def test_tc_bst_gemms_match_oracle(case, dtype):
    """The wgmma attention GEMMs (csrc/tc_bst.cuh): NT at every output dtype, NN and TN, each on NaN-poisoned output
    memory and elementwise within mma_gemm_bound of the float64 product (k_terms: head_state for NT, 64 x the LUT row
    length of each output block, per head, for NN / TN). The relative l2 error against the same reference is kept as a
    second metric."""
    lh, heads, qb, kb, density, hs, batch, holes, *opt = case
    lay, rng = bst_case_layout(case)
    empty_q, empty_k = holes or ((), ())
    bst = BlocksparseTransformer(lay if lh > 1 else lay[0], 64, heads=heads)
    if density == 1.0:
        assert bst.nn_max == kb and bst.tn_max == qb
    elif density != "tril" and density > 0.8:
        assert bst.nn_max > 8 and bst.tn_max > 8
    orc = TransformerOracle(lay if lh > 1 else lay[0], 64, heads=heads)
    S = heads * hs
    lo = 0 if "pos" in opt else -1
    mk = lambda *shape: torch.as_tensor(rng.uniform(lo, 1, shape).astype(np.float32)).to(dtype)
    Q, K, V = mk(batch, qb * 64, S), mk(batch, kb * 64, S), mk(batch, kb * 64, S)
    DY = mk(batch, qb * 64, S)
    P = torch.as_tensor(rng.uniform(0, 1, (batch, heads, bst.blocks, 64, 64)).astype(np.float32)).to(dtype)
    Qn, Kn, Vn, DYn, Pn = (t.float().numpy() for t in (Q, K, V, DY, P))
    Qd, Kd, Vd, DYd, Pd = Q.cuda(), K.cuda(), V.cuda(), DY.cuda(), P.cuda()
    F = _lib.FLAG_FORCE_TC
    tol = 4e-3 if dtype == torch.bfloat16 else 1e-3

    def check(run, op, a, b, kern, l2_tol):
        got = _on_poisoned_output(run)
        assert _lib.device_error() == 0, "a wgmma kernel hit its bounded-wait timeout or faulted: " + _lib.device_error_text()
        assert _lib.last_kernel() == kern, _lib.last_kernel()
        out = dtype_name(got.dtype)
        what = "%s -> %s (%s)" % (op, out, kern)
        assert not bool(torch.isnan(got).any()), "%s: %d elements never written" % (what, int(torch.isnan(got).sum()))
        ref, ref_abs = bst_dense(orc, op, a, b, with_abs=True)
        k = bst_terms(orc, op, hs)
        assert_within(got, ref, mma_gemm_bound(ref, ref_abs, out, k), what, ref_abs, k, out, "wgmma_bst")
        mx, l2 = ref_errors(got.double().cpu().numpy(), ref)
        assert l2 <= l2_tol, "%s l2 %.3e" % (what, l2)
        return got

    for c_dtype, l2_tol in BST_NT_OUT:
        check(lambda: bst._nt(Qd, Kd, c_dtype, flags=F), "nt", Qn, Kn, "wgmma_bst_nt", l2_tol)
    c = check(lambda: bst._xn(Pd, Vd, False, flags=F), "nn", Pn, Vn, "wgmma_bst_nn", tol)
    _assert_zero_blocks(c, empty_q, 64, "nn")
    c = check(lambda: bst._xn(Pd, DYd, True, flags=F), "tn", Pn, DYn, "wgmma_bst_tn", tol)
    _assert_zero_blocks(c, empty_k, 64, "tn")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_bst_misaligned_views_take_the_cuda_core_route(dtype):
    """Dense operands at an odd element offset into a larger buffer are legal torch, but TMA needs 16-byte aligned
    bases: the public nt_op / nn_op / tn_op run them on the CUDA-core kernels, elementwise within fma_gemm_bound."""
    lay = np.tril(np.ones((4, 4), np.int32))
    heads, hs, batch = 2, 64, 2
    bst = BlocksparseTransformer(lay, 64, heads=heads)
    orc = TransformerOracle(lay, 64, heads=heads)
    rng = np.random.default_rng(31)
    shape = (batch, 4 * 64, heads * hs)
    n = int(np.prod(shape))

    def misaligned(offset):
        host = torch.as_tensor(rng.uniform(-1, 1, shape).astype(np.float32)).to(dtype)
        t = torch.zeros(n + offset, dtype=dtype, device="cuda")[offset:].view(shape)
        t.copy_(host.cuda())
        assert t.is_contiguous() and t.data_ptr() % 16
        return t, host.float().numpy()
    (Q, Qn), (K, Kn), (DY, DYn) = misaligned(1), misaligned(3), misaligned(5)
    P = torch.as_tensor(rng.uniform(0, 1, (batch, heads, bst.blocks, 64, 64)).astype(np.float32)).to(dtype)
    Pn, Pd = P.float().numpy(), P.cuda()
    for run, op, a, b, kern in [(lambda: bst.nt_op(Q, K), "nt", Qn, Kn, "fma_dds_nt"),
                                (lambda: bst.nn_op(Pd, K), "nn", Pn, Kn, "fma_sdd_xn"),
                                (lambda: bst.tn_op(Pd, DY), "tn", Pn, DYn, "fma_sdd_xn")]:
        got = _on_poisoned_output(run)
        assert _lib.device_error() == 0, _lib.device_error_text()
        assert _lib.last_kernel() == kern, (op, _lib.last_kernel())
        assert not bool(torch.isnan(got).any()), "%s: elements never written" % op
        ref, ref_abs = bst_dense(orc, op, a, b, with_abs=True)
        out = dtype_name(got.dtype)
        k = bst_terms(orc, op, hs)
        assert_within(got, ref, fma_gemm_bound(ref, ref_abs, out, k), "misaligned %s (%s)" % (op, kern))


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

    def check(got, ref, ref_abs, k_terms, what):
        g = got.double().cpu().numpy().reshape(ref.shape)
        bound = fma_gemm_bound(ref.astype(np.float64), ref_abs.astype(np.float64), dtype_name(got.dtype), k_terms)
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
        got = _on_poisoned_output(lambda: bst._xn(Pd, dense, transpose, flags=flags))
        assert _lib.device_error() == 0 and _lib.last_kernel() == "fma_sdd_xn", _lib.last_kernel()
        assert got.dtype == dtype
        op = orc.tn if transpose else orc.nn
        ref, ref_abs = op(Pn, dn), op(np.abs(Pn), np.abs(dn))
        check(got, ref, ref_abs, lmax * bs, what)
        _assert_zero_blocks(got, empty, bs, what)


X2_CASES = [
    # CB, KB, density, N[, "pos"]    (32 x 32 blocks; csrc/tc_xprop2.cuh wide tiles)
    (8, 8, 0.3, 128),
    (5, 37, 0.5, 200),            # odd number of input blocks (last pair is half out of range), ragged N
    (7, 20, 1.0, 257),            # dense: every pair-group overflows its W slots and is split
    (40, 33, 0.08, 1),
    (6, 32, -1, 136),             # checkerboard: 8 isolated runs per half (the record's run limit)
    (64, 64, 0.2, 640),
    (10, 12, 0.4, 136, "pos"),
]


def wide_terms(lay, bprop, tb, axis):
    """k_terms of the wide-tile kernel: every output block of a tile of tb walks the tile's merged LUT row, one entry
    per input block that any of them consumes."""
    m = np.asarray(lay) != 0
    m = m if bprop else m.T                                  # (output blocks, input blocks)
    merged = [int(m[t:t + tb].any(axis=0).sum()) for t in range(0, m.shape[0], tb)]
    kf = np.repeat(np.repeat(merged, tb)[:m.shape[0]] * 32, 32).astype(np.float64)
    return kf[None, :] if axis else kf[:, None]


@pytest.mark.parametrize("variant", [1, 2, 3])
@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", X2_CASES)
def test_tc_xprop2_variants_match_oracle(case, dtype, axis, variant, monkeypatch):
    """Every variant of the wide-activation-tile kernel (forced through matmul._X2_FORCE), both feature axes."""
    import blocksparse_b200.matmul as mm
    monkeypatch.setattr(mm, "_X2_FORCE", variant)
    CB, KB, density, N, *opt = case
    if axis == 0:
        N = max(8, (N + 7) // 8 * 8)
    rng = np.random.default_rng(CB * 1000 + KB * 10 + N)
    if density < 0:
        lay = ((np.arange(CB)[:, None] + np.arange(KB)[None, :]) % 2).astype(np.int32)
    else:
        lay = layout(rng, CB, KB, density, empty_col=KB // 2 if density < 1 else None, empty_row=1 if density < 1 and CB > 2 else None)
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=axis)
    orc = MatmulOracle(lay, 32, axis)
    W, X, E = operands(rng, bsmm, N, dtype, "pos" in opt)
    Wd = W.cuda()
    for bprop, inp in [(False, X), (True, E)]:
        fn = bsmm.bprop if bprop else bsmm.fprop
        xd = inp.cuda()
        got, kern = check_xprop(orc, lay, 32, bprop, inp, W, lambda: fn(xd, Wd, flags=_lib.FLAG_FORCE_TC),
                                "%s variant %d" % ("bprop" if bprop else "fprop", variant),
                                k=wide_terms(lay, bprop, mm._X2_VARIANTS[variant], axis), family="wgmma_xprop2")
        assert kern == "wgmma_xprop2_bs32", kern
        again = fn(xd, Wd, flags=_lib.FLAG_FORCE_TC)
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


PAIR_CASES = [
    # CB, KB, density, N[, "pos"]
    (8, 8, 0.3, 128),
    (40, 33, 0.08, 1),
    (64, 64, 0.2, 640),
    (9, 47, 0.3, 200),
    (128, 128, 0.25, 1024),
    (12, 20, 0.3, 300),           # three 128-row tiles: the last cluster's partner CTA lies wholly past N
    (10, 12, 0.4, 136, "pos"),
]


@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", PAIR_CASES)
def test_tc_xprop_pair_tiles_match_oracle(case, dtype, axis, monkeypatch):
    """2-CTA clusters sharing every W block by TMA multicast (BSMM_PAIR_TILES, csrc/tc.cuh CL = 2): same results, bit for
    bit, as the single-CTA kernel (each output block still sees its MMAs in LUT order), and within the bound of the
    oracle for fprop and bprop."""
    import blocksparse_b200.matmul as mm
    CB, KB, density, N, *opt = case
    positive = "pos" in opt
    if axis == 0:
        N = max(8, (N + 7) // 8 * 8)
    rng = np.random.default_rng(CB * 1000 + KB * 10 + N)
    lay = layout(rng, CB, KB, density, empty_col=KB // 2, empty_row=1)
    w_shape = (int(lay.sum()), 32, 32)
    W = torch.as_tensor((rng.uniform(0, 1, w_shape) if positive else rng.normal(0, 0.1, w_shape)).astype(np.float32)).to(dtype)
    orc = MatmulOracle(lay, 32, axis)
    Wd = W.cuda()
    res = {}
    for pair in (0, 1):
        monkeypatch.setattr(mm, "_PAIR_TILES", pair)
        bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=axis)
        draw = (lambda r, shape: r.uniform(0, 1, shape)) if positive else (lambda r, shape: r.normal(0, 1, shape))
        X = torch.as_tensor(draw(np.random.default_rng(1), bsmm.i_shape(N)).astype(np.float32)).to(dtype)
        E = torch.as_tensor(draw(np.random.default_rng(2), bsmm.o_shape(N)).astype(np.float32)).to(dtype)
        Xd, Ed = X.cuda(), E.cuda()
        if pair:
            y, k1 = check_xprop(orc, lay, 32, False, X, W, lambda: bsmm.fprop(Xd, Wd, flags=_lib.FLAG_FORCE_TC), "fprop",
                                family="wgmma_xprop_pair")
            dx, k2 = check_xprop(orc, lay, 32, True, E, W, lambda: bsmm.bprop(Ed, Wd, flags=_lib.FLAG_FORCE_TC), "bprop",
                                 family="wgmma_xprop_pair")
        else:
            y = bsmm.fprop(Xd, Wd, flags=_lib.FLAG_FORCE_TC); k1 = _lib.last_kernel()
            dx = bsmm.bprop(Ed, Wd, flags=_lib.FLAG_FORCE_TC); k2 = _lib.last_kernel()
            assert _lib.device_error() == 0, _lib.device_error_text()
        assert k1 == k2 == ("wgmma_xprop_bs32_pair" if pair else "wgmma_xprop_bs32"), (k1, k2)
        res[pair] = (y, dx)
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_bs8_runs_padded_on_tcgen05(dtype, axis, monkeypatch):
    """8 x 8 blocks: 2 x 2 neighbourhoods padded into 16 x 16 super-blocks (csrc/wutil.cuh pad/unpad) and run by the wgmma
    kernels; fprop / bprop (plain, gated, positive operands) and updat (alpha, accumulate, gate) elementwise against the
    oracle, and against the CUDA-core path."""
    rng = np.random.default_rng(8 + axis)
    lay = layout(rng, 20, 14, 0.3, empty_col=3, empty_row=5)
    lay[:, 2] = 0                  # an empty super-block column (8 x 8 columns 2-3) and row (rows 4-5) too
    lay[4, :] = 0
    bsmm = BlocksparseMatMul(lay, block_size=8, feature_axis=axis)
    assert bsmm._shadow is not None and bsmm._shadow.bsize == 16
    orc = MatmulOracle(lay, 8, 0)
    orc.axis = axis
    N = 136
    W = torch.as_tensor(rng.normal(0, 0.2, bsmm.w_shape).astype(np.float32)).to(dtype)
    X = torch.as_tensor(rng.normal(0, 1, bsmm.i_shape(N)).astype(np.float32)).to(dtype)
    E = torch.as_tensor(rng.normal(0, 1, bsmm.o_shape(N)).astype(np.float32)).to(dtype)
    gate = ((rng.random(bsmm.blocks) < 0.7) * rng.uniform(0.5, 1.5, bsmm.blocks)).astype(np.float32)
    g = torch.as_tensor(gate).cuda()
    Wg = (W.float() * torch.as_tensor(gate)[:, None, None]).to(dtype)      # what bsmm_pad_blocks feeds the kernel
    P = lambda shape: torch.as_tensor(rng.uniform(0, 1, shape).astype(np.float32)).to(dtype)
    Wp, Xp, Ep = P(bsmm.w_shape), P(bsmm.i_shape(N)), P(bsmm.o_shape(N))
    name = dtype_name(dtype)
    for what, bprop, inp, w, gt, w_ref in [("fprop", False, X, W, None, W), ("bprop", True, E, W, None, W),
                                           ("fprop gated", False, X, W, g, Wg), ("bprop gated", True, E, W, g, Wg),
                                           ("fprop positive", False, Xp, Wp, None, Wp), ("bprop positive", True, Ep, Wp, None, Wp)]:
        xd, wd = inp.cuda(), w.cuda()
        fn = bsmm.bprop if bprop else bsmm.fprop
        _, kern = check_xprop(orc, lay, 8, bprop, inp, w_ref, lambda: fn(xd, wd, gate=gt), what,
                              k=feature_terms(bsmm._shadow.layout, 16, bprop, axis))
        assert kern == "wgmma_xprop_bs16", kern
    Xd, Ed = X.cuda(), E.cuda()
    Xn, En = X.float().numpy(), E.float().numpy()
    ref_dw, abs_dw = oracle_dense(orc, "updat", Xn, En), oracle_dense(orc, "updat", np.abs(Xn), np.abs(En))

    seen = []
    record_kernels(monkeypatch, bsmm._shadow, ("updat",), seen)      # the padded product behind each updat

    def check_dw(got, r, a, extra, what):
        assert _lib.device_error() == 0 and _lib.last_kernel() == "unpad_blocks", _lib.last_kernel()
        assert seen.pop() == ("updat", "wgmma_updat_bs16") and not seen
        assert not bool(torch.isnan(got).any()), "%s: dw elements never written" % what
        out = dtype_name(got.dtype)
        assert_within(got, r, mma_gemm_bound(r, a, out, N, extra), what, a, N, out, "wgmma_updat")
        mx, l2 = ref_errors(got.double().cpu().numpy(), r)
        assert l2 <= {"float32": 1e-5, "bfloat16": 4e-3, "float16": 1e-3}[out], "%s l2 %.3e" % (what, l2)

    dw = _on_poisoned_output(lambda: bsmm.updat([Xd], [Ed], dw_dtype=torch.float32))
    check_dw(dw, ref_dw, abs_dw, 0, "updat")
    old = dw.double().cpu().numpy()
    bsmm.updat([Xd], [Ed], dw=dw, alpha=0.5)                           # in-place accumulate
    check_dw(dw, old + 0.5 * ref_dw, np.abs(old) + 0.5 * abs_dw, 2, "accumulate")
    dwg = _on_poisoned_output(lambda: bsmm.updat([Xd], [Ed], gate=g, dw_gated=True))
    gn = gate.astype(np.float64)[:, None, None]
    check_dw(dwg, ref_dw * gn, abs_dw * gn, 1, "gated %s dw" % name)
    Wd = W.cuda()
    fma = bsmm.fprop(Xd, Wd, flags=_lib.FLAG_FORCE_GENERIC)
    assert _lib.last_kernel().startswith("fma_")
    assert (fma.float() - bsmm.fprop(Xd, Wd).float()).abs().max().item() <= 2.0 ** -7 * fma.float().abs().max().item()
    assert _lib.device_error() == 0
