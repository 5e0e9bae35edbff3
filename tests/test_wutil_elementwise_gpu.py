"""Elementwise GPU checks of the weight utilities (csrc/wutil.cuh) against float64 evaluations of oracle/wutil_oracle.py
on the inputs as rounded to their storage dtype:

* l2_normalize and its gradient through the autograd op: 16-bit and fp32 outputs, with and without a gain, an empty
  output block column, a column of 24 blocks, and output features whose sum of squares is zero or below epsilon;
* block norm, threshold and top-k pruning and l2_decay: a tie at the threshold, tied blocks at the top-k keep boundary,
  sparsity 0 and 1, decays that clamp to 1, gated-out blocks;
* identity_init at every block size and dtype, bit for bit;
* the block-reduced full dW at all eight (axis, block size) pairs and both norms, including a zero scale;
* SparseProj gather / scatter / scatter_add / scatter_mul and their gradients, bit for bit, up to 70001 rows.

Each error bound is derived in the docstring of its test, in the terms of chain_bound. Outputs the library allocates are
checked on NaN-poisoned memory, so an element that no kernel writes fails the check."""
import numpy as np
import pytest
import torch

from tests._util import _on_poisoned_output, assert_within, chain_bound, dtype_name
from blocksparse_b200 import (BlocksparseMatMul, SparseProj, _lib, block_reduced_full_dw, blocksparse_l2_decay, blocksparse_norm,
                              blocksparse_prune, blocksparse_reduced_dw)
from oracle import wutil_oracle
from oracle.bsmm_oracle import MatmulOracle

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
DTYPES = [F32, F16, BF16]
BSIZES = [8, 16, 32, 64]
EPS = float(np.float32(1e-12))         # the default epsilon as the kernels receive it (a C float)


def f64(t):
    return t.detach().double().cpu().numpy()


def rounded(a, dtype):
    """float64 array a rounded once to dtype, as a CPU tensor."""
    return torch.as_tensor(np.asarray(a, dtype=np.float64)).to(dtype)


def check(got, ref, ref_abs, out_dtype, k_terms, what):
    """assert_within(chain_bound(...)); BSMM_BOUND_LOG records the share of the accumulation budget used."""
    name = dtype_name(out_dtype)
    assert_within(got, ref, chain_bound(ref, ref_abs, name, k_terms), what, ref_abs=ref_abs, k_terms=k_terms, out_dtype=name,
                  family="wutil " + what.split()[0])


# ---- l2_normalize ---------------------------------------------------------------------------------------------------
L2N_CASES = [(dt, out) for dt in DTYPES for out in ([F32] if dt == F32 else [dt, F32])]


def l2n_layout():
    rng = np.random.default_rng(5)
    lay = (rng.random((24, 5)) < 0.3).astype(np.int32)
    lay[:, 0] = 1                     # a column of 24 blocks
    lay[:, 2] = 0                     # an empty output block column
    lay[3, 1] = lay[7, 3] = lay[11, 4] = 1
    return lay


def l2n_grad_budgets(cols, Wn, Un, gain, bs, k_ss, chain):
    """Weighted absolute sums that bound dx and dg (k_terms = 1), per the derivation in test_l2_normalize_elementwise."""
    bx, bg = np.zeros_like(Wn), np.zeros((max(cols) + 1) * bs)
    for k, ws in cols.items():
        if not ws:
            continue
        x, d = Wn[ws].reshape(-1, bs), Un[ws].reshape(-1, bs)
        g = np.ones(bs) if gain is None else gain[k * bs:(k + 1) * bs]
        ss = (x * x).sum(0)
        mx = np.maximum(ss, EPS)
        norm, live = 1 / np.sqrt(mx), ss >= EPS
        A = np.abs(d * g * x).sum(0) / mx
        red = (-d * g * x).sum(0) / mx * live
        B = (np.abs(d * g) + np.abs(x * red)) * norm
        bx[ws] = ((7 + 0.5 * k_ss[k]) * B + (chain[k] + 4 + k_ss[k]) * norm * np.abs(x) * A * live).reshape(len(ws), bs, bs)
        bg[k * bs:(k + 1) * bs] = (chain[k] + 6 + 0.5 * k_ss[k]) * np.abs(d * x).sum(0) * norm
    return bx, bg


@pytest.mark.parametrize("with_gain", [False, True])
@pytest.mark.parametrize("bs", BSIZES)
@pytest.mark.parametrize("dtype,out_dtype", L2N_CASES, ids=lambda d: dtype_name(d))
def test_l2_normalize_elementwise(dtype, out_dtype, bs, with_gain):
    """y = g w / sqrt(max(ss, eps)) per output feature of a block column, its gradient and the kept sums of squares.

    One CTA per block column; thread (r, j) sums w^2 over its ceil(bs / R) rows of each of the column's n blocks
    (R = 128 / bs row groups), then R partials are added in order: chain = n ceil(bs / R) + R additions, and
    k_ss = chain + 1 with the product rounding, as the relative error of ss. rsqrtf adds 4 eps32 (2 ulp), the gain and
    the weight product one each, and y carries half of ss's error: k_y = k_ss / 2 + 6.
    The gradient: norm2_i = 1 / max(ss, eps) carries k_ss + 1, each term (-d g x) norm2_i three more roundings, so
    red = sum(-d g x) / mx is off by at most (chain + 4 + k_ss) eps32 A with A = sum |d g x| / mx. Then
    dx = (d g + x red) norm_i rounds d g, x red, their sum and the product once each and norm_i carries
    k_ss / 2 + 4: the budget is (7 + k_ss / 2) eps32 (|d g| + |x red|) norm + (chain + 4 + k_ss) eps32 norm |x| A, where
    red is zero (exactly, in the kernel too) for features with ss < eps. dg = sum d x norm_i: chain additions, the two
    products and norm_i, (chain + 6 + k_ss / 2) eps32 sum |d x| norm. Output features with ss = 0 or 0 < ss < eps take
    the eps floor; their dy is scaled by 2^-16 so that dy g / sqrt(eps) stays finite in fp16."""
    rng = np.random.default_rng(bs * 10 + with_gain + 3 * DTYPES.index(dtype))
    lay = l2n_layout()
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=0)
    flist = MatmulOracle(lay, 32, 1).fprop_list
    cols = {k: [w for _, w in col] for k, col in flist}
    Wf, Uf = rng.normal(0, 1, bsmm.w_shape), rng.normal(0, 1, bsmm.w_shape)
    c1 = cols[1]
    Wf[c1, :, 0] = Wf[c1, :, 1] = 0.0                     # feature 0 of column 1: all zero
    tiny = np.sqrt(0.4e-12 / bs)                           # feature 1: 0 < ss < eps, from one block (fp16 subnormals)
    Wf[c1[0], :, 1] = rng.uniform(0.5, 1, bs) * rng.choice([-1, 1], bs) * tiny
    Wf[cols[3]] = 0.0                                      # every feature of column 3: all zero
    for k, feats in ((1, [0, 1]), (3, list(range(bs)))):
        for j in feats:
            Uf[cols[k], :, j] *= 2.0 ** -16
    W, U = rounded(Wf, dtype), rounded(Uf, out_dtype)
    Wn, Un = f64(W), f64(U)
    ss_tiny = (Wn[c1, :, 1] ** 2).sum()
    assert 0.05 * EPS < ss_tiny < 0.6 * EPS, ss_tiny / EPS      # well clear of eps: the comparison is not ambiguous
    gain = rng.uniform(0.5, 2.0, bsmm.K).astype(np.float32) if with_gain else None
    g64 = None if gain is None else gain.astype(np.float64)

    R = 128 // bs
    chain = {k: len(ws) * -(-bs // R) + R for k, ws in cols.items()}
    k_ss = {k: c + 1 for k, c in chain.items()}
    k_blk = np.zeros(bsmm.blocks)
    for k, ws in cols.items():
        k_blk[ws] = k_ss[k]

    w = W.cuda().requires_grad_()
    G = None if gain is None else torch.as_tensor(gain).cuda().requires_grad_()
    y = _on_poisoned_output(lambda: bsmm.l2_normalize(w, gain=G, dtype=out_dtype))
    assert _lib.last_kernel() == "l2_normalize" and y.dtype == out_dtype
    ss = y.grad_fn.saved_tensors[2]
    yref, ss_all = wutil_oracle.l2_normalize(flist, Wn, bs, gain=g64, epsilon=EPS)
    ss_ref = np.zeros((bsmm.KB, bs))
    for k, v in ss_all.items():
        ss_ref[k] = v
    k_col = np.array([k_ss[k] for k in range(bsmm.KB)])[:, None]
    check(ss.view(bsmm.KB, bs), ss_ref, ss_ref, F32, k_col, "l2_normalize sum_sqr")
    assert f64(ss)[bs + 1] < EPS and f64(ss)[bs] == 0.0
    check(y, yref, np.abs(yref), out_dtype, (0.5 * k_blk + 6)[:, None, None], "l2_normalize y")

    def backward():
        return torch.autograd.grad(y, (w,) if G is None else (w, G), U.cuda())
    grads = _on_poisoned_output(backward)
    dx_ref, dg_ref = wutil_oracle.l2_normalize_grad(flist, Wn, Un, bs, gain=g64, epsilon=EPS)
    bx, bg = l2n_grad_budgets(cols, Wn, Un, g64, bs, k_ss, chain)
    check(grads[0], dx_ref, bx, dtype, 1, "l2_normalize dx")
    if G is not None:
        check(grads[1], dg_ref, bg, F32, 1, "l2_normalize dgain")


def test_l2_normalize_rejects_other_output_dtypes():
    """The output is the weight dtype or fp32; an fp32 weight with a 16-bit output, or a 16-bit weight with the other
    16-bit dtype, is refused rather than computed."""
    lay = np.ones((2, 3), dtype=np.int32)
    bsmm = BlocksparseMatMul(lay, block_size=16, feature_axis=0)
    for wd, yd in ((F32, F16), (F32, BF16), (F16, BF16), (BF16, F16)):
        with pytest.raises(ValueError, match="output dtype"):
            bsmm.l2_normalize(torch.ones(bsmm.w_shape, dtype=wd, device="cuda"), dtype=yd)


# ---- block norm / pruning / l2_decay --------------------------------------------------------------------------------
DUPS = [3, 20, 31]


def ranked_blocks(rng, blocks, bs, dtype):
    """Blocks that are sign-flipped permutations of one unit-norm pattern scaled by 1.05^level: max and l2 norm rank
    them alike, 5 % apart. DUPS are exact copies at the level with 18 blocks above, so a keep of 20 splits them."""
    base = rng.normal(0, 1, bs * bs)
    base /= np.linalg.norm(base)
    levels = np.empty(blocks)
    others = [b for b in range(blocks) if b not in DUPS]
    levels[others] = rng.permutation(list(range(18)) + list(range(19, blocks - 2)))
    levels[DUPS] = 18
    Wf = np.stack([rng.permutation(base) * rng.choice([-1, 1], bs * bs) * 1.05 ** levels[b] for b in range(blocks)]).reshape(blocks, bs, bs)
    W = rounded(Wf, dtype)
    W[DUPS[1:]] = W[DUPS[0]].clone()
    return W


@pytest.mark.parametrize("bs", BSIZES)
@pytest.mark.parametrize("dtype", DTYPES, ids=dtype_name)
def test_norm_prune_decay_elementwise(dtype, bs):
    """One warp per block, 4 blocks per CTA, 39 blocks. Lane l sums bs^2 / 32 squares serially, then 5 shuffle levels:
    k_s = bs^2 / 32 + 6 with the product rounding. The l2 norm sqrtf(s) carries k_s / 2 + 1; the max norm is exact.
    l2_decay: s + eps rounds once more, the decay d = min(rate rsqrtf(s + eps), 1) carries (k_s + 1) / 2 + 4 + 1, and
    w - w d rounds the product and the difference: the budget is |w| d ((k_s + 1) / 2 + 6) + |w - w d| (k_terms = 1),
    then the output rounding. Blocks whose decay clamps come out exactly 0, gated-out blocks bit-identical."""
    rng = np.random.default_rng(200 + bs + 7 * DTYPES.index(dtype))
    blocks, name = 39, dtype_name(dtype)
    Wt = ranked_blocks(rng, blocks, bs, dtype)
    Wn, W = f64(Wt), Wt.cuda()
    k_s = bs * bs // 32 + 6
    l2 = wutil_oracle.block_norm(Wn, "l2")
    distinct = np.sort(np.delete(l2, DUPS[1:]))
    assert (distinct[1:] / distinct[:-1] > 1.01).all()           # no near-ties the kernel's rounding could reorder

    for norm in ("max", "l2"):
        got = _on_poisoned_output(lambda: blocksparse_norm(W, norm=norm))
        assert _lib.last_kernel() == "block_norm"
        ref = wutil_oracle.block_norm(Wn, norm)
        if norm == "max":
            assert np.array_equal(f64(got), ref), "max norm is not exact"
        else:
            check(got, ref, ref, F32, 0.5 * k_s + 1, "block_norm l2")

        # a threshold equal to a block's norm keeps it: for max the oracle's tie, for l2 the kernel's own value
        for thr in (float(got[DUPS[0]]), float(np.sqrt(np.sort(ref)[10] * np.sort(ref)[11]))):
            gate = torch.full((blocks,), float("nan"), device="cuda")
            blocksparse_prune(W, gate, step=4, threshold=thr, norm=norm, frequency=2)
            assert _lib.last_kernel() == "threshold_prune"
            expect = wutil_oracle.threshold_prune(Wn, thr, norm)
            if norm == "l2" and thr == float(got[DUPS[0]]):
                expect[DUPS] = 1.0
            assert np.array_equal(gate.cpu().numpy(), expect), "threshold %s %.9g" % (norm, thr)
        assert ref[DUPS[0]] == float(got[DUPS[0]]) or norm == "l2"

        for sparsity in (0.0, 0.5, 1.0):
            gate = torch.full((blocks,), float("nan"), device="cuda")
            blocksparse_prune(W, gate, step=0, sparsity=sparsity, norm=norm)
            assert _lib.last_kernel() == "prune_topk"
            expect = wutil_oracle.prune_topk(ref, sparsity)
            assert np.array_equal(gate.cpu().numpy(), expect), "top-k %s sparsity %g" % (norm, sparsity)
            if sparsity == 0.5:
                assert list(expect[DUPS]) == [1, 1, 0]            # the stable order splits the tied blocks

    srt = np.sort(l2)
    rate = float(np.float32(np.sqrt(srt[13] * srt[14])))        # 14 blocks clamp, the rest decay by < 1 / 1.02
    assert (np.abs(rate / l2 - 1) > 1e-2).all()
    gate = (rng.random(blocks) < 0.7).astype(np.float32)
    gate[np.argsort(l2)[[0, 20]]] = 0.0
    gate[np.argsort(l2)[[1, 2, 25, 26]]] = 1.0
    off, clamp = gate == 0, (gate != 0) & (l2 < rate)
    live = (gate != 0) & ~clamp
    Wd = W.clone()
    blocksparse_l2_decay(Wd, gate=torch.as_tensor(gate).cuda(), rate=rate, epsilon=1e-12)
    assert _lib.last_kernel() == "l2_decay"
    ref = wutil_oracle.l2_decay(Wn, gate, rate, epsilon=EPS)
    off_t, clamp_t = torch.as_tensor(off).cuda(), torch.as_tensor(clamp).cuda()
    assert torch.equal(Wd[off_t], W[off_t]), "gated-out blocks changed"
    assert bool((Wd[clamp_t] == 0).all()), "clamped blocks are not exactly zero"
    d = (rate / np.sqrt((Wn * Wn).sum(axis=(1, 2)) + EPS))[:, None, None]
    budget = np.abs(Wn) * d * (0.5 * (k_s + 1) + 6) + np.abs(ref)
    check(Wd[torch.as_tensor(live).cuda()], ref[live], budget[live], dtype, 1, "l2_decay")


# ---- identity_init --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bs", BSIZES)
@pytest.mark.parametrize("dtype", DTYPES, ids=dtype_name)
def test_identity_init_bit_exact(dtype, bs):
    """scale I on the blocks with (c % KB) == (k % CB), zero elsewhere, on poisoned memory, bit for bit with the
    oracle's fp32 result rounded to dtype. 0.3 is not a 16-bit value; the rectangular dense layouts put the wrapped
    diagonal on blocks with c != k."""
    rng = np.random.default_rng(bs)
    for shape, density in (((5, 5), 0.5), ((4, 7), 1.0), ((9, 3), 1.0), ((6, 10), 0.5)):
        lay = (rng.random(shape) < density).astype(np.int32)
        for i in range(max(shape)):
            lay[i % shape[0], i % shape[1]] = 1
        bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=0)
        W = _on_poisoned_output(lambda: bsmm.identity_init(scale=0.3, dtype=dtype))
        assert _lib.last_kernel() == "identity_init"
        orc = MatmulOracle(lay, 32, 0)
        ref = rounded(wutil_oracle.identity_init(orc.updat_list, orc.CB, orc.KB, bs, 0.3), dtype)
        assert torch.equal(W.cpu(), ref), "%s: %d elements differ" % (shape, int((W.cpu() != ref).sum()))
        if shape[0] != shape[1]:
            assert any(c != k and c % orc.KB == k % orc.CB for c, k in orc.updat_list)


# ---- block-reduced full dW ------------------------------------------------------------------------------------------
def contract(X, Y, axis):
    """sum over pairs and minibatch of X_RED x Y_RED in the oracle's layouts: (bC, bK)."""
    return X.reshape(X.shape[0], -1) @ Y.reshape(Y.shape[0], -1).T if axis == 0 else X.reshape(-1, X.shape[-1]).T @ Y.reshape(-1, Y.shape[-1])


@pytest.mark.parametrize("norm", ["max", "l2"])
@pytest.mark.parametrize("axis,bs", [(a, b) for a in (0, 1) for b in BSIZES])
@pytest.mark.parametrize("dtype", [F16, BF16], ids=dtype_name)
def test_reduced_dw_elementwise(dtype, axis, bs, norm):
    """x_red / y_red: max|.| is exact; the l2 norm sums bs exact 16-bit squares serially and takes sqrtf, so it carries
    bs / 2 + 1, then rounds to the activation dtype. dw: each of 8 row splits of the P N rows is one serial fp32 chain
    of ceil(P N / 8) terms, then 8 partials, the scale and the accumulation: k = ceil(P N / 8) + 10, relative to the
    product of the reduced values the kernel stored (all >= 0). The oracle multiplies X_RED / Y_RED rounded to the
    activation dtype; where the kernel's l2 value rounded to the neighbouring 16-bit number (it is checked above), the
    bound adds exactly that difference's share of the product.

    Cases: 1 pair with N = 5 (most splits empty); 8 pairs with N = 100; 3 more accumulated into that dw, and the same
    11 pairs grouped 8 + 3 through block_reduced_full_dw. bC = 19 and bK = 21 are not multiples of the 16 x 16 tile."""
    rng = np.random.default_rng(bs + 10 * axis + (norm == "l2") + 100 * (dtype == BF16))
    name, bx, by = dtype_name(dtype), 19, 21

    def acts(n_blk, N, count):
        shape = (n_blk * bs, N) if axis == 0 else (N, n_blk * bs)
        return [rounded(rng.normal(0, 1, shape), dtype) for _ in range(count)]

    def check_red(got, ref, what):
        if norm == "max":
            assert np.array_equal(f64(got), ref), what + ": max-reduced values are not exact"
        else:
            check(got, ref, ref, dtype, 0.5 * bs + 1, "reduced_dw " + what)

    def run(xs, ys, scale, dwi=None, what=""):
        XS, YS = [f64(t) for t in xs], [f64(t) for t in ys]
        xd, yd = [t.cuda() for t in xs], [t.cuda() for t in ys]
        out = {}

        def call():
            out["dw"], xr, yr = blocksparse_reduced_dw(xd, yd, scale, dwi=dwi, bsize=bs, norm=norm, axis=axis)
            return (xr, yr) if dwi is not None else (out["dw"], xr, yr)
        res = _on_poisoned_output(call)
        assert _lib.last_kernel() == "reduced_dw"
        xr, yr = res[-2:]
        _, XR, YR = wutil_oracle.reduced_dw(XS, YS, scale, bs, axis, norm)
        check_red(xr, XR, what + " x_red")
        check_red(yr, YR, what + " y_red")
        return out["dw"], f64(xr), f64(yr)

    def check_dw(dw, ref, xg, yg, xo, yo, dwa, scale, k, what):
        """ref from the rounded oracle values xo / yo; xg / yg: what the kernel stored. First the product of the stored
        values (the GEMM alone, logged), then the oracle with the stored values' differences from it added."""
        ref_abs = scale * contract(xg, yg, axis) + np.abs(dwa)
        check(dw, ref_abs, ref_abs, F32, k, "reduced_dw " + what)
        dx, dy = np.abs(xg - xo), np.abs(yg - yo)
        shift = scale * (contract(dx, yo, axis) + contract(xo, dy, axis) + contract(dx, dy, axis))
        assert_within(dw, ref, chain_bound(ref, ref_abs, "float32", k) + shift, "reduced_dw " + what + " vs oracle")

    rnd = lambda a: f64(rounded(a, dtype))

    xs, ys = acts(bx, 5, 1), acts(by, 5, 1)
    dw, xg, yg = run(xs, ys, 0.25, what="1 pair N=5")
    DW, XO, YO = wutil_oracle.reduced_dw([f64(t) for t in xs], [f64(t) for t in ys], 0.25, bs, axis, norm, round_red=rnd)
    check_dw(dw, DW, xg, yg, XO, YO, 0, 0.25, 1 + 10, "1 pair N=5 dw")

    N = 100
    xs, ys = acts(bx, N, 11), acts(by, N, 11)
    scale = float(np.float32(1.0 / (N * 11)))              # the value the kernel multiplies by
    XS, YS = [f64(t) for t in xs], [f64(t) for t in ys]
    dw8, xg8, yg8 = run(xs[:8], ys[:8], scale, what="8 pairs")
    DW8, XO8, YO8 = wutil_oracle.reduced_dw(XS[:8], YS[:8], scale, bs, axis, norm, round_red=rnd)
    k8 = -(-8 * N // 8) + 10
    check_dw(dw8, DW8, xg8, yg8, XO8, YO8, 0, scale, k8, "8 pairs dw")
    dw_acc = dw8.clone()
    _, xg3, yg3 = run(xs[8:], ys[8:], scale, dwi=dw_acc, what="3 pairs accumulated")
    DW3, XO3, YO3 = wutil_oracle.reduced_dw(XS[8:], YS[8:], scale, bs, axis, norm, round_red=rnd)
    k3 = -(-3 * N // 8) + 10
    dw_total = DW8 + DW3
    stack = lambda a, b: np.concatenate([a, b], axis=1 if axis == 0 else 0)
    check_dw(dw_acc, dw_total, stack(xg8, xg3), stack(yg8, yg3), stack(XO8, XO3), stack(YO8, YO3), 0, scale, k8 + k3 + 1,
             "8 + 3 pairs accumulated dw")
    full = block_reduced_full_dw([(a.cuda(), b.cuda()) for a, b in zip(xs, ys)], scale=scale, norm=norm, group_size=8, bsize=bs, axis=axis)
    assert torch.equal(full, dw_acc), "block_reduced_full_dw differs from the same two calls made by hand"


@pytest.mark.parametrize("dtype", [F16, BF16], ids=dtype_name)
def test_reduced_dw_scale_zero(dtype):
    """A zero scale computes nothing: with dwi, dw keeps its values bit for bit; without, dw is exactly zero; x_red and
    y_red are zero-filled. Checked on NaN-poisoned memory, so uninitialised reductions cannot leak into dw."""
    rng = np.random.default_rng(41)
    for axis, bs in ((0, 16), (1, 32), (0, 64)):
        shape = lambda nb: (nb * bs, 24) if axis == 0 else (24, nb * bs)
        xs = [rounded(rng.normal(0, 1, shape(5)), dtype).cuda() for _ in range(3)]
        ys = [rounded(rng.normal(0, 1, shape(7)), dtype).cuda() for _ in range(3)]
        dwi = torch.as_tensor(rng.normal(0, 1, (5, 7)).astype(np.float32)).cuda()
        keep = dwi.clone()
        xr, yr = _on_poisoned_output(lambda: blocksparse_reduced_dw(xs, ys, 0.0, dwi=dwi, bsize=bs, axis=axis)[1:])
        assert torch.equal(dwi, keep), "axis %d bs %d: dw changed at scale 0 (%d NaN)" % (axis, bs, int(torch.isnan(dwi).sum()))
        assert bool((xr == 0).all()) and bool((yr == 0).all()), "x_red / y_red not zero-filled"
        dw, xr, yr = _on_poisoned_output(lambda: blocksparse_reduced_dw(xs, ys, 0.0, bsize=bs, axis=axis, norm="l2"))
        assert bool((dw == 0).all()), "axis %d bs %d: dw not zero at scale 0 (%d NaN)" % (axis, bs, int(torch.isnan(dw).sum()))
        assert bool((xr == 0).all()) and bool((yr == 0).all()), "x_red / y_red not zero-filled"


def test_reduced_dw_rejects_fp32():
    x = torch.ones(64, 8, device="cuda")
    with pytest.raises(ValueError, match="16-bit"):
        blocksparse_reduced_dw([x], [x], 1.0, bsize=32)


# ---- SparseProj -----------------------------------------------------------------------------------------------------
def sparse_proj(nhidden, lut, seed):
    if lut == "stride":
        return SparseProj(nhidden, proj_stride=3, block_size=8)
    state = np.random.get_state()                 # nproj= shuffles with NumPy's global generator
    np.random.seed(seed)
    try:
        return SparseProj(nhidden, nproj=min(nhidden, 40), block_size=8)
    finally:
        np.random.set_state(state)


def check_sparse_proj(sp, N, dtype, rng):
    """Forward ops and gradients bit for bit against torch indexing in the same dtype, on poisoned outputs."""
    def t(rows):
        return rounded(rng.normal(0, 1, (rows, N)), dtype).cuda()
    gl = torch.as_tensor(sp.gather_lut.astype(np.int64)).cuda()
    assert (sp.scatter_lut < 0).any()                  # unmapped rows: scatter must write their zeros
    x, y = t(sp.nhidden).requires_grad_(), t(sp.nproj).requires_grad_()
    xv, yv = x.detach(), y.detach()

    def same(got, ref, what):
        assert torch.equal(got, ref), "%s N=%d %s: %d elements differ" % (what, N, dtype, int((got != ref).sum()))

    g = _on_poisoned_output(lambda: sp.gather(x))
    same(g, xv[gl], "gather")
    s = _on_poisoned_output(lambda: sp.scatter(y))
    ref = torch.zeros_like(xv)
    ref[gl] = yv
    same(s, ref, "scatter")
    za = _on_poisoned_output(lambda: sp.scatter_add(x, y))
    ref = xv.clone()
    ref[gl] += yv
    same(za, ref, "scatter_add")
    zm = _on_poisoned_output(lambda: sp.scatter_mul(x, y))
    ref = xv.clone()
    ref[gl] *= yv
    same(zm, ref, "scatter_mul")

    dg, dh = t(sp.nproj), t(sp.nhidden)
    (dx,) = _on_poisoned_output(lambda: torch.autograd.grad(g, x, dg))
    ref = torch.zeros_like(xv)
    ref[gl] = dg
    same(dx, ref, "gather grad")
    (dy,) = _on_poisoned_output(lambda: torch.autograd.grad(s, y, dh))
    same(dy, dh[gl], "scatter grad")
    got = {}

    def add_grad():
        got["dx"], dy = torch.autograd.grad(za, (x, y), dh)
        return (dy,)
    (dy,) = _on_poisoned_output(add_grad)
    same(got["dx"], dh, "scatter_add grad x")
    same(dy, dh[gl], "scatter_add grad y")
    dx, dy = _on_poisoned_output(lambda: torch.autograd.grad(zm, (x, y), dh))
    ref = dh.clone()
    ref[gl] *= yv
    same(dx, ref, "scatter_mul grad x")
    same(dy, (dh * xv)[gl], "scatter_mul grad y")


@pytest.mark.parametrize("lut", ["nproj", "stride"])
@pytest.mark.parametrize("N", [1, 40, 40000])
@pytest.mark.parametrize("dtype", DTYPES, ids=dtype_name)
def test_sparse_proj_bit_exact(dtype, N, lut):
    """N = 40000 is more than the 64 x 256 columns one pass of the row kernel covers."""
    rng = np.random.default_rng(N)
    sp = sparse_proj(96, lut, 7)
    check_sparse_proj(sp, N, dtype, rng)


@pytest.mark.parametrize("dtype", DTYPES, ids=dtype_name)
def test_sparse_proj_many_rows(dtype):
    """70001 rows: more than the 65535 blocks a grid's y dimension can hold."""
    rng = np.random.default_rng(70001)
    for lut in ("nproj", "stride"):
        sp = sparse_proj(70001, lut, 11)
        assert sp.nhidden == 70001
        check_sparse_proj(sp, 3, dtype, rng)
