"""fp8 weight gradients on the GPU: quantize_fp8_t, updat_fp8 and matmul_fp8(fp8_dw=True).

quantize_fp8_t is checked bit for bit against quantize_fp8. updat_fp8 is checked elementwise against the float64 product
of the dequantised operands x^ = q_x * scale_inv_x, dy^ = q_dy * scale_inv_dy:

    |dw - dw64| <= (EPS_STAGE + (chunks + 3) 2^-24) * S + u_out |dw64|,   S = sum |x^||dy^|

chunks is the number of 128-row stages summed over all pairs. EPS_STAGE bounds the tensor cores' error on one stage's
fp8 partial: DESIGN.md 6e measured 2^-13 per chained k32 step for the xprop kernel, and a stage chains four, so
EPS_STAGE = 4 * 2^-13. Each stage's fragment is added to the fp32 total with one fma (one rounding per stage), the
scale_p = x_scale_inv * dy_scale_inv product is one more rounding, and the accumulation into dw (beta = 1) and the final
conversion are in the last two terms (dw64 includes the old dw then). Every case prints its estimate of EPS_STAGE,
max((|d| - bound without EPS_STAGE) / S), with -s.
"""
import gc

import numpy as np
import pytest
import torch

from tests._util import U_OUT, dtype_name
from blocksparse_b200 import BlocksparseMatMul, _lib, group_param_grads, quantize_fp8
from blocksparse_b200.fp8 import quantize_fp8_t, quantize_fp8_weights, updat_fp8, xprop_fp8
from blocksparse_b200.layouts import barabasi_albert_layout, bernoulli_layout

pytestmark = pytest.mark.gpu

E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2
EPS_STAGE = 4 * 2.0 ** -13
EPS32 = 2.0 ** -24
GB = 2.0 ** 30
SRC = [torch.float32, torch.float16, torch.bfloat16]


def u8(t):
    return t.view(torch.uint8)


def bits_equal(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ---- quantize_fp8_t ------------------------------------------------------------------------------------------------
def check_quantize_t(x, fp8):
    q0, s0 = quantize_fp8(x, fp8)
    q, q_t, s = quantize_fp8_t(x, fp8)
    rows, cols = x.shape
    pitch = (rows + 15) // 16 * 16
    assert q.shape == (rows, cols) and q_t.shape == (cols, pitch) and q.dtype == q_t.dtype == fp8
    assert bits_equal(q, q0)
    assert bits_equal(s, s0) or (torch.isnan(s).all() and torch.isnan(s0).all())
    assert torch.equal(u8(q_t)[:, :rows], u8(q0).t())
    assert (u8(q_t)[:, rows:] == 0).all()
    none, q_t2, s2 = quantize_fp8_t(x, fp8, with_rows=False)
    assert none is None and bits_equal(q_t2, q_t)
    return s


@pytest.mark.parametrize("fp8", [E4, E5])
@pytest.mark.parametrize("dtype", SRC)
@pytest.mark.parametrize("rows", [1, 15, 16, 4099, 65544])
def test_quantize_t_matches_quantize(fp8, dtype, rows):
    rng = np.random.default_rng(rows)
    for cols in (33, 7):
        x = rng.normal(0, 3, (rows, cols)).astype(np.float32)
        x[rng.random(x.shape) < 0.01] *= 1e-6                  # subnormal fp8 results
        x.flat[rng.integers(0, x.size)] = -40.0
        check_quantize_t(torch.as_tensor(x).to(dtype).cuda(), fp8)


@pytest.mark.parametrize("fp8", [E4, E5])
@pytest.mark.parametrize("case", ["zeros", "nan", "inf", "-inf", "empty"])
def test_quantize_t_special_tensors(fp8, case):
    x = np.random.default_rng(1).normal(0, 1, 3000).astype(np.float32)
    if case == "zeros":
        x[:] = 0.0
        x[::7] = -0.0
    elif case == "nan":
        x[17] = np.nan
    elif case == "inf":
        x[5] = np.inf
    elif case == "-inf":
        x[2999] = -np.inf
    x = x.reshape(1000, 3)
    if case == "empty":
        x = x[:0]
    s = check_quantize_t(torch.as_tensor(x).bfloat16().cuda(), fp8)
    if case in ("nan", "inf", "-inf"):
        assert torch.isnan(s).all()
    if case in ("zeros", "empty"):
        assert s.item() == 1.0


# ---- updat_fp8 -----------------------------------------------------------------------------------------------------
def make_layout(kind, rng):
    if kind == "dense":
        return np.ones((8, 6), np.int32)
    if kind == "random25":
        return bernoulli_layout(rng, 8, 6, 0.25)
    if kind == "ba":
        return barabasi_albert_layout(8, 0.25, rng)
    if kind == "wide":                                          # more kept output blocks per group than one tile holds
        lay = bernoulli_layout(rng, 4, 20, 0.7)
        lay[0, :] = 1
        return lay
    lay = bernoulli_layout(rng, 8, 6, 0.5)                       # "empty": input block row 2 and output block column 4
    lay[2, :] = 0
    lay[:, 4] = 0
    return lay


def blocks_of(bsmm, D):
    bs = bsmm.bsize
    cs = torch.as_tensor([c for c, _ in bsmm.updat_list], device=D.device)
    ks = torch.as_tensor([k for _, k in bsmm.updat_list], device=D.device)
    return D.view(bsmm.CB, bs, bsmm.KB, bs).permute(0, 2, 1, 3)[cs, ks]


def reference(bsmm, xts, dyts, xsis, dsis, N):
    """(dw64, S) per block in float64 from the dequantised feature-major operands."""
    D = torch.zeros((bsmm.C, bsmm.K), dtype=torch.float64, device="cuda")
    S = torch.zeros_like(D)
    for xt, dyt, a, b in zip(xts, dyts, xsis, dsis):
        xh = xt[:, :N].float().double() * float(a.item())
        dh = dyt[:, :N].float().double() * float(b.item())
        D += xh @ dh.t()
        S += xh.abs() @ dh.abs().t()
    return blocks_of(bsmm, D), blocks_of(bsmm, S)


def check_within(dw, ref, S, chunks, what):
    """Asserts the bound; prints and returns the estimate max((|d| - bound without EPS_STAGE) / S)."""
    u = U_OUT[dtype_name(dw.dtype)]
    err = (dw.double() - ref).abs()
    rest = (chunks + 3) * EPS32 * S + u * ref.abs() + (2.0 ** -25 if dw.dtype == torch.float16 else 0.0)
    b = EPS_STAGE * S + rest
    if (err > b).any():
        i = int((err - b).argmax())
        raise AssertionError("%s: %d elements past the bound, worst |d| %.3e > %.3e" % (
            what, int((err > b).sum()), float(err.flatten()[i]), float(b.flatten()[i])))
    live = S > 0
    est = float(((err - rest)[live] / S[live]).max()) if live.any() else 0.0
    print("fp8-updat-eps-estimate %s: %.3e (2^%.2f)" % (what, est, np.log2(est) if est > 0 else -np.inf))
    if not live.any():
        assert (dw.double() == ref).all()
    return est


def fp8_pairs(bsmm, N, pcount, xf, df, rng):
    xts, dyts, xsis, dsis = [], [], [], []
    for p in range(pcount):
        x = torch.as_tensor(rng.normal(0, 1 + p, (N, bsmm.C)).astype(np.float32)).bfloat16().cuda()
        dy = torch.as_tensor(rng.normal(0, 0.01 * (p + 1), (N, bsmm.K)).astype(np.float32)).bfloat16().cuda()
        _, xt, xs = quantize_fp8_t(x, xf, with_rows=False)
        _, dyt, ds = quantize_fp8_t(dy, df, with_rows=False)
        xts.append(xt); dyts.append(dyt); xsis.append(xs); dsis.append(ds)
    return xts, dyts, xsis, dsis


CASES = [(1, torch.float32, (E4, E5), False), (3, torch.bfloat16, (E4, E4), True), (8, torch.float16, (E5, E5), False),
         (3, torch.float32, (E5, E4), True)]


@pytest.mark.parametrize("bs", [32, 64])
@pytest.mark.parametrize("kind", ["dense", "random25", "ba", "empty", "wide"])
@pytest.mark.parametrize("N", [1, 127, 128, 4099])
def test_updat_fp8_elementwise(bs, kind, N):
    rng = np.random.default_rng(N * 7 + bs)
    bsmm = BlocksparseMatMul(make_layout(kind, rng), block_size=bs, feature_axis=1)
    for pcount, out, (xf, df), beta in CASES:
        ops = fp8_pairs(bsmm, N, pcount, xf, df, rng)
        ref, S = reference(bsmm, *ops, N)
        if beta:
            old = torch.as_tensor(rng.normal(0, 1, bsmm.w_shape).astype(np.float32)).to(out).cuda()
            dw = updat_fp8(bsmm, *ops, N, dw=old.clone())
            ref = ref + old.double()
        else:
            dw = updat_fp8(bsmm, *ops, N, dw_dtype=out)
        assert _lib.last_kernel() == "wgmma_updat_fp8_bs%d" % bs and dw.dtype == out
        chunks = pcount * ((N + 127) // 128)
        check_within(dw, ref, S, chunks, "%s bs %d N %d pairs %d %s %s x %s beta %d" % (
            kind, bs, N, pcount, dtype_name(out), xf, df, beta))


@pytest.mark.parametrize("bs", [32, 64])
def test_updat_fp8_error_estimate(bs):
    """Dense 1024 x 256, N = 8192, fp32 dw: the output rounding is negligible, so the printed estimate is the tensor
    cores' error per stage."""
    rng = np.random.default_rng(bs)
    bsmm = BlocksparseMatMul(np.ones((1024 // bs, 256 // bs), np.int32), block_size=bs, feature_axis=1)
    N = 8192
    for xf, df in ((E4, E5), (E4, E4), (E5, E5)):
        ops = fp8_pairs(bsmm, N, 1, xf, df, rng)
        ref, S = reference(bsmm, *ops, N)
        check_within(updat_fp8(bsmm, *ops, N, dw_dtype=torch.float32), ref, S, N // 128,
                     "dense 1024 x 256 bs %d %s x %s" % (bs, xf, df))


def test_updat_fp8_without_rows():
    """N = 0 as bsmm_updat: an empty sum, so dw = 0, or dw unchanged when accumulating."""
    bsmm = BlocksparseMatMul(bernoulli_layout(np.random.default_rng(0), 8, 6, 0.4), block_size=32, feature_axis=1)
    xt = torch.zeros((bsmm.C, 16), dtype=E4, device="cuda")
    dyt = torch.zeros((bsmm.K, 16), dtype=E5, device="cuda")
    s = torch.ones(1, device="cuda")
    dw = updat_fp8(bsmm, xt, dyt, s, s, 0, dw_dtype=torch.float32)
    assert (dw == 0).all()
    old = torch.randn(bsmm.w_shape, device="cuda")
    assert torch.equal(updat_fp8(bsmm, xt, dyt, s, s, 0, dw=old.clone()), old)


# ---- matmul_fp8(fp8_dw=True) ---------------------------------------------------------------------------------------
def tensors(bsmm, shape, dtype, rng):
    I = torch.as_tensor(rng.normal(0, 1, shape + (bsmm.C,)).astype(np.float32)).to(dtype).cuda()
    W = torch.as_tensor(rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)).to(dtype).cuda()
    dy = torch.as_tensor(rng.normal(0, 1, shape + (bsmm.K,)).astype(np.float32)).to(dtype).cuda()
    return I, W, dy


def run(bsmm, I, W, dy, fp8_dw):
    I, W = I.clone().requires_grad_(), W.clone().requires_grad_()
    y = bsmm.matmul_fp8(I, W, fp8_dw=fp8_dw)
    y.backward(dy)
    return y, I.grad, W.grad


@pytest.mark.parametrize("bs", [32, 64])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_matmul_fp8_dw(bs, dtype):
    rng = np.random.default_rng(bs + 5)
    bsmm = BlocksparseMatMul(bernoulli_layout(rng, 8, 6, 0.3), block_size=bs, feature_axis=1)
    I, W, dy = tensors(bsmm, (3, 700), dtype, rng)
    y0, dx0, dw0 = run(bsmm, I, W, dy, False)
    y1, dx1, dw1 = run(bsmm, I, W, dy, True)
    assert bits_equal(y1, y0) and bits_equal(dx1, dx0)
    assert dw1.dtype == dtype and dw1.shape == bsmm.w_shape
    N = 3 * 700
    _, xt, xs = quantize_fp8_t(I.reshape(N, -1), E4, with_rows=False)
    _, dyt, ds = quantize_fp8_t(dy.reshape(N, -1), E5, with_rows=False)
    ref, S = reference(bsmm, [xt], [dyt], [xs], [ds], N)
    check_within(dw1, ref, S, (N + 127) // 128, "matmul_fp8 dw bs %d %s" % (bs, dtype_name(dtype)))


def test_matmul_fp8_dw_keeps_no_16bit_copy_of_i():
    rng = np.random.default_rng(3)
    bsmm = BlocksparseMatMul(bernoulli_layout(rng, 8, 6, 0.3), block_size=32, feature_axis=1)
    I, W, _ = tensors(bsmm, (1000,), torch.bfloat16, rng)
    y = bsmm.matmul_fp8(I.requires_grad_(), W.requires_grad_(), fp8_dw=True)
    saved = y.grad_fn.saved_tensors
    assert not any(t.dtype in (torch.float16, torch.bfloat16, torch.float32) and t.numel() >= I.numel() for t in saved)
    assert any(t.dtype == E4 and t.shape == (bsmm.C, 1008) for t in saved)
    y_ref = bsmm.matmul_fp8(I, W)
    assert any(t.dtype == torch.bfloat16 and t.numel() == I.numel() for t in y_ref.grad_fn.saved_tensors)


def test_group_param_grads_fp8():
    """10 uses in one block: two updat_fp8 launches (8 + 2 pairs) accumulating into one dw, bit for bit the explicit
    composition of the two launches."""
    rng = np.random.default_rng(4)
    bsmm = BlocksparseMatMul(bernoulli_layout(rng, 8, 6, 0.3), block_size=32, feature_axis=1)
    _, W, _ = tensors(bsmm, (1,), torch.bfloat16, rng)
    Is, dys = zip(*[tensors(bsmm, (300,), torch.bfloat16, rng)[::2] for _ in range(10)])
    W = W.requires_grad_()
    with group_param_grads(bsmm, W) as pending:
        for I, dy in zip(Is, dys):
            bsmm.matmul_fp8(I, W, fp8_dw=True).backward(dy)
    assert pending.fp8_launches == 2 and pending.launches == 2
    ops = [(quantize_fp8_t(I, E4, with_rows=False), quantize_fp8_t(dy, E5, with_rows=False)) for I, dy in zip(Is, dys)]
    xts, xss = [o[0][1] for o in ops], [o[0][2] for o in ops]
    dyts, dss = [o[1][1] for o in ops], [o[1][2] for o in ops]
    ref = updat_fp8(bsmm, xts[:8], dyts[:8], xss[:8], dss[:8], 300, dw_dtype=torch.bfloat16)
    ref = updat_fp8(bsmm, xts[8:], dyts[8:], xss[8:], dss[8:], 300, dw=ref)
    assert bits_equal(W.grad, ref)
    d64, S = reference(bsmm, xts, dyts, xss, dss, 300)
    err = (W.grad.double() - d64).abs()
    assert (err <= (EPS_STAGE + 13 * EPS32) * S + 2 * U_OUT["bfloat16"] * (S + d64.abs())).all()


def test_group_param_grads_mixed():
    """One bsmm() use and one fp8 use of the same weight: dw is the sum of both (fp8 pairs first, then 16-bit)."""
    rng = np.random.default_rng(5)
    bsmm = BlocksparseMatMul(bernoulli_layout(rng, 8, 6, 0.3), block_size=32, feature_axis=1)
    I1, W, dy1 = tensors(bsmm, (500,), torch.bfloat16, rng)
    I2, _, dy2 = tensors(bsmm, (400,), torch.bfloat16, rng)
    W = W.requires_grad_()
    with group_param_grads(bsmm, W) as pending:
        bsmm(I1, W).backward(dy1)
        bsmm.matmul_fp8(I2, W, fp8_dw=True).backward(dy2)
    assert pending.fp8_launches == 1 and pending.launches == 2
    _, xt, xs = quantize_fp8_t(I2, E4, with_rows=False)
    _, dyt, ds = quantize_fp8_t(dy2, E5, with_rows=False)
    ref = bsmm.updat([I1], [dy1], dw=updat_fp8(bsmm, xt, dyt, xs, ds, 400, dw_dtype=torch.bfloat16))
    assert bits_equal(W.grad, ref)


# ---- determinism and execution context ----------------------------------------------------------------------------
def ctx_case(seed):
    rng = np.random.default_rng(seed)
    bsmm = BlocksparseMatMul(bernoulli_layout(rng, 16, 12, 0.25), block_size=32, feature_axis=1)
    N = 4099
    x = torch.as_tensor(rng.normal(0, 1, (3, N, bsmm.C)).astype(np.float32)).bfloat16().cuda()
    dy = torch.as_tensor(rng.normal(0, 1, (3, N, bsmm.K)).astype(np.float32)).bfloat16().cuda()
    return bsmm, x, dy, N


def fp8_dw_pass(bsmm, x, dy, N):
    """quantize_fp8_t of three (x, dy) pairs and one three-pair updat_fp8 (capturable: no host sync)."""
    ops = [(quantize_fp8_t(x[p], E4, with_rows=False), quantize_fp8_t(dy[p], E5, with_rows=False)) for p in range(3)]
    return updat_fp8(bsmm, [o[0][1] for o in ops], [o[1][1] for o in ops], [o[0][2] for o in ops],
                     [o[1][2] for o in ops], N, dw_dtype=torch.float32)


def test_determinism():
    bsmm, x, dy, N = ctx_case(0)
    assert bits_equal(fp8_dw_pass(bsmm, x, dy, N), fp8_dw_pass(bsmm, x, dy, N))


def test_side_stream():
    bsmm, x, dy, N = ctx_case(1)
    ref = fp8_dw_pass(bsmm, x, dy, N)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 20)
        got = fp8_dw_pass(bsmm, x, dy, N)
    torch.cuda.current_stream().wait_stream(s)
    assert bits_equal(got, ref)


def test_graph_replay():
    bsmm, x, dy, N = ctx_case(2)
    _, x2, dy2, _ = ctx_case(3)
    fp8_dw_pass(bsmm, x, dy, N)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fp8_dw_pass(bsmm, x, dy, N)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fp8_dw_pass(bsmm, x, dy, N)
    x.copy_(x2)
    dy.copy_(dy2)
    graph.replay()
    torch.cuda.synchronize()
    assert bits_equal(out, fp8_dw_pass(bsmm, x2, dy2, N))


# ---- large offsets -----------------------------------------------------------------------------------------------
def test_large_offsets():
    """x (N = 2^19 + 128 rows, C = 4096): q_t's byte offsets pass 2^31 in its last feature rows. Sampled blocks,
    the last input block among them, against float64."""
    N, C = (1 << 19) + 128, 4096
    need = N * C * 3 + (1 << 30)                                 # bf16 x + fp8 q_t + slack
    gc.collect()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip("the large-offset fp8 updat case needs %.1f GB of free device memory, %.1f GB are free" % (need / GB, free / GB))
    rng = np.random.default_rng(12)
    lay = bernoulli_layout(rng, C // 32, 4, 0.25)
    lay[-1, :] = 1
    bsmm = BlocksparseMatMul(lay, block_size=32, feature_axis=1)
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((N, C), generator=gen, device="cuda", dtype=torch.bfloat16)
    _, xt, xs = quantize_fp8_t(x, E4, with_rows=False)
    del x
    dy = torch.randn((N, bsmm.K), generator=gen, device="cuda", dtype=torch.bfloat16)
    _, dyt, ds = quantize_fp8_t(dy, E5, with_rows=False)
    dw = updat_fp8(bsmm, xt, dyt, xs, ds, N, dw_dtype=torch.float32)
    last = [b for b, (c, _) in enumerate(bsmm.updat_list) if c == bsmm.CB - 1]
    picks = sorted(set(last + [0] + [int(b) for b in rng.integers(0, bsmm.blocks, 6)]))
    for b in picks:
        c, k = bsmm.updat_list[b]
        xh = xt[c * 32:(c + 1) * 32, :N].float().double() * float(xs.item())
        dh = dyt[k * 32:(k + 1) * 32, :N].float().double() * float(ds.item())
        ref, S = xh @ dh.t(), xh.abs() @ dh.abs().t()
        check_within(dw[b], ref, S, (N + 127) // 128, "large offsets block %d (c %d, k %d)" % (b, c, k))
