"""fp8 quantisation and fp8 block-sparse fprop / bprop on the GPU.

Quantisation is checked bit for bit against oracle/fp8_oracle.py. Products are checked elementwise against float64
products of the dequantised fp8 operands x^ = q_x * scale_inv_x, w^ = q_w * scale_inv_w:

    |y - y64| <= (EPS_TC + (entries + 2) 2^-24) * sum|x^||w^| + u_out |y64|

EPS_TC bounds the tensor cores' error on one LUT entry's fp8 partial. Hopper's fp8 MMA is reported to keep fewer
accumulator bits than fp32 and no documentation gives the figure. The working assumption was 2^-13 per entry; on an
H100 a 64 x 64 bprop entry (two chained k32 MMAs) showed 2^-12.9, so the bound takes 2^-13 per k32 MMA step:
EPS_TC = (bs / 32) 2^-13 (DESIGN.md 6e records the measurements; every case prints its estimate with -s). The kernel
adds each entry's fragment into an fp32 total (one rounding per entry) and scales it once by x_scale_inv *
w_scale_inv (two more roundings); u_out is the unit roundoff of the final conversion to fp16 / bf16.
"""
import gc

import numpy as np
import pytest
import torch

from tests._util import U_OUT, dtype_name
from blocksparse_b200 import BlocksparseMatMul, _lib, group_param_grads, quantize_fp8
from blocksparse_b200.fp8 import quantize_fp8_weights, xprop_fp8
from blocksparse_b200.layouts import barabasi_albert_layout, bernoulli_layout
from oracle import fp8_oracle as fo

pytestmark = pytest.mark.gpu

E4, E5 = torch.float8_e4m3fn, torch.float8_e5m2
FMT = {E4: "e4m3", E5: "e5m2"}
EPS_TC_STEP = 2.0 ** -13                                         # per k32 MMA step of one entry
EPS32 = 2.0 ** -24
GB = 2.0 ** 30


def codes(t):
    return t.view(torch.uint8).cpu().numpy()


def f32(t):
    return np.float32(t.item())


def same_f32(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


# ---- quantisation ----------------------------------------------------------------------------------------------------
def special_values(rng, n, dtype):
    x = rng.normal(0, 3, n).astype(np.float32)
    x[rng.integers(0, n, 16)] *= 1e-6                           # subnormal fp8 results
    x[rng.integers(0, n, 8)] = 0.0
    x[rng.integers(0, n, 8)] = -0.0
    x[n // 2] = -40.0                                            # the amax element: lands exactly on -max
    x[n // 3] = 39.97                                            # rounds to +max
    return torch.as_tensor(x).to(dtype)


@pytest.mark.parametrize("fp8", [E4, E5])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("n, offset", [(4099, 0), (65536 + 8, 0), (1001, 1), (1, 0)])
def test_quantize_matches_oracle(fp8, dtype, n, offset):
    """offset 1 starts x one element into its buffer, so the kernels take their scalar path."""
    x = special_values(np.random.default_rng(n), n + offset, dtype)[offset:]
    xd = x.cuda()
    q, si = quantize_fp8(xd, fp8)
    rq, am, rsi = fo.quantize(x.float().numpy(), FMT[fp8])
    assert q.dtype == fp8 and q.shape == x.shape
    assert np.array_equal(codes(q), rq)
    assert same_f32(f32(si), rsi)
    amax = torch.empty(2, dtype=torch.float32, device="cuda")
    qq = torch.empty_like(q)
    _lib.check(_lib.load().bsmm_fp8_quantize(_lib.dtype_code(dtype), _lib.fp8_code(fp8), xd.data_ptr(), n, amax.data_ptr(),
                                             amax.data_ptr() + 4, qq.data_ptr(), _lib.stream_ptr()), "bsmm_fp8_quantize")
    assert same_f32(f32(amax[0]), am) and torch.equal(qq.view(torch.uint8), q.view(torch.uint8))


@pytest.mark.parametrize("fp8", [E4, E5])
@pytest.mark.parametrize("case", ["zeros", "nan", "inf", "-inf", "empty"])
def test_quantize_special_tensors(fp8, case):
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
    else:
        x = x[:0]
    xd = torch.as_tensor(x).bfloat16().cuda()
    q, si = quantize_fp8(xd, fp8)
    rq, am, rsi = fo.quantize(xd.float().cpu().numpy(), FMT[fp8])
    assert np.array_equal(codes(q), rq)
    assert same_f32(f32(si), rsi) or (np.isnan(f32(si)) and np.isnan(rsi))
    if case in ("nan", "inf", "-inf"):
        assert np.isnan(f32(si))
    if case in ("zeros", "empty"):
        assert f32(si) == 1.0


@pytest.mark.parametrize("fp8", [E4, E5])
@pytest.mark.parametrize("bs", [32, 64])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_weights_match_oracle(fp8, bs, dtype):
    rng = np.random.default_rng(bs)
    bsmm = BlocksparseMatMul(bernoulli_layout(rng, 6, 5, 0.4), block_size=bs, feature_axis=1)
    w = special_values(rng, bsmm.blocks * bs * bs, dtype).reshape(bsmm.w_shape)
    wq, wq_t, si = quantize_fp8_weights(bsmm, w.cuda(), fp8)
    rq, rqt, am, rsi = fo.quantize_weights(w.float().numpy(), FMT[fp8])
    assert np.array_equal(codes(wq), rq) and np.array_equal(codes(wq_t), rqt)
    assert np.array_equal(codes(wq_t), codes(wq).transpose(0, 2, 1))
    assert same_f32(f32(si), rsi)


# ---- products --------------------------------------------------------------------------------------------------------
def make_layout(kind, rng):
    if kind == "dense":
        return np.ones((8, 6), np.int32)
    if kind == "random25":
        return bernoulli_layout(rng, 8, 6, 0.25)
    if kind == "ba":
        return barabasi_albert_layout(8, 0.25, rng)
    lay = bernoulli_layout(rng, 8, 6, 0.5)                       # "empty": input block row 2 and output block column 4
    lay[2, :] = 0
    lay[:, 4] = 0
    return lay


def dense_w(bsmm, blocks):
    bs = bsmm.bsize
    W = np.zeros((bsmm.C, bsmm.K))
    for b, (c, k) in enumerate(bsmm.updat_list):
        W[c * bs:(c + 1) * bs, k * bs:(k + 1) * bs] = blocks[b]
    return W


def reference(bsmm, xq, xs, wq, ws, bprop):
    """(y64, sum|x^||w^|, LUT entries per output column) in float64 from the dequantised operands."""
    xh = fo.decode(codes(xq), FMT[xq.dtype]).reshape(-1, xq.shape[-1]) * float(xs.item())
    W = dense_w(bsmm, fo.decode(codes(wq), FMT[wq.dtype]) * float(ws.item()))
    if bprop:
        W = W.T
    ent = np.repeat((bsmm.layout.T if bprop else bsmm.layout).sum(axis=0), bsmm.bsize).astype(np.float64)
    return xh @ W, np.abs(xh) @ np.abs(W), ent


def eps_tc(bs):
    return bs // 32 * EPS_TC_STEP


def bound(y64, sabs, ent, out_dtype, eps):
    b = (eps + (ent + 2) * EPS32) * sabs + U_OUT[dtype_name(out_dtype)] * np.abs(y64)
    return b + (2.0 ** -25 if out_dtype == torch.float16 else 0.0)   # fp16 subnormals round with an absolute error


def check_within(y, y64, sabs, ent, out_dtype, bs, what):
    """Asserts the bound; prints and returns the tensor-core error estimate max((|d| - bound without EPS_TC) / sum)."""
    got = y.detach().double().cpu().numpy().reshape(y64.shape)
    err = np.abs(got - y64)
    b = bound(y64, sabs, ent, out_dtype, eps_tc(bs))
    worst = np.unravel_index(np.argmax(err - b), err.shape)
    assert (err <= b).all(), "%s: |d| %.3e > bound %.3e at %s (y64 %.3e)" % (what, err[worst], b[worst], worst, y64[worst])
    live = sabs > 0
    est = float(((err - bound(y64, sabs, ent, out_dtype, 0.0))[live] / sabs[live]).max()) if live.any() else 0.0
    print("fp8-eps-estimate %s: %.3e (2^%.2f)" % (what, est, np.log2(est) if est > 0 else -np.inf))
    return est


def operands(bsmm, N, dtype, rng, bprop):
    feat = bsmm.K if bprop else bsmm.C
    x = torch.as_tensor(rng.normal(0, 1, (N, feat)).astype(np.float32)).to(dtype).cuda()
    w = torch.as_tensor(rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)).to(dtype).cuda()
    return x, w


@pytest.mark.parametrize("bs", [32, 64])
@pytest.mark.parametrize("kind", ["dense", "random25", "ba", "empty"])
@pytest.mark.parametrize("N", [1, 127, 128, 4099])
def test_xprop_elementwise(bs, kind, N):
    rng = np.random.default_rng(N * 7 + bs)
    lay = make_layout(kind, rng)
    bsmm = BlocksparseMatMul(lay, block_size=bs, feature_axis=1)
    for bprop, xfmt in ((False, E4), (True, E5)):
        for out in (torch.float16, torch.bfloat16):
            x, w = operands(bsmm, N, torch.bfloat16, rng, bprop)
            xq, xs = quantize_fp8(x, xfmt)
            wq, wq_t, ws = quantize_fp8_weights(bsmm, w, E4)
            y = xprop_fp8(bsmm, xq, wq if bprop else wq_t, xs, ws, bprop=bprop, out_dtype=out)
            assert _lib.last_kernel() == "wgmma_xprop_fp8_bs%d" % bs
            y64, sabs, ent = reference(bsmm, xq, xs, wq, ws, bprop)
            check_within(y, y64, sabs, ent, out, bs, "%s %s bs %d N %d %s" % (kind, "bprop" if bprop else "fprop", bs, N, out))
            if kind == "empty":
                col = slice(2 * bs, 3 * bs) if bprop else slice(4 * bs, 5 * bs)
                assert (y[:, col].view(torch.int16) == 0).all(), "an empty LUT row must give +0"


@pytest.mark.parametrize("bs", [32, 64])
def test_tensor_core_error_estimate(bs):
    """Dense 4096-wide fprop / bprop with fp16 output: there |y| ~ sum|x^||w^| / 64, so the output rounding stays far
    below the accumulation error, and (|y - y64| - u_out |y64| - (entries + 2) 2^-24 sum) / sum estimates EPS_TC."""
    rng = np.random.default_rng(5)
    bsmm = BlocksparseMatMul(np.ones((4096 // bs, 256 // bs), np.int32), block_size=bs, feature_axis=1)
    for bprop, xfmt in ((False, E4), (True, E5)):
        x, w = operands(bsmm, 1024, torch.bfloat16, rng, bprop)
        xq, xs = quantize_fp8(x, xfmt)
        wq, wq_t, ws = quantize_fp8_weights(bsmm, w, E4)
        y = xprop_fp8(bsmm, xq, wq if bprop else wq_t, xs, ws, bprop=bprop, out_dtype=torch.float16)
        y64, sabs, ent = reference(bsmm, xq, xs, wq, ws, bprop)
        check_within(y, y64, sabs, ent, torch.float16, bs, "dense 4096 %s bs %d" % ("bprop" if bprop else "fprop", bs))


# ---- autograd ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bs", [32, 64])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_matmul_fp8_autograd(bs, dtype):
    rng = np.random.default_rng(bs + 3)
    bsmm = BlocksparseMatMul(bernoulli_layout(rng, 8, 6, 0.3), block_size=bs, feature_axis=1)
    I = torch.as_tensor(rng.normal(0, 1, (3, 700, bsmm.C)).astype(np.float32)).to(dtype).cuda().requires_grad_()
    W = torch.as_tensor(rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)).to(dtype).cuda().requires_grad_()
    dy = torch.as_tensor(rng.normal(0, 1, (3, 700, bsmm.K)).astype(np.float32)).to(dtype).cuda()
    y = bsmm.matmul_fp8(I, W)
    assert y.dtype == dtype and y.shape == (3, 700, bsmm.K)
    y.backward(dy)
    assert I.grad.dtype == dtype and I.grad.shape == I.shape
    xq, xs = quantize_fp8(I.detach(), E4)
    wq, wq_t, ws = quantize_fp8_weights(bsmm, W.detach(), E4)
    y64, sabs, ent = reference(bsmm, xq, xs, wq, ws, False)
    check_within(y, y64, sabs, ent, dtype, bs, "matmul_fp8 y")
    dq, ds = quantize_fp8(dy, E5)
    dx64, sabs, ent = reference(bsmm, dq, ds, wq, ws, True)
    check_within(I.grad, dx64, sabs, ent, dtype, bs, "matmul_fp8 dx")
    ref_dw = bsmm.updat([I.detach()], [dy])
    assert torch.equal(W.grad.view(torch.int16), ref_dw.view(torch.int16))
    # inside group_param_grads the dw of every use goes to the group, as with bsmm(I, W)
    grads = []
    for op in (bsmm.matmul_fp8, bsmm):
        W2 = W.detach().clone().requires_grad_()
        with group_param_grads(bsmm, W2):
            (op(I.detach(), W2).float() * dy.float()).sum().backward()
            (op(I.detach() * 2, W2).float() * dy.float()).sum().backward()
        grads.append(W2.grad)
    assert torch.equal(grads[0].view(torch.int16), grads[1].view(torch.int16))


# ---- determinism and execution context ----------------------------------------------------------------------------
def fp8_pass(bsmm, I, W, dy):
    """matmul_fp8 forward and the fp8 bprop of dy, without autograd (so it can be captured)."""
    with torch.no_grad():
        y = bsmm.matmul_fp8(I, W)
        wq, _, ws = quantize_fp8_weights(bsmm, W, E4)
        dq, ds = quantize_fp8(dy, E5)
        dx = xprop_fp8(bsmm, dq, wq, ds, ws, bprop=True, out_dtype=I.dtype)
    return y, dx


def case(seed=0, N=4099, bsmm=None):
    rng = np.random.default_rng(seed)
    bsmm = bsmm or BlocksparseMatMul(bernoulli_layout(rng, 16, 12, 0.25), block_size=32, feature_axis=1)
    I = torch.as_tensor(rng.normal(0, 1, (N, bsmm.C)).astype(np.float32)).bfloat16().cuda()
    W = torch.as_tensor(rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)).bfloat16().cuda()
    dy = torch.as_tensor(rng.normal(0, 1, (N, bsmm.K)).astype(np.float32)).bfloat16().cuda()
    return bsmm, I, W, dy


def bits_equal(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_determinism():
    bsmm, I, W, dy = case()
    a, b = fp8_pass(bsmm, I, W, dy), fp8_pass(bsmm, I, W, dy)
    assert bits_equal(a[0], b[0]) and bits_equal(a[1], b[1])


def test_side_stream():
    bsmm, I, W, dy = case(1)
    ref = fp8_pass(bsmm, I, W, dy)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 20)                               # the side stream's work starts late
        got = fp8_pass(bsmm, I, W, dy)
    torch.cuda.current_stream().wait_stream(s)
    assert bits_equal(got[0], ref[0]) and bits_equal(got[1], ref[1])


def test_graph_replay():
    """Scales are computed and consumed on the device, so the whole pass captures without a host sync; a replay with
    new inputs gives what eager gives for them."""
    bsmm, I, W, dy = case(2)
    _, I2, W2, dy2 = case(3, bsmm=bsmm)
    fp8_pass(bsmm, I, W, dy)                                     # uploads the LUTs and configures the kernels
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fp8_pass(bsmm, I, W, dy)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fp8_pass(bsmm, I, W, dy)
    for src, dst in ((I2, I), (W2, W), (dy2, dy)):
        dst.copy_(src)
    graph.replay()
    torch.cuda.synchronize()
    ref = fp8_pass(bsmm, I2, W2, dy2)
    assert bits_equal(out[0], ref[0]) and bits_equal(out[1], ref[1])


# ---- large offsets -----------------------------------------------------------------------------------------------
def test_large_offsets():
    """x (N = 2^19 + 128 rows, C = 4096) has element offsets past 2^31 in bf16 and in fp8; sampled rows against float64."""
    N, C = (1 << 19) + 128, 4096
    need = N * C * 3 + (1 << 30)                                 # bf16 x + fp8 x + slack
    gc.collect()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip("the large-offset fp8 case needs %.1f GB of free device memory, %.1f GB are free" % (need / GB, free / GB))
    rng = np.random.default_rng(11)
    bsmm = BlocksparseMatMul(bernoulli_layout(rng, C // 32, 4, 0.25), block_size=32, feature_axis=1)
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((N, C), generator=gen, device="cuda", dtype=torch.bfloat16)
    w = torch.as_tensor(rng.normal(0, 0.1, bsmm.w_shape).astype(np.float32)).bfloat16().cuda()
    xq, xs = quantize_fp8(x, E4)
    del x
    wq, wq_t, ws = quantize_fp8_weights(bsmm, w, E4)
    y = xprop_fp8(bsmm, xq, wq_t, xs, ws, out_dtype=torch.bfloat16)
    cross = (1 << 31) // C
    rows = sorted(set([0, 1, cross - 1, cross, cross + 1, N - 2, N - 1] + [int(r) for r in rng.integers(0, N, 24)]))
    idx = torch.as_tensor(rows, device="cuda")
    sub = xq.index_select(0, idx)
    y64, sabs, ent = reference(bsmm, sub, xs, wq, ws, False)
    check_within(y.index_select(0, idx), y64, sabs, ent, torch.bfloat16, 32, "large offsets")
