"""fused_lstm_gates, split4 / concat4 and sparse_relu on the GPU: elementwise against the float64 oracle with per-element
bounds, bit for bit where the results are data movement or must not depend on the layout, against the reference's own
kernels, in every execution context, past 2^31 element offsets, and inside an unrolled block-sparse LSTM.

Gate bounds. Every fp32 quantity the kernel forms from exact inputs (the 16-bit inputs convert exactly) carries a
relative error of a few units of u = 2^-24: expf and tanhf are within 2 ulp (CUDA C Programming Guide, mathematical
functions), the IEEE division and each add or multiply within 1/2 ulp, so a sigmoid or tanh is within 4u. We allow 16u
per quantity and propagate it through the formula with the magnitudes of its terms (absolute values, every minus read as
a plus), so cancellation in sf c + si tu, 1 - t^2 or s - s^2 is covered; tanh' <= 1 carries the error of c_next into
tanh(c_next). The output is then rounded once: |ref| * u_out (2^-24 fp32, 2^-11 fp16, 2^-8 bf16), plus half the fp16
subnormal spacing (2^-25) and, for sigmoids that underflow, 1e-30.
"""
import threading

import numpy as np
import pytest
import torch

from blocksparse_b200 import (BlocksparseMatMul, bias_relu, concat4, dropout, fused_lstm_gates, layer_norm,
                              set_entropy, sparse_relu, split4)
from blocksparse_b200 import lstm
from oracle import lstm_oracle
from oracle import ref_lstm
from oracle.bsmm_oracle import MatmulOracle

gpu = pytest.mark.gpu
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
U32 = 2.0 ** -24
U_OUT = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
C_FN = 16 * U32
SLEEP_CYCLES = 1 << 22


def _abs_floor(dtype):
    return 1e-30 + (2.0 ** -25 if dtype == torch.float16 else 0.0)


def _np(t):
    return t.detach().double().cpu().numpy()


def _bits(t):
    return t.detach().contiguous().view(-1).view(torch.uint8)


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert torch.equal(_bits(a), _bits(b)), "%s differs bit for bit" % what


def _check(got, ref, bound, what):
    err = np.abs(_np(got) - ref)
    bad = err > bound
    assert not bad.any(), "%s: %d of %d outside the bound; worst err %.3e bound %.3e at ref %.3e" % (
        what, bad.sum(), bad.size, err[bad].max(), bound[bad][np.argmax(err[bad])], ref[bad][np.argmax(err[bad])])


def _gate_bounds(c, i, u, f, o, ec, eh, bias, fb, dtype):
    """Per-element bounds of (c_next, h_next) and (dc, di, du, df, do), derived as the module docstring says."""
    c, si, tu, sf, so, cn, tc = lstm_oracle._gates(c, i, u, f, o, bias, fb)
    ec = 0.0 if ec is None else np.asarray(ec, np.float64)
    eh = 0.0 if eh is None else np.asarray(eh, np.float64)
    uo, fl = U_OUT[dtype], _abs_floor(dtype)
    e_cn = C_FN * (np.abs(sf * c) + np.abs(si * tu))
    e_tc = e_cn + C_FN * np.abs(tc)
    hn = so * tc
    fwd = (e_cn + np.abs(cn) * uo + fl, so * e_cn + C_FN * np.abs(hn) + np.abs(hn) * uo + fl)
    m_dC = np.abs(eh * so) * (1 + tc * tc) + np.abs(ec)
    e_dC = C_FN * m_dC + np.abs(eh * so) * 2 * np.abs(tc) * e_tc
    grads = lstm_oracle.lstm_gates_grad(c, i, u, f, o, ec=None if np.isscalar(ec) else ec,
                                        eh=None if np.isscalar(eh) else eh, bias=bias, forget_bias=fb)
    raw = (e_dC * sf + C_FN * m_dC * sf,
           e_dC * np.abs(tu) * si * (1 - si) + C_FN * m_dC * np.abs(tu) * (si + si * si),
           e_dC * si * (1 - tu * tu) + C_FN * m_dC * si * (1 + tu * tu),
           e_dC * np.abs(c) * sf * (1 - sf) + C_FN * m_dC * np.abs(c) * (sf + sf * sf),
           np.abs(eh) * e_tc * so * (1 - so) + C_FN * np.abs(eh * tc) * (so + so * so))
    bwd = tuple(r + np.abs(g) * uo + fl for r, g in zip(raw, grads))
    return fwd, grads, bwd


def _inputs(shape, K, dtype, seed, odd=False, saturate=True):
    """c (shape), h (shape[:-1] + (4K,)), ec, eh: normal(0, 2), with some gate entries at +-30, +-60 and +-100 so that
    the sigmoids and tanh saturate. odd: every tensor starts one element past a 16-byte boundary."""
    g = torch.Generator().manual_seed(seed)
    hs = tuple(shape[:-1]) + (4 * K,)
    h = torch.randn(hs, generator=g) * 2
    if saturate:
        sel = torch.rand(hs, generator=g) < 0.05
        h[sel] = torch.tensor([30.0, -30.0, 60.0, -60.0, 100.0, -100.0])[torch.randint(0, 6, (int(sel.sum()),),
                                                                                          generator=g)]
    ts = [torch.randn(shape, generator=g) * 2, h, torch.randn(shape, generator=g), torch.randn(shape, generator=g)]
    out = []
    for t in ts:
        t = t.to(dtype)
        if odd:
            buf = torch.empty(t.numel() + 1, dtype=dtype, device="cuda")
            buf[1:].copy_(t.view(-1))
            out.append(buf[1:].view(t.shape))
        else:
            out.append(t.cuda())
    return out


SHAPES = {1: (3, 5, 1), 33: (2, 7, 33), 64: (64,), 4096: (6, 4096)}


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("K", list(SHAPES))
@pytest.mark.parametrize("bias", [None, torch.float32, torch.float16, torch.bfloat16],
                         ids=["nobias", "bias_f32", "bias_f16", "bias_bf16"])
def test_gates_against_float64(dtype, K, bias):
    shape = SHAPES[K]
    for odd in (False, True):
        c, h, ec, eh = _inputs(shape, K, dtype, seed=K + 7 * odd, odd=odd)
        b = None if bias is None else (torch.randn(4 * K, generator=torch.Generator().manual_seed(K)) * 0.5).to(bias).cuda()
        bn = None if b is None else _np(b)
        gates = np.split(_np(h), 4, axis=-1)
        for fb in (0.0, 1.0):
            for which in ("both", "ec", "eh"):
                hr = h.detach().requires_grad_()
                br = None if b is None else b.detach().requires_grad_()
                cn, hn = fused_lstm_gates(c, hr, bias=br, forget_bias=fb)
                fwd, grads, bwd = _gate_bounds(_np(c), *gates, None if which == "eh" else _np(ec),
                                               None if which == "ec" else _np(eh), bn, fb, dtype)
                what = "%s K %d fb %g %s odd %d" % (dtype, K, fb, which, odd)
                if which == "both":
                    refs = lstm_oracle.lstm_gates(_np(c), *gates, bias=bn, forget_bias=fb)
                    _check(cn, refs[0], fwd[0], "c_next " + what)
                    _check(hn, refs[1], fwd[1], "h_next " + what)
                outs, gouts = [], []
                if which != "eh":
                    outs.append(cn); gouts.append(ec)
                if which != "ec":
                    outs.append(hn); gouts.append(eh)
                got = torch.autograd.grad(outs, [hr] + ([br] if br is not None else []), gouts)
                _check(got[0], np.concatenate(grads[1:], axis=-1), np.concatenate(bwd[1:], axis=-1), "dh " + what)
                if br is not None:
                    # db is the column sum of dh as stored: bitwise bias_relu's db of that dh
                    x = torch.zeros_like(got[0]).requires_grad_()
                    b2 = b.clone().requires_grad_()
                    bias_relu(x, b2).backward(got[0])
                    _same(got[1], b2.grad, "db against bias_relu's db " + what)
        # dc against the oracle (c's gradient, both incoming gradients present)
        cr = c.detach().requires_grad_()
        cn, hn = fused_lstm_gates(cr, h, bias=b, forget_bias=1.0)
        torch.autograd.backward((cn, hn), (ec, eh))
        fwd, grads, bwd = _gate_bounds(_np(c), *gates, _np(ec), _np(eh), bn, 1.0, dtype)
        _check(cr.grad, grads[0], bwd[0], "dc %s K %d odd %d" % (dtype, K, odd))


@gpu
def test_missing_gradients():
    """A missing gradient of c_next or h_next reads as zero; with neither, every gradient is None."""
    c, h, ec, eh = _inputs((4, 8), 8, torch.float32, seed=3)
    b = torch.randn(32, device="cuda")
    leaves = [t.clone().requires_grad_() for t in (c, h, b)]
    cn, hn = fused_lstm_gates(leaves[0], leaves[1], bias=leaves[2])
    for outs, gouts, full in (((hn,), (eh,), (torch.zeros_like(ec), eh)), ((cn,), (ec,), (ec, torch.zeros_like(eh)))):
        got = torch.autograd.grad(outs, leaves, gouts, retain_graph=True)
        ref = torch.autograd.grad((cn, hn), leaves, full, retain_graph=True)
        for a, r in zip(got, ref):
            assert torch.equal(a, r)
    assert lstm._LstmGatesFunction.backward(cn.grad_fn, None, None) == (None,) * 7


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("shape,K", [((70000, 16), 16), ((5, 3, 33), 33), ((2, 1024), 1024)])
def test_fused_equals_four_tensor_form_over_split4(dtype, shape, K):
    """fused_lstm_gates(c, h) and fused_lstm_gates(c, *split4(h)) agree bit for bit, forward and backward (concat4 of the
    four gate gradients); split4 / concat4 are exact inverses. shape (70000, 16) has rows past the reference's grid."""
    c, h, ec, eh = _inputs(shape, K, dtype, seed=11)
    parts = split4(h)
    for j, p in enumerate(parts):
        _same(p, h[..., j * K:(j + 1) * K].contiguous(), "split4 block %d" % j)
    _same(concat4(*parts), h, "concat4(split4(h))")
    outs = []
    for fused in (True, False):
        cr, hr = c.clone().requires_grad_(), h.clone().requires_grad_()
        cn, hn = fused_lstm_gates(cr, hr, forget_bias=0.5) if fused else fused_lstm_gates(cr, *split4(hr),
                                                                                          forget_bias=0.5)
        torch.autograd.backward((cn, hn), (ec, eh))
        outs.append((cn, hn, cr.grad, hr.grad))
    for a, b, what in zip(outs[0], outs[1], ("c_next", "h_next", "dc", "dh")):
        _same(a, b, what)
    # rows are independent: the whole equals the rows run in two halves (each within the reference's grid)
    half = shape[0] // 2
    if len(shape) == 2 and shape[0] > 65535:
        for lo, hi in ((0, half), (half, shape[0])):
            cn, hn = fused_lstm_gates(c[lo:hi], h[lo:hi], forget_bias=0.5)
            _same(cn, outs[0][0][lo:hi], "c_next rows %d:%d" % (lo, hi))
            _same(hn, outs[0][1][lo:hi], "h_next rows %d:%d" % (lo, hi))


def _run_all(c, h, b, ec, eh, x):
    """Every op forward and backward; returns all outputs and gradients."""
    c, h, b, x = (t.detach().requires_grad_() for t in (c, h, b, x))
    cn, hn = fused_lstm_gates(c, h, bias=b, forget_bias=0.5)
    g1 = torch.autograd.grad((cn, hn), (c, h, b), (ec, eh))
    cn4, hn4 = fused_lstm_gates(c, *split4(h))
    g2 = torch.autograd.grad((cn4, hn4), (c, h), (ec, eh))
    y = sparse_relu(x, alpha=0.5)
    g3 = torch.autograd.grad(y, x, x)
    return [cn, hn, *g1, cn4, hn4, *g2, y, *g3]


def _make(seed, device, dtype=torch.bfloat16, N=48, K=40):
    g = torch.Generator().manual_seed(seed)
    shapes = [(N, K), (N, 4 * K), (4 * K,), (N, K), (N, K), (N, 3, 300)]
    return [(torch.randn(s, generator=g) * 2).to(device=device, dtype=dtype) for s in shapes]


@gpu
def test_two_runs_are_bitwise_identical():
    ins = _make(0, "cuda")
    for a, b in zip(_run_all(*ins), _run_all(*ins)):
        _same(a, b, "second run")
    x = torch.randn(9, 100000, device="cuda")
    _same(sparse_relu(x), sparse_relu(x), "sparse_relu long rows")


@gpu
def test_side_stream_with_inputs_still_being_written():
    staging = _make(7, "cuda")
    ref = _run_all(*staging)
    bufs = [torch.full_like(t, float("nan")) for t in staging]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for b, t in zip(bufs, staging):
            b.copy_(t)
        out = _run_all(*bufs)
    s.synchronize()
    for a, r in zip(out, ref):
        _same(a, r, "side stream")


@gpu
def test_graph_replay_with_new_inputs():
    static = _make(0, "cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _run_all(*static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = _run_all(*static)
    for i in range(1, 4):
        new = _make(i, "cuda")
        for t, n in zip(static, new):
            t.copy_(n)
        graph.replay()
        for a, r in zip(out, _run_all(*new)):
            _same(a, r, "replay %d" % i)


@gpu
def test_two_host_threads():
    ins = [_make(10 + i, "cuda") for i in range(2)]
    refs = [_run_all(*x) for x in ins]
    results, errors = [None, None], []

    def worker(i):
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                for _ in range(3):
                    results[i] = _run_all(*ins[i])
                torch.cuda.current_stream().synchronize()
        except Exception as e:                       # noqa: BLE001  (re-raised in the main thread)
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for i in range(2):
        for a, r in zip(results[i], refs[i]):
            _same(a, r, "thread %d" % i)


@gpu
def test_second_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    ref = _run_all(*_make(5, "cuda:0"))
    out = _run_all(*_make(5, "cuda:1"))
    for a, r in zip(out, ref):
        assert a.device == torch.device("cuda:1")
        _same(a.to("cuda:0"), r, "cuda:1")


# ---- sparse_relu -------------------------------------------------------------------------------------------------------
def _srelu_bound(xn, alpha, ref, dtype):
    """The cutoff mean + alpha std is formed in fp32: each lane adds ceil(K / 32) values in order, then a tree of at
    most 13 levels, so the mean and the centred sum of squares carry at most n = ceil(K / 32) + 32 roundings each; the
    cutoff is off by at most 2 n u (mean|x| + |alpha| std) + u |cutoff|, and y = x - cutoff adds u |y| before the
    rounding to the output."""
    K = xn.shape[-1]
    n = -(-K // 32) + 32
    m_abs = np.abs(xn).mean(axis=-1, keepdims=True)
    sd = xn.std(axis=-1, keepdims=True)
    cut = xn.mean(axis=-1, keepdims=True) + alpha * sd
    e_cut = 2 * n * U32 * (m_abs + abs(alpha) * sd) + U32 * np.abs(cut)
    return e_cut + U32 * np.abs(ref) + U_OUT[dtype] * np.abs(ref) + _abs_floor(dtype)


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("K", [1, 2, 7, 33, 64, 1000, 1024, 1025, 4096, 8192, 8193, 100000])
def test_sparse_relu_against_float64(dtype, K):
    rows = max(1, min(64, 400000 // K))
    g = torch.Generator().manual_seed(K)
    for alpha in (1.0, 0.25, -0.5):
        for odd in (False, True):
            x = (torch.randn(rows, K, generator=g) * 3 + 1).to(dtype)
            if odd:
                buf = torch.empty(x.numel() + 1, dtype=dtype, device="cuda")
                buf[1:].copy_(x.view(-1))
                xc = buf[1:].view(x.shape)
            else:
                xc = x.cuda()
            xr = xc.detach().requires_grad_()
            y = sparse_relu(xr, alpha=alpha)
            xn = _np(x)
            ref = lstm_oracle.sparse_relu(xn, alpha)
            _check(y, ref, _srelu_bound(xn, alpha, ref, dtype), "sparse_relu %s K %d alpha %g odd %d" % (dtype, K, alpha,
                                                                                                       odd))
            if K == 1:
                assert not y.any()
            dy = torch.randn(x.shape, generator=g).to(dtype).cuda()
            y.backward(dy)
            _same(xr.grad, torch.where(y > 0, dy, torch.zeros_like(dy)), "sparse_relu grad")


@gpu
def test_sparse_relu_constant_rows_and_cancellation():
    for dtype in DTYPES:
        for v in (3.25, 0.1, -7.0):
            x = torch.full((5, 777), v, dtype=dtype, device="cuda")
            for alpha in (0.0, 1.0, -1.0):
                assert not sparse_relu(x, alpha).any(), (dtype, v, alpha)
    # mean 1e3, std 1: E[x^2] - E[x]^2 in fp32 would lose the variance (1e6 * 2^-24 * K >> 1)
    g = torch.Generator().manual_seed(0)
    for K in (512, 4096, 20000):
        x = torch.randn(16, K, generator=g, dtype=torch.float64) + 1000.0
        xf = x.float()
        y = sparse_relu(xf.cuda(), 1.0)
        xn = xf.double().numpy()
        ref = lstm_oracle.sparse_relu(xn, 1.0)
        _check(y, ref, _srelu_bound(xn, 1.0, ref, torch.float32), "sparse_relu mean 1e3 K %d" % K)
        assert np.abs(_np(y) - ref).max() < 0.05
        assert (ref > 0).mean() > 0.1


@gpu
def test_sparse_relu_rows_past_the_grid_and_in_halves():
    x = torch.randn(70000, 48, device="cuda", dtype=torch.bfloat16)
    y = sparse_relu(x)
    _same(torch.cat([sparse_relu(x[:35000]), sparse_relu(x[35000:])]), y, "sparse_relu 70000 rows")


# ---- against the reference's kernels --------------------------------------------------------------------------------------
def _ulp16(a, dtype):
    mant, emin = (7, -126) if dtype == torch.bfloat16 else (10, -14)
    e = np.floor(np.log2(np.maximum(np.abs(a), 2.0 ** emin)))
    return 2.0 ** (e - mant)


def _ref_close(ours, theirs, mag, dtype, what):
    """fp32: the reference's approximate exp / reciprocal differ from ours in the last bits (64 u of the terms'
    magnitude); 16-bit: at most one output ulp, plus that fp32 difference before the rounding."""
    a, b = _np(ours), _np(theirs)
    bound = 64 * U32 * mag
    if dtype != torch.float32:
        bound = bound + _ulp16(np.maximum(np.abs(a), np.abs(b)), dtype)
    err = np.abs(a - b)
    assert (err <= bound).all(), "%s: worst %.3e against the reference (bound %.3e)" % (what, err.max(),
                                                                                         bound[np.argmax(err - bound)])


@gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("K", [64, 33])
def test_against_reference_kernels(dtype, K):
    why = ref_lstm.missing()
    if why:
        pytest.skip(why)
    N = 100
    c, h, ec, eh = _inputs((N, K), K, dtype, seed=K, saturate=False)
    gates = np.split(_np(h), 4, axis=-1)
    for bias in (None, (torch.randn(4 * K, generator=torch.Generator().manual_seed(1)) * 0.5).cuda()):
        bn = None if bias is None else _np(bias)
        _, si, tu, sf, so, cn_, tc = lstm_oracle._gates(_np(c), *gates, bn, 1.0)
        m_c = np.abs(sf * _np(c)) + np.abs(si * tu) + np.abs(cn_)
        ours = fused_lstm_gates(c, h, bias=bias)
        theirs = ref_lstm.lstm_gates(c, h, bias=bias)
        _ref_close(ours[0], theirs[0], m_c, dtype, "c_next")
        _ref_close(ours[1], theirs[1], m_c + 1, dtype, "h_next")
        cr, hr = c.clone().requires_grad_(), h.clone().requires_grad_()
        torch.autograd.backward(fused_lstm_gates(cr, hr, bias=bias), (ec, eh))
        tdc, tdh = ref_lstm.lstm_gates_grad(c, h, eh, ec=ec, bias=bias)
        m_g = (np.abs(_np(eh)) * (1 + m_c) + np.abs(_np(ec))) * (1 + np.abs(_np(c)))
        _ref_close(cr.grad, tdc, m_g, dtype, "dc")
        _ref_close(hr.grad, tdh, np.concatenate([m_g] * 4, axis=-1), dtype, "dh")
    i, u, f, o = split4(h)
    m = np.abs(_np(c)) + 2
    ours = fused_lstm_gates(c, i, u, f, o, forget_bias=0.5)
    theirs = ref_lstm.lstm_gates4(c, i, u, f, o, forget_bias=0.5)
    for a, b, w in zip(ours, theirs, ("c_next4", "h_next4")):
        _ref_close(a, b, m, dtype, w)
    leaves = [t.clone().requires_grad_() for t in (c, i, u, f, o)]
    torch.autograd.backward(fused_lstm_gates(*leaves, forget_bias=0.5), (ec, eh))
    theirs = ref_lstm.lstm_gates4_grad(c, i, u, f, o, eh, ec=ec, forget_bias=0.5)
    m_g = (np.abs(_np(eh)) * (1 + m) + np.abs(_np(ec))) * m
    for t, b, w in zip(leaves, theirs, ("dc4", "di", "du", "df", "do")):
        _ref_close(t.grad, b, m_g, dtype, w)
    # sparse_relu on well-conditioned rows (the reference's E[x^2] - E[x]^2 is accurate there)
    for k in (K, 3000):
        x = torch.randn(32, k, device="cuda").to(dtype)
        xn = _np(x)
        bound = _srelu_bound(xn, 1.0, lstm_oracle.sparse_relu(xn, 1.0), dtype) * 2
        a, b = _np(sparse_relu(x)), _np(ref_lstm.sparse_relu(x))
        assert (np.abs(a - b) <= bound + (0 if dtype == torch.float32 else _ulp16(np.maximum(abs(a), abs(b)), dtype))).all()


# ---- element offsets past 2^31 -----------------------------------------------------------------------------------------------
@gpu
def test_large_offsets_bf16():
    """bf16, about 12 GiB at the peak: the rows past element 2^31 equal the same rows run alone, bit for bit."""
    K = 1 << 14
    N = (1 << 31) // (4 * K) + 8
    torch.manual_seed(0)
    h = torch.randn(N, 4 * K, device="cuda", dtype=torch.bfloat16)
    c = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    eh = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    cn, hn = fused_lstm_gates(c, h)
    cs, hs = fused_lstm_gates(c[-5:], h[-5:])
    _same(cn[-5:], cs, "c_next past 2^31")
    _same(hn[-5:], hs, "h_next past 2^31")
    del cn, hn
    hr = h.requires_grad_()
    dh, = torch.autograd.grad(fused_lstm_gates(c, hr)[1], hr, eh)
    hs = h[-5:].detach().requires_grad_()
    dhs, = torch.autograd.grad(fused_lstm_gates(c[-5:], hs)[1], hs, eh[-5:])
    _same(dh[-5:], dhs, "dh past 2^31")
    del h, hr, c, eh, dh
    torch.cuda.empty_cache()
    rows = (1 << 31) // 4096 + 8
    x = torch.randn(rows, 4096, device="cuda", dtype=torch.bfloat16)
    y = sparse_relu(x)
    _same(y[-5:], sparse_relu(x[-5:]), "sparse_relu past 2^31")
    del x
    dy = torch.randn_like(y)
    dx = lstm._relu_mask_grad(dy, y)
    _same(dx[-5:], torch.where(y[-5:] > 0, dy[-5:], torch.zeros_like(dy[-5:])), "relu mask past 2^31")
    del y, dy, dx
    torch.cuda.empty_cache()


# ---- an unrolled block-sparse LSTM ---------------------------------------------------------------------------------------------
T, BS = 4, 32


def _layout(rows, cols, seed):
    lay = (np.random.default_rng(seed).random((rows, cols)) < 0.5).astype(np.int32)
    lay[:, 0] = 1
    return lay


def _sig64(z):
    return torch.sigmoid(z)


def _ln64(z, g, b, segments, axis):
    if axis == 0:
        m, v = z.mean(0, keepdim=True), z.var(0, unbiased=False, keepdim=True)
        return (z - m) / torch.sqrt(v + 1e-6) * g.view(-1, 1) + b.view(-1, 1)
    N, K = z.shape
    zs = z.view(N, segments, K // segments)
    m, v = zs.mean(-1, keepdim=True), zs.var(-1, unbiased=False, keepdim=True)
    return ((zs - m) / torch.sqrt(v + 1e-6)).view(N, K) * g + b


class _FeaturesLast:
    """x_t (N, 4K) plus BlocksparseMatMul(feature_axis=1) of h (K -> 4K), layer_norm(segments=4), the fused form."""
    N, K = 32, 128

    def __init__(self):
        self.lay = _layout(self.K // BS, 4 * self.K // BS, 0)
        self.bsmm = BlocksparseMatMul(self.lay, block_size=BS, feature_axis=1)
        self.orc = MatmulOracle(self.lay, BS, 1)

    def make(self, seed):
        g = torch.Generator().manual_seed(seed)
        r = lambda *s: torch.randn(*s, generator=g)             # noqa: E731
        return [r(*self.bsmm.w_shape) * 0.1, torch.rand(4 * self.K, generator=g) + 0.5, r(4 * self.K) * 0.1,
                r(T, self.N, 4 * self.K), r(self.N, self.K), r(self.N, self.K), r(T, self.N, self.K), r(self.N, self.K)]

    def run(self, w, g, b, xs, c, h, es, ec):
        """(loss terms' outputs..., grads of w, g, b, xs, c0, h0) with our ops."""
        w, g, b, xs, c0, h0 = (t.detach().requires_grad_() for t in (w, g, b, xs, c, h))
        c, h, loss = c0, h0, 0
        for t in range(T):
            z = layer_norm(self.bsmm(h, w) + xs[t], g, b, axis=1, segments=4)
            c, h = fused_lstm_gates(c, z)
            loss = loss + (h * es[t]).sum()
        loss = loss + (c * ec).sum()
        return [c, h] + list(torch.autograd.grad(loss, (w, g, b, xs, c0, h0))), None

    def ref(self, w, g, b, xs, c, h, es, ec, extra):
        D = torch.tensor(self.orc.dense_weight(w.double().cpu().numpy()), requires_grad=True)
        g, b, xs, c0, h0 = (t.detach().double().cpu().requires_grad_() for t in (g, b, xs, c, h))
        es, ec = es.double().cpu(), ec.double().cpu()
        c, h, loss = c0, h0, 0
        for t in range(T):
            z = _ln64(h @ D + xs[t], g, b, 4, 1)
            i, u, f, o = z.split(self.K, -1)
            c = _sig64(f + 1.0) * c + _sig64(i) * torch.tanh(u)
            h = _sig64(o) * torch.tanh(c)
            loss = loss + (h * es[t]).sum()
        loss = loss + (c * ec).sum()
        grads = torch.autograd.grad(loss, (D, g, b, xs, c0, h0))
        return [c, h, grads[0]] + list(grads[1:])

    def dw(self, w):
        return torch.tensor(self.orc.dense_weight(w.double().cpu().numpy()))


class _FeatureAxis0:
    """mLSTM style, (K, N) activations: per gate BlocksparseMatMul(feature_axis=0) of h plus x_t, layer_norm(axis=0),
    dropout on u, the four-tensor form."""
    N, K = 48, 96

    def __init__(self):
        self.lays = [_layout(self.K // BS, self.K // BS, 1 + j) for j in range(4)]
        self.bsmms = [BlocksparseMatMul(lay, block_size=BS, feature_axis=0) for lay in self.lays]
        self.orcs = [MatmulOracle(lay, BS, 0) for lay in self.lays]

    def make(self, seed):
        g = torch.Generator().manual_seed(seed)
        r = lambda *s: torch.randn(*s, generator=g)             # noqa: E731
        ws = [r(*m.w_shape) * 0.1 for m in self.bsmms]
        return ws + [torch.rand(4, self.K, generator=g) + 0.5, r(4, self.K) * 0.1, r(T, 4, self.K, self.N),
                     r(self.K, self.N), r(self.K, self.N), r(T, self.K, self.N), r(self.K, self.N)]

    def run(self, *args):
        ws, (g, b, xs, c, h, es, ec) = args[:4], args[4:]
        ws = [w.detach().requires_grad_() for w in ws]
        g, b, xs, c0, h0 = (t.detach().requires_grad_() for t in (g, b, xs, c, h))
        c, h, loss, masks = c0, h0, 0, []
        for t in range(T):
            z = [layer_norm(self.bsmms[j](h, ws[j]) + xs[t, j], g[j], b[j], axis=0) for j in range(4)]
            u, mask = dropout(z[1], 0.9)
            masks.append(mask)
            c, h = fused_lstm_gates(c, z[0], u, z[2], z[3])
            loss = loss + (h * es[t]).sum()
        loss = loss + (c * ec).sum()
        return [c, h] + list(torch.autograd.grad(loss, ws + [g, b, xs, c0, h0])), masks

    def ref(self, *args):
        ws, (g, b, xs, c, h, es, ec), masks = args[:4], args[4:11], args[11]
        Ds = [torch.tensor(o.dense_weight(w.double().cpu().numpy()), requires_grad=True) for o, w in zip(self.orcs, ws)]
        g, b, xs, c0, h0 = (t.detach().double().cpu().requires_grad_() for t in (g, b, xs, c, h))
        es, ec = es.double().cpu(), ec.double().cpu()
        c, h, loss = c0, h0, 0
        for t in range(T):
            z = [_ln64(Ds[j].t() @ h + xs[t, j], g[j], b[j], 1, 0) for j in range(4)]
            keep = dropout(torch.ones(self.K, self.N, device="cuda"), 0.9, mask=masks[t])[0].double().cpu()
            u = z[1] * keep
            c = _sig64(z[2] + 1.0) * c + _sig64(z[0]) * torch.tanh(u)
            h = _sig64(z[3]) * torch.tanh(c)
            loss = loss + (h * es[t]).sum()
        loss = loss + (c * ec).sum()
        return [c, h] + list(torch.autograd.grad(loss, Ds + [g, b, xs, c0, h0]))


def _compare_lstm(model, got, ref, what, weights):
    """fp32 through four steps of matmul, layer norm and gates: within 1e-4 of each quantity's largest magnitude (the
    float64 composition has no rounding; fp32 accumulates a few ulp per op over about 40 ops)."""
    for n, (a, r) in enumerate(zip(got, ref)):
        a = a.detach().double().cpu()
        if n - 2 < weights and n >= 2:
            orc = model.orc if hasattr(model, "orc") else model.orcs[n - 2]
            a = torch.tensor(orc.dense_weight(a.numpy()))
            r = r * (torch.tensor(orc.dense_weight(np.ones(orc_wshape(orc)))) > 0)
        r = r.detach()
        err = (a - r).abs().max().item()
        scale = r.abs().max().item()
        assert err <= 1e-4 * scale + 1e-6, "%s output %d: max err %.3e, max |ref| %.3e" % (what, n, err, scale)


def orc_wshape(orc):
    return (len(orc.updat_list), orc.bsize, orc.bsize)


@gpu
@pytest.mark.parametrize("model", [_FeaturesLast, _FeatureAxis0], ids=["features_last", "feature_axis0"])
def test_unrolled_blocksparse_lstm(model):
    m = model()
    nw = 1 if model is _FeaturesLast else 4
    set_entropy(5)
    ins = [t.cuda() for t in m.make(0)]
    got, masks = m.run(*ins)
    ref = m.ref(*ins, masks)
    _compare_lstm(m, got, ref, "eager", nw)
    # the same step captured in a CUDA graph, replayed with new inputs
    static = [t.clone() for t in ins]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            m.run(*static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, omasks = m.run(*static)
    for i in range(1, 3):
        new = [t.cuda() for t in m.make(i)]
        for t, n in zip(static, new):
            t.copy_(n)
        graph.replay()
        torch.cuda.synchronize()
        ref = m.ref(*new, omasks)
        _compare_lstm(m, out, ref, "replay %d" % i, nw)
        if omasks is None:
            for a, b in zip(out, m.run(*new)[0]):
                _same(a, b, "replay %d against eager" % i)
