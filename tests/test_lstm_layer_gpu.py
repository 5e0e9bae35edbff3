"""grouped_lstm and FusedBasicLSTMCell on the GPU: against the float64 oracle, the layer without layer norm bit for bit
against a loop of cells, the fused layer-norm step against layer_norm followed by fused_lstm_gates, the kernel's
gradient as one dw_matmul_large_n over the saved rows, in every execution context, and past 2^31 element offsets.

Tolerance. The oracle runs in float64 on the operands as the layer sees them (inputs and states in their dtype, the
kernel cast to it). Each step rounds z, c_t and h_t (and in the backward dz, dc and dh) once to the dtype: 4u per step
with u = 2^-24 (fp32), 2^-11 (fp16), 2^-8 (bf16); each step also sums up to L terms in fp32, 4 sqrt(L) 2^-24 with
L = max(in + width, 4 width, T N). Over T + 1 steps (the backward's extra dW / reduce) the l2-relative error of every
output and gradient is held to (T + 1) (4u + 4 sqrt(L) 2^-24).
"""
import math

import numpy as np
import pytest
import torch

from blocksparse_b200 import FusedBasicLSTMCell, _lib, dw_matmul_large_n, fused_lstm_gates, grouped_lstm, layer_norm
from blocksparse_b200 import lstm_layer
from oracle import lstm_layer_oracle

pytestmark = pytest.mark.gpu
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
U = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
# (N, T, in, width, 2-D input): block multiples, odd widths, T = 1 in the (N, in) form
SHAPES = [(64, 5, 64, 32, False), (7, 3, 13, 20, False), (5, 1, 13, 5, True), (9, 1, 32, 32, False)]


def _np(t):
    return None if t is None else t.detach().double().cpu().numpy()


def _bits(t):
    return t.detach().contiguous().view(-1).view(torch.uint8)


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert torch.equal(_bits(a), _bits(b)), "%s differs bit for bit" % what


def _tol(dtype, N, T, In, W):
    L = max(In + W, 4 * W, T * N)
    return (T + 1) * (4 * U[dtype] + 4 * math.sqrt(L) * 2.0 ** -24)


def _close(got, ref, tol, what):
    ref = np.asarray(ref, np.float64)
    err = np.linalg.norm(_np(got) - ref) / max(np.linalg.norm(ref), 1e-30)
    assert err <= tol, "%s: l2-relative error %.3e above %.3e" % (what, err, tol)


def _make(N, T, In, W, dtype, seed, two_d=False, layernorm=True, pdtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((N, In) if two_d else (N, T, In), generator=g)
    c, h = torch.randn(N, W, generator=g), torch.randn(N, W, generator=g) * 0.5
    kernel = torch.randn(In + W, 4 * W, generator=g) / math.sqrt(In + W)
    bias = torch.randn(4 * W, generator=g) * 0.3
    gain = 1 + torch.randn(4 * W, generator=g) * 0.2 if layernorm else None
    d_out, d_c, d_h = torch.randn(N, T, W, generator=g), torch.randn(N, W, generator=g), torch.randn(N, W, generator=g)
    cu = lambda t, d: None if t is None else t.to(d).cuda()
    return (cu(x, dtype), cu(c, dtype), cu(h, dtype), cu(kernel, pdtype), cu(bias, pdtype), cu(gain, pdtype),
            cu(d_out, dtype), cu(d_c, dtype), cu(d_h, dtype))


def _run(x, c, h, kernel, bias, gain, d_out, d_c, d_h, layernorm, T, W):
    leaves = [t.detach().requires_grad_() for t in (x, c, h, kernel, bias)] + \
             ([gain.detach().requires_grad_()] if layernorm else [])
    out, (cT, hT) = grouped_lstm(leaves[0], W, T, [leaves[1], leaves[2]], leaves[3], leaves[4],
                                 leaves[5] if layernorm else None, layernorm=layernorm)
    grads = torch.autograd.grad((out, cT, hT), leaves, (d_out, d_c, d_h))
    return (out, cT, hT) + tuple(grads)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("layernorm", [True, False], ids=["ln", "noln"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "N%d_T%d_in%d_w%d%s" % (s[:4] + ("_2d" if s[4] else "",)))
def test_against_float64(dtype, layernorm, shape):
    N, T, In, W, two_d = shape
    ins = _make(N, T, In, W, dtype, seed=N + T + W, two_d=two_d, layernorm=layernorm)
    x, c, h, kernel, bias, gain, d_out, d_c, d_h = ins
    res = _run(*ins, layernorm, T, W)
    out, cT, hT = res[:3]
    assert out.shape == (N, T, W) and out.dtype == dtype and cT.shape == hT.shape == (N, W)
    _same(out[:, -1], hT, "output[:, -1] and h_T")
    kq = _np(kernel.to(dtype))                    # the oracle sees the kernel as the product does
    args = (_np(x), _np(c), _np(h), kq, _np(bias), _np(gain), layernorm)
    ro, rc, rh = lstm_layer_oracle.grouped_lstm(*args)
    refs = lstm_layer_oracle.grouped_lstm_grad(*args, _np(d_out), _np(d_c), _np(d_h))
    tol = _tol(dtype, N, T, In, W)
    what = "%s ln %d N %d T %d in %d W %d" % (dtype, layernorm, N, T, In, W)
    for got, ref, name in zip(res, (ro, rc, rh) + refs, ("out", "c_T", "h_T", "dx", "dc0", "dh0", "dkernel", "dbias",
                                                         "dgain")):
        if ref is None:
            continue
        assert got.dtype == (kernel.dtype if name in ("dkernel", "dbias", "dgain") else dtype), name
        assert tuple(got.shape) == np.shape(ref), name
        _close(got, ref, tol, "%s %s" % (name, what))


@pytest.mark.parametrize("pdtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_parameters_in_16_bit(pdtype):
    """kernel, bias and gain in a 16-bit dtype under fp32 inputs: gradients come back in their dtype."""
    N, T, In, W = 6, 3, 13, 20
    ins = _make(N, T, In, W, torch.float32, seed=11, pdtype=pdtype)
    res = _run(*ins, True, T, W)
    x, c, h, kernel, bias, gain, d_out, d_c, d_h = ins
    args = (_np(x), _np(c), _np(h), _np(kernel), _np(bias), _np(gain), True)
    refs = lstm_layer_oracle.grouped_lstm_grad(*args, _np(d_out), _np(d_c), _np(d_h))
    for got, ref, name in zip(res[6:], refs[3:], ("dkernel", "dbias", "dgain")):
        assert got.dtype == pdtype
        _close(got, ref, _tol(pdtype, N, T, In, W), name)


def test_empty_minibatch_launches_nothing():
    for layernorm in (True, False):
        ins = list(_make(0, 3, 13, 20, torch.bfloat16, seed=1, layernorm=layernorm))
        before = _lib.last_kernel()
        res = _run(*ins, layernorm, 3, 20)
        assert _lib.last_kernel() == before
        assert res[0].shape == (0, 3, 20) and res[1].shape == res[2].shape == (0, 20)
        assert res[3].shape == (0, 3, 13)
        for g in res[6:]:
            assert not g.any()


def test_argument_errors_on_the_gpu():
    x, c, h, kernel, bias, gain = _make(4, 2, 13, 20, torch.float16, seed=2)[:6]
    before = _lib.last_kernel()
    bad = [lambda: grouped_lstm(x, 20, 3, [c, h], kernel, bias, gain),             # timesteps
           lambda: grouped_lstm(x[:, 0], 20, 2, [c, h], kernel, bias, gain),       # 2-D needs T = 1
           lambda: grouped_lstm(x, 21, 2, [c, h], kernel, bias, gain),             # width
           lambda: grouped_lstm(x, 20, 2, [c.float(), h], kernel, bias, gain),     # state dtype
           lambda: grouped_lstm(x, 20, 2, [c[:3], h], kernel, bias, gain),
           lambda: grouped_lstm(x, 20, 2, [c], kernel, bias, gain),
           lambda: grouped_lstm(x, 20, 2, [c, h.cpu()], kernel, bias, gain),       # mixed devices
           lambda: grouped_lstm(x, 20, 2, [c, h], kernel[:-1], bias, gain),
           lambda: grouped_lstm(x, 20, 2, [c, h], kernel.double(), bias, gain),
           lambda: grouped_lstm(x, 20, 2, [c, h], kernel, bias[:-1], gain),
           lambda: grouped_lstm(x, 20, 2, [c, h], kernel, bias, None),             # layernorm needs a gain
           lambda: grouped_lstm(x, 20, 2, [c, h], kernel, bias, gain.half()),      # gain and bias dtypes
           lambda: grouped_lstm(x, 20, 2, [c, h], kernel, bias, gain, layernorm=False)]
    cell = FusedBasicLSTMCell(20, 13, device="cuda")
    bad += [lambda: cell(x[:, 0].float(), (c.float(), h.float())[:1]),
            lambda: cell(x[:, 0].float(), (c, h)),                              # state dtype
            lambda: cell(x[:, 0, :12].float(), (c.float(), h.float())),
            lambda: FusedBasicLSTMCell(20, 13, state_is_tuple=False, device="cuda")(x[:, 0].float(), c.float())]
    for call in bad:
        with pytest.raises(ValueError):
            call()
    assert _lib.last_kernel() == before


# ---- against the cell and the two-op composition -------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("shape", SHAPES[:2], ids=["blocks", "odd"])
def test_without_layernorm_equals_a_loop_of_cells(dtype, shape):
    N, T, In, W, _ = shape
    cell = FusedBasicLSTMCell(W, In, forget_bias=1.0, device="cuda")
    with torch.no_grad():
        cell.bias.normal_(0, 0.3)
    x, c, h, _, _, _, d_out, d_c, d_h = _make(N, T, In, W, dtype, seed=5, layernorm=False)
    res = _run(x, c, h, cell.kernel, cell.bias, None, d_out, d_c, d_h, False, T, W)
    leaves = [t.detach().requires_grad_() for t in (x, c, h)]
    cc, hh, outs = leaves[1], leaves[2], []
    for t in range(T):
        hh, (cc, _) = cell(leaves[0][:, t], (cc, hh))
        outs.append(hh)
    out = torch.stack(outs, 1)
    _same(res[0], out, "output")
    _same(res[1], cc, "c_T")
    _same(res[2], hh, "h_T")
    grads = torch.autograd.grad((out, cc, hh), leaves + [cell.kernel, cell.bias], (d_out, d_c, d_h))
    tol = _tol(dtype, N, T, In, W)
    for a, b, name in zip(res[3:], grads, ("dx", "dc0", "dh0", "dkernel", "dbias")):
        _close(a, _np(b), tol, name)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("K", [5, 20, 256, 1024, 3000])
def test_fused_step_against_layer_norm_then_gates(dtype, K):
    """The fused step differs from layer_norm(segments=4) + fused_lstm_gates only by that composition's rounding of
    the normalised value (and, in the backward, of its gradient) to the dtype, and by the order of the fp32 row sums.
    Forward: at round-off in fp32 (64 units of 2^-24 of max |v| + 1); in 16-bit within the gates' slope (<= 1) times
    u |v| plus one rounding of the output, 2u (max |v| + 1). Gradients, relative to each one's largest magnitude: the
    fp32 row sums over 4K terms, 16 sqrt(4K) 2^-24; in 16-bit 8u for the roundings of v, dv and the output."""
    N = 37
    g = torch.Generator().manual_seed(K)
    z = (torch.randn(N, 4 * K, generator=g) * 3 + 1).to(dtype).cuda()
    c = torch.randn(N, K, generator=g).to(dtype).cuda()
    gain = (1 + 0.2 * torch.randn(4 * K, generator=g)).cuda()
    bias = (0.3 * torch.randn(4 * K, generator=g)).cuda()
    e_c, e_h = torch.randn(N, K, generator=g).to(dtype).cuda(), torch.randn(N, K, generator=g).to(dtype).cuda()
    leaves = [t.detach().requires_grad_() for t in (z, c, gain, bias)]
    fused = _ln_gates(*leaves)
    comp_leaves = [t.detach().requires_grad_() for t in (z, c, gain, bias)]
    v = layer_norm(comp_leaves[0], comp_leaves[2], comp_leaves[3], axis=1, segments=4)
    comp = fused_lstm_gates(comp_leaves[1], v, forget_bias=1.0)
    vmax = float(v.detach().abs().max())
    u = U[dtype]
    tol = 64 * 2.0 ** -24 * (vmax + 1) if dtype == torch.float32 else 2 * u * (vmax + 1)
    for a, b, name in zip(fused, comp, ("c_next", "h_next")):
        assert float((a.double() - b.double()).abs().max()) <= tol, name
    ga = torch.autograd.grad(fused, leaves, (e_c, e_h))
    gb = torch.autograd.grad(comp, comp_leaves, (e_c, e_h))
    for a, b, name in zip(ga, gb, ("dz", "dc", "dgain", "dbias")):
        scale = float(b.double().abs().max()) + 1e-30
        err = float((a.double() - b.double()).abs().max()) / scale
        assert err <= (16 * 2.0 ** -24 * math.sqrt(4 * K) if dtype == torch.float32 else 8 * u), "%s %.3e" % (name, err)


class _LnGates(torch.autograd.Function):
    """The fused step alone through the raw entries: (c_next, h_next) of z (N, 4K) and c (N, K)."""

    @staticmethod
    def forward(ctx, z, c, g, b):
        N, K = c.shape
        lib = _lib.load()
        cn, hn = torch.empty_like(c), torch.empty_like(c)
        mean = torch.empty(N, 4, device=c.device)
        rstd = torch.empty_like(mean)
        dt, gdt = _lib.dtype_code(c.dtype), _lib.dtype_code(g.dtype)
        _lib.check(lib.bsmm_lstm_ln_gates(dt, gdt, c.data_ptr(), z.data_ptr(), z.stride(0), g.data_ptr(), b.data_ptr(),
                                          cn.data_ptr(), hn.data_ptr(), mean.data_ptr(), rstd.data_ptr(), N, K, 1e-6,
                                          1.0, _lib.stream_ptr()), "ln_gates")
        ctx.save_for_backward(z, c, g, b, mean, rstd)
        return cn, hn

    @staticmethod
    def backward(ctx, ec, eh):
        z, c, g, b, mean, rstd = ctx.saved_tensors
        N, K = c.shape
        lib = _lib.load()
        dz, dc = torch.empty_strided(z.shape, z.stride(), dtype=z.dtype, device=z.device), torch.empty_like(c)
        dg, db = torch.empty_like(g), torch.empty_like(b)
        ws = torch.empty(lib.bsmm_lstm_ln_gates_workspace_bytes(N, K) // 4, device=c.device)
        dt, gdt = _lib.dtype_code(c.dtype), _lib.dtype_code(g.dtype)
        _lib.check(lib.bsmm_lstm_ln_gates_grad(dt, gdt, c.data_ptr(), z.data_ptr(), z.stride(0), g.data_ptr(),
                                               b.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                                               ec.contiguous().data_ptr(), eh.contiguous().data_ptr(), dc.data_ptr(),
                                               dz.data_ptr(), ws.data_ptr(), 0, N, K, 1.0, _lib.stream_ptr()), "grad")
        _lib.check(lib.bsmm_lstm_ln_gates_grad_reduce(gdt, ws.data_ptr(), N, K, dg.data_ptr(), db.data_ptr(),
                                                      _lib.stream_ptr()), "reduce")
        return dz, dc, dg, db


def _ln_gates(z, c, g, b):
    return _LnGates.apply(z, c, g, b)


# ---- the kernel's gradient is one dw_matmul_large_n ------------------------------------------------------------------------
@pytest.mark.parametrize("layernorm", [True, False], ids=["ln", "noln"])
@pytest.mark.parametrize("shape", SHAPES[:2], ids=["blocks", "odd"])
def test_kernel_gradient_is_one_dw_matmul_over_the_saved_rows(monkeypatch, layernorm, shape):
    N, T, In, W, _ = shape
    calls = []

    def recording(x, e, **kw):
        u = dw_matmul_large_n(x, e, **kw)
        calls.append((x.clone(), e.clone(), u))
        return u

    monkeypatch.setattr(lstm_layer, "dw_matmul_large_n", recording)
    ins = _make(N, T, In, W, torch.bfloat16, seed=9, layernorm=layernorm)
    res = _run(*ins, layernorm, T, W)
    assert len(calls) == 1
    xr, er, u = calls[0]
    x, h0 = ins[0], ins[2]
    hs = torch.cat([h0[None], res[0].transpose(0, 1)[:-1]], 0)              # h_{t-1} for t = 0 .. T-1
    rows = torch.cat([x.transpose(0, 1), hs], 2).reshape(T * N, In + W)
    _same(xr, rows, "saved rows [x_t, h_{t-1}]")
    assert tuple(er.shape) == (T * N, 4 * W)
    _same(res[6], u, "dkernel")
    _same(dw_matmul_large_n(rows, er), res[6], "dkernel against a fresh call")


# ---- determinism and execution contexts ------------------------------------------------------------------------------------
def _all(seed, layernorm=True):
    return _make(7, 3, 13, 20, torch.bfloat16, seed=seed, layernorm=layernorm)


def test_two_runs_are_bitwise_identical():
    for layernorm in (True, False):
        ins = _all(0, layernorm)
        for a, b in zip(_run(*ins, layernorm, 3, 20), _run(*ins, layernorm, 3, 20)):
            _same(a, b, "second run")


def test_side_stream_and_graph_replay():
    static = list(_all(0))
    ref = _run(*static, True, 3, 20)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(1 << 22)
        bufs = [t.clone() for t in static]
        out = _run(*bufs, True, 3, 20)
    s.synchronize()
    for a, r in zip(out, ref):
        _same(a, r, "side stream")
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            _run(*static, True, 3, 20)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = _run(*static, True, 3, 20)
    for i in range(1, 3):
        new = _all(i)
        for t, n in zip(static, new):
            t.copy_(n)
        graph.replay()
        for a, r in zip(captured, _run(*new, True, 3, 20)):
            _same(a, r, "replay %d" % i)


# ---- element offsets past 2^31 ---------------------------------------------------------------------------------------------
def test_fused_kernels_past_2_31_elements():
    """bf16, z (N, 4K) with a padded row stride: the rows past element 2^31 equal the same rows run alone, bit for bit."""
    K = 1 << 13
    stride = 4 * K + 64
    N = (1 << 31) // stride + 8
    assert N * stride > 2 ** 31
    free, _ = torch.cuda.mem_get_info()
    if free < 16 * 2 ** 30:
        pytest.skip("needs 16 GB of free device memory")
    torch.manual_seed(0)
    zbuf = torch.randn(N, stride, device="cuda", dtype=torch.bfloat16)
    z = zbuf[:, :4 * K]
    c = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    g, b = torch.ones(4 * K, device="cuda"), torch.zeros(4 * K, device="cuda")
    cn, hn = _LnGates.forward(_Ctx(), z, c, g, b)
    cs, hs = _LnGates.forward(_Ctx(), z[-5:], c[-5:], g, b)
    _same(cn[-5:], cs, "c_next past 2^31")
    _same(hn[-5:], hs, "h_next past 2^31")
    del cn, hn
    eh = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    ctx = _Ctx()
    _LnGates.forward(ctx, z, c, g, b)
    dz, dc = _LnGates.backward(ctx, eh, eh)[:2]
    ctx = _Ctx()
    _LnGates.forward(ctx, z[-5:], c[-5:], g, b)
    dzs, dcs = _LnGates.backward(ctx, eh[-5:], eh[-5:])[:2]
    _same(dz[-5:, :4 * K], dzs[:, :4 * K], "dz past 2^31")
    _same(dc[-5:], dcs, "dc past 2^31")
    torch.cuda.synchronize()
    assert _lib.device_error() == 0


class _Ctx(object):
    """Stands in for autograd's ctx when _LnGates is driven directly."""

    def save_for_backward(self, *ts):
        self.saved_tensors = ts
